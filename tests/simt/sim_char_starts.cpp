// sim_char_starts.cpp -- cfbpe_encode_batch_char_starts on the CPU SIMT emulator (tests/simt/cusim.h).
// TEST INFRASTRUCTURE: built by tests/simt/char_starts_lib.py into tests/simt/_build/libcfbpe_sim_char_starts.so and loaded only by
// the non-GPU tests.  The kernels and the launch sequence (csrc/bpe_kernels.cuh, csrc/pipeline.cuh) are the product sources, compiled
// unchanged.  The vocabularies come in as the packed table blobs the table builder makes (simlib.SimVocab.blob()).
#include "cusim.h"

#define CFBPE_LAUNCH(kernel, grid, block, stream, ...) cusim::launch((grid), (block), [&] { kernel(__VA_ARGS__); })
#define CFBPE_LAUNCH_SMEM(kernel, grid, block, smem, stream, ...) cusim::launch((grid), (block), [&] { kernel(__VA_ARGS__); })
#define CFBPE_ZERO(ptr, bytes, stream) std::memset((ptr), 0, (bytes))
#define CFBPE_MARK(prof, idx, stream, begin) ((void)0)
#define CFBPE_FORK(main, aux, ev) ((void)0)
#define CFBPE_JOIN(main, aux, ev) ((void)0)

#include <algorithm>
#include <cstring>
#include <type_traits>
#include <vector>

#include "../../cyberfabric-core_b200/csrc/pipeline.cuh"
#include "../../cyberfabric-core_b200/csrc/pretok_ctx.h"
#include "../../cyberfabric-core_b200/csrc/unicode_tables.h"
#include "../../include/cfbpe.h"

using namespace cfbpe;

static UcTables uc_tables() {
    static uint16_t fsm[kNumPatterns * kPretokTableSize];
    static uint8_t ascii[128];
    static SplitTablesHost st;
    static bool init = false;
    if (!init) { build_pretok_tables(fsm); build_ascii_classes(ascii); build_split_tables(&st); init = true; }
    return UcTables{cfbpe_uc_stage1, cfbpe_uc_stage2, ascii, fsm, st.cls256, st.fsm16, st.ctx16, st.prod, st.prod_info, st.prod_skip, st.prod_start};
}

extern "C" {

// cfbpe_encode_batch_char_starts on host memory, one pass as run_lane without pipelining.  blobs: the packed tables of n_vocabs
// vocabularies (slots past n_vocabs alias slot 0, as the library's unloaded slots do); unit: a CFBPE_UNIT_* value; out_starts: room
// for out_cap entries; out_lens: n_prompts entries or NULL.  The batch gets 64 zero bytes of padding; the workspace is the extent of
// one pass (workspace_extent).
__attribute__((visibility("default"))) int sim_encode_batch_char_starts(const uint8_t* const* blobs, uint32_t n_vocabs, uint32_t n_prompts,
                                                                        const uint8_t* bytes, const uint64_t* offsets, const uint8_t* vocab_ids,
                                                                        uint32_t unit, uint32_t* out_ids, uint32_t* out_starts, uint64_t out_cap,
                                                                        uint64_t* out_offsets, uint32_t* out_counts, uint32_t* out_lens) {
    if (unit_args_error(unit, out_ids, out_starts)) return CFBPE_EINVAL;
    if (!n_vocabs) return CFBPE_ENOENT;
    VocabSet vs{};
    for (uint32_t i = 0; i < kMaxVocabs; ++i) {
        const uint8_t* blob = blobs[i < n_vocabs ? i : 0];
        TablesHeader h;
        std::memcpy(&h, blob, sizeof h);
        vs.v[i] = make_view(blob, h);
    }
    vs.loaded_mask = n_vocabs >= 32 ? 0xFFFFFFFFu : ((1u << n_vocabs) - 1u);
    const uint64_t total = offsets[n_prompts];
    std::vector<uint8_t> padded(total + 64, 0);
    if (total) std::memcpy(padded.data(), bytes, total);
    const BatchView b{padded.data(), offsets, vocab_ids, n_prompts, total};

    std::vector<std::vector<uint64_t>> store;
    DeviceStatus st{};
    Workspace w{};
    const WsSizes s = workspace_extent(total);
    for_each_ws_buffer(w, [&](auto*& p, WsKind kind) {
        store.emplace_back((s.n[kind] * sizeof(*p) + 7) / 8);
        p = reinterpret_cast<std::remove_reference_t<decltype(*p)>*>(store.back().data());
    });
    set_workspace_caps(w, s);
    w.status = &st;

    const UnitView uv{unit == CFBPE_UNIT_UTF16 ? 1u : 0u, out_lens};
    int* prof = nullptr;
    enqueue_encode(b, vs, uc_tables(), w, out_ids, out_cap, out_offsets, out_counts, 4u, 0, 0, 0, 0, 0, 0, prof, nullptr, out_starts,
                   nullptr, nullptr, &uv);
    if (const int rc = status_error(st).code) return rc;
    if (st.n_tokens > out_cap) { out_offsets[n_prompts] = st.n_tokens; return CFBPE_ENOSPC; }
    return 0;
}

}  // extern "C"
