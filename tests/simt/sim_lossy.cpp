// sim_lossy.cpp -- cfbpe_encode_batch_lossy on the CPU SIMT emulator (tests/simt/cusim.h).
// TEST INFRASTRUCTURE: built by tests/simt/lossy_lib.py into tests/simt/_build/libcfbpe_sim_lossy.so and loaded only by the non-GPU
// tests.  The kernels and the launch sequence (csrc/utf8_repair.cuh, csrc/bpe_kernels.cuh, csrc/pipeline.cuh) are the product
// sources, compiled unchanged.  The vocabularies come in as the packed table blobs the table builder makes (simlib.SimVocab.blob()).
#include "cusim.h"

#define CFBPE_LAUNCH(kernel, grid, block, stream, ...) cusim::launch((grid), (block), [&] { kernel(__VA_ARGS__); })
#define CFBPE_LAUNCH_SMEM(kernel, grid, block, smem, stream, ...) cusim::launch((grid), (block), [&] { kernel(__VA_ARGS__); })
#define CFBPE_ZERO(ptr, bytes, stream) std::memset((ptr), 0, (bytes))
#define CFBPE_MARK(prof, idx, stream, begin) ((void)0)
#define CFBPE_FORK(main, aux, ev) ((void)0)
#define CFBPE_JOIN(main, aux, ev) ((void)0)

#include <sys/mman.h>
#include <unistd.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <type_traits>
#include <vector>

#include "../../cyberfabric-core_b200/csrc/pipeline.cuh"
#include "../../cyberfabric-core_b200/csrc/pretok_ctx.h"
#include "../../cyberfabric-core_b200/csrc/unicode_tables.h"
#include "../../cyberfabric-core_b200/csrc/utf8_repair.cuh"
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

// The batch's bytes in their own mapping: the first byte at an address = misalign (mod 16), `fill` repeated over the bytes before
// it and the padding after the last one.  guard 0: 64 bytes of padding; 1: exactly 32 bytes of padding (what include/cfbpe.h asks
// of a caller), then a PROT_NONE page (misalign not used); 2: a PROT_NONE page before the page that holds the first byte.  An
// access to a guard page stops the process with SIGSEGV.
struct PlacedBytes {
    uint8_t* p = nullptr;
    void* map = nullptr;
    size_t map_len = 0;
    PlacedBytes(const uint8_t* bytes, uint64_t total, uint32_t misalign, const uint8_t* fill, uint32_t n_fill, uint32_t guard) {
        const size_t page = static_cast<size_t>(sysconf(_SC_PAGESIZE));
        const uint64_t pad = guard == 1 ? 32 : 64, lead = guard == 1 ? 0 : misalign;
        const size_t readable = (lead + total + pad + page - 1) / page * page;
        map_len = readable + (guard ? page : 0);
        map = mmap(nullptr, map_len, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
        if (map == MAP_FAILED) { std::perror("mmap"); std::abort(); }
        uint8_t* r = static_cast<uint8_t*>(map);
        if (guard == 2) r += page;
        p = guard == 1 ? r + readable - pad - total : r + lead;
        for (uint8_t* q = r; q < p; ++q) *q = fill[static_cast<size_t>(q - r) % n_fill];
        if (total) std::memcpy(p, bytes, total);
        for (uint64_t i = 0; i < pad; ++i) p[total + i] = fill[i % n_fill];
        if (guard == 1 && mprotect(r + readable, page, PROT_NONE)) { std::perror("mprotect"); std::abort(); }
        if (guard == 2 && mprotect(map, page, PROT_NONE)) { std::perror("mprotect"); std::abort(); }
    }
    ~PlacedBytes() { munmap(map, map_len); }
    PlacedBytes(const PlacedBytes&) = delete;
    PlacedBytes& operator=(const PlacedBytes&) = delete;
};

extern "C" {

// cfbpe_encode_batch_lossy on host memory, one pass as run_lane_lossy: the scan, the host's look at its status (lossy_scan_result),
// then the ordinary path on the bytes as they are, or the repair and the ordinary path on the repaired batch R.  blobs: the packed
// tables of n_vocabs vocabularies (slots past n_vocabs alias slot 0); max_bytes: the context's max_batch_bytes (R above it is
// CFBPE_EINVAL); misalign / fill / guard: where the batch's bytes lie (PlacedBytes).  status_out: the scan's status word;
// *repaired: whether the repair ran, and then out_r (room for r_cap bytes) and out_r_offsets (n_prompts + 1) get R and its
// offsets.  R lies in a buffer whose padding is 0xFF; the workspace has room for three times the batch.
__attribute__((visibility("default"))) int sim_encode_batch_lossy(const uint8_t* const* blobs, uint32_t n_vocabs, uint32_t n_prompts,
                                                                  const uint8_t* bytes, const uint64_t* offsets, const uint8_t* vocab_ids,
                                                                  uint32_t* out_ids, uint64_t out_cap, uint64_t* out_offsets, uint32_t* out_counts,
                                                                  uint32_t* out_replaced, uint64_t max_bytes, uint32_t misalign,
                                                                  const uint8_t* fill, uint32_t n_fill, uint32_t guard, uint8_t* out_r, uint64_t r_cap,
                                                                  uint64_t* out_r_offsets, uint64_t* status_out, int* repaired) {
    if (!n_vocabs) return CFBPE_ENOENT;
    if (misalign > 15 || !fill || !n_fill || guard > 2) return CFBPE_EINVAL;
    VocabSet vs{};
    for (uint32_t i = 0; i < kMaxVocabs; ++i) {
        const uint8_t* blob = blobs[i < n_vocabs ? i : 0];
        TablesHeader h;
        std::memcpy(&h, blob, sizeof h);
        vs.v[i] = make_view(blob, h);
    }
    vs.loaded_mask = n_vocabs >= 32 ? 0xFFFFFFFFu : ((1u << n_vocabs) - 1u);
    const uint64_t total = offsets[n_prompts];
    const PlacedBytes placed(bytes, total, misalign, fill, n_fill, guard);
    const BatchView b{placed.p, offsets, vocab_ids, n_prompts, total};

    std::vector<std::vector<uint64_t>> store;
    DeviceStatus st{};
    Workspace w{};
    const WsSizes s = workspace_extent(3 * total);
    for_each_ws_buffer(w, [&](auto*& p, WsKind kind) {
        store.emplace_back((s.n[kind] * sizeof(*p) + 7) / 8);
        p = reinterpret_cast<std::remove_reference_t<decltype(*p)>*>(store.back().data());
    });
    set_workspace_caps(w, s);
    w.status = &st;
    for (uint32_t* p : {w.ids_by_pos, w.dense.by_piece, w.dense.extras}) std::fill_n(p, s.n[kWsPerByte], 0xDEADBEEFu);

    std::vector<uint32_t> replaced(n_prompts + 1, 0xDEADBEEFu);
    std::vector<uint64_t> r_offsets(n_prompts + 1, ~0ull);
    LossyStatus lst{~0ull};
    const LossyWork lw{replaced.data(), r_offsets.data(), &lst};
    enqueue_utf8_scan(b, vs, w, lw, 0);
    *status_out = lst.lanes_growth;
    const LossyScanResult r = lossy_scan_result(lst, total);
    *repaired = 0;
    BatchView eb = b;
    std::vector<uint8_t> rbuf;
    if (r.dirty) {
        if (r.total > max_bytes) return CFBPE_EINVAL;
        rbuf.assign(r.total + 64, 0xFFu);
        enqueue_utf8_repair(b, w, lw, rbuf.data(), r.total, 0);
        *repaired = 1;
        if (out_r && r_cap >= r.total) std::memcpy(out_r, rbuf.data(), r.total);
        std::memcpy(out_r_offsets, r_offsets.data(), (static_cast<uint64_t>(n_prompts) + 1) * sizeof(uint64_t));
        eb = BatchView{rbuf.data(), r_offsets.data(), vocab_ids, n_prompts, r.total};
    }
    int* prof = nullptr;
    enqueue_encode(eb, vs, uc_tables(), w, out_ids, out_cap, out_offsets, out_counts, 4u, 0, 0, 0, 0, 0, 0, prof);
    if (out_replaced && n_prompts) std::memcpy(out_replaced, replaced.data(), n_prompts * sizeof(uint32_t));
    if (const int rc = status_error(st).code) return rc;
    if (out_ids && st.n_tokens > out_cap) { out_offsets[n_prompts] = st.n_tokens; return CFBPE_ENOSPC; }
    return 0;
}

}  // extern "C"
