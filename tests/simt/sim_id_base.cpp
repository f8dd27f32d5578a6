// sim_id_base.cpp -- id bases (cfbpe_vocab_set_id_base) on the CPU SIMT emulator (tests/simt/cusim.h).
// TEST INFRASTRUCTURE: built by tests/simt/id_base_lib.py into tests/simt/_build/libcfbpe_sim_id_base.so and loaded only by the non-GPU
// tests.  The kernels and the launch sequences (csrc/bpe_kernels.cuh, csrc/pipeline.cuh, csrc/specials.cuh) and the host checks
// (csrc/specials.h) are the product sources, compiled unchanged.  The vocabularies come in as packed table blobs (simlib.SimVocab).
#include "cusim.h"

#define CFBPE_LAUNCH(kernel, grid, block, stream, ...) cusim::launch((grid), (block), [&] { kernel(__VA_ARGS__); })
#define CFBPE_LAUNCH_SMEM(kernel, grid, block, smem, stream, ...) cusim::launch((grid), (block), [&] { kernel(__VA_ARGS__); })
#define CFBPE_ZERO(ptr, bytes, stream) std::memset((ptr), 0, (bytes))
#define CFBPE_MARK(prof, idx, stream, begin) ((void)0)
#define CFBPE_FORK(main, aux, ev) ((void)0)
#define CFBPE_JOIN(main, aux, ev) ((void)0)

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <type_traits>
#include <vector>

template <typename T> inline T atomicAnd(T* p, T v) { T o = *p; *p = o & v; return o; }   // (specials.cuh's; not in cusim.h)

#include "../../cyberfabric-core_b200/csrc/pipeline.cuh"
#include "../../cyberfabric-core_b200/csrc/specials.cuh"
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

static VocabSet vocab_set(const uint8_t* const* blobs, uint32_t n_vocabs) {
    VocabSet vs{};
    for (uint32_t i = 0; i < kMaxVocabs; ++i) {
        const uint8_t* blob = blobs[i < n_vocabs ? i : 0];
        TablesHeader h;
        std::memcpy(&h, blob, sizeof h);
        vs.v[i] = make_view(blob, h);
    }
    vs.loaded_mask = (1u << n_vocabs) - 1u;
    return vs;
}

// the workspace of one pass over `total` bytes (workspace_extent), on host memory
struct Ws {
    std::vector<std::vector<uint64_t>> store;
    DeviceStatus st{};
    Workspace w{};
    explicit Ws(uint64_t total) {
        const WsSizes s = workspace_extent(total);
        for_each_ws_buffer(w, [&](auto*& p, WsKind kind) {
            store.emplace_back((s.n[kind] * sizeof(*p) + 7) / 8 + 1);
            p = reinterpret_cast<std::remove_reference_t<decltype(*p)>*>(store.back().data());
        });
        set_workspace_caps(w, s);
        w.status = &st;
    }
};

// special tables of the vocabularies: n[v] specials of vocabulary v, their bytes / offsets / ids concatenated over v (n == NULL: none)
static std::vector<std::vector<uint32_t>> special_tables(uint32_t n_vocabs, const uint32_t* n, const uint8_t* bytes, const uint64_t* offsets,
                                                         const uint32_t* ids) {
    std::vector<std::vector<uint32_t>> t(kMaxVocabs);
    uint64_t k0 = 0;
    for (uint32_t v = 0; n && v < n_vocabs; ++v) {
        std::vector<uint64_t> offs(offsets + k0, offsets + k0 + n[v] + 1);
        std::string e;
        if (n[v] && build_special_table(n[v], bytes, offs.data(), ids + k0, t[v], e)) { std::fprintf(stderr, "%s\n", e.c_str()); std::abort(); }
        k0 += n[v];
    }
    return t;
}

extern "C" {

// cfbpe_encode_batch on host memory, cut into sub-batches at prompts cuts[0] = 0 < ... < cuts[n_cuts] = n_prompts, as a pipelined host
// call runs them: every sub-batch is an encode pass of its own whose token ranks continue the previous one's (token_base), its
// offsets in the lane layout (sub_batch_offsets_at), then the rebase on its ids.  bases: the id base of every vocabulary slot, or NULL
// (no rebase: the ids are ranks, as before id bases existed).  out_offsets gets the call's n_prompts + 1 offsets.
__attribute__((visibility("default"))) int sim_encode_based(const uint8_t* const* blobs, uint32_t n_vocabs, const uint32_t* bases, uint32_t n_prompts,
                                                            const uint8_t* bytes, const uint64_t* offsets, const uint8_t* vocab_ids, const uint32_t* cuts,
                                                            uint32_t n_cuts, uint32_t* out_ids, uint64_t out_cap, uint64_t* out_offsets) {
    const VocabSet vs = vocab_set(blobs, n_vocabs);
    IdBases ib{};
    for (uint32_t v = 0; bases && v < kMaxVocabs; ++v) ib.v[v] = bases[v < n_vocabs ? v : 0];
    std::vector<uint64_t> lane_offsets(n_prompts + 1 + n_cuts), local(n_prompts + 1 + n_cuts);
    std::vector<uint32_t> counts(n_prompts + 1);
    uint64_t prev_end = 0;
    for (uint32_t k = 0; k < n_cuts; ++k) {
        const uint32_t p0 = cuts[k], p1 = cuts[k + 1], nk = p1 - p0;
        const uint64_t o0 = offsets[p0], len = offsets[p1] - o0, q0 = sub_batch_offsets_at(p0, k);
        for (uint32_t i = 0; i <= nk; ++i) local[q0 + i] = offsets[p0 + i] - o0;
        std::vector<uint8_t> sub(len + 64, 0);
        std::memcpy(sub.data(), bytes + o0, len);
        const BatchView b{sub.data(), local.data() + q0, vocab_ids ? vocab_ids + p0 : nullptr, nk, len};
        Ws ws(len);
        int* prof = nullptr;
        enqueue_encode(b, vs, uc_tables(), ws.w, out_ids, out_cap, lane_offsets.data() + q0, counts.data() + p0, 4u, 0, 0, 0, 0, 0, 0, prof,
                       k ? &prev_end : nullptr);
        enqueue_rebase(b, bases ? &ib : nullptr, out_ids, lane_offsets.data() + q0, out_cap, ws.w.status, 0);
        if (const int rc = status_error(ws.st).code) return rc;
        prev_end = ws.st.tok_end;
        for (uint32_t i = 0; i <= nk; ++i) out_offsets[p0 + i] = lane_offsets[q0 + i];
    }
    return prev_end > out_cap ? CFBPE_ENOSPC : 0;
}

// cfbpe_encode_batch_special with every special ALLOWED, on host memory, as enqueue_special_call runs it: the scan, then the ordinary
// path on the prompts as they are (no match; the rebase follows it) or on the stretches (the rebase runs on their ids before the
// splice).  Specials: n_sp[v] of vocabulary v (special_tables).  *spliced: which of the two ran.
__attribute__((visibility("default"))) int sim_encode_special_based(const uint8_t* const* blobs, uint32_t n_vocabs, const uint32_t* bases,
                                                                    const uint32_t* n_sp, const uint8_t* sp_bytes, const uint64_t* sp_offsets,
                                                                    const uint32_t* sp_ids, uint32_t n_prompts, const uint8_t* bytes,
                                                                    const uint64_t* offsets, const uint8_t* vocab_ids, uint32_t* out_ids, uint64_t out_cap,
                                                                    uint64_t* out_offsets, int* spliced) {
    const VocabSet vs = vocab_set(blobs, n_vocabs);
    IdBases ib{};
    for (uint32_t v = 0; bases && v < kMaxVocabs; ++v) ib.v[v] = bases[v < n_vocabs ? v : 0];
    const std::vector<std::vector<uint32_t>> tables = special_tables(n_vocabs, n_sp, sp_bytes, sp_offsets, sp_ids);
    std::vector<std::vector<uint8_t>> modes(kMaxVocabs);
    const uint32_t* words[kMaxVocabs] = {};
    SpecialView views[kMaxVocabs] = {};
    const uint8_t* mode_ptrs[kMaxVocabs] = {};
    for (uint32_t v = 0; v < kMaxVocabs; ++v) {
        if (tables[v].empty()) continue;
        words[v] = tables[v].data();
        views[v] = make_special_view(tables[v].data(), tables[v]);
        modes[v].assign(tables[v][0], kSpAllow);
        mode_ptrs[v] = modes[v].data();
    }
    SpecialSet sp;
    bool scan = false;
    uint32_t bad[2];
    if (fill_special_set(words, views, mode_ptrs, &sp, &scan, bad)) return CFBPE_EINVAL;
    const uint64_t total = offsets[n_prompts], mp = n_prompts + 2 * total + 2;     // (room for a match at every byte)
    std::vector<uint8_t> placed(total + 64, 0);
    std::memcpy(placed.data(), bytes, total);
    const BatchView b{placed.data(), offsets, vocab_ids, n_prompts, total};
    Ws ws(total);
    std::vector<uint32_t> kept_n(mp + 1), st_id(mp + 1), ord_ids(total + 1), ord_counts(mp + 1), counts(n_prompts + 1);
    std::vector<uint64_t> kept_base(mp + 1), st_off(mp + 2), st_base(mp + 1), ord_offsets(mp + 2);
    std::vector<uint8_t> st_vocab(mp + 1);
    SpecialStatus ss{};
    const SpecialWork sw{kept_n.data(), kept_base.data(), st_off.data(), st_vocab.data(), st_id.data(), st_base.data(), &ss};
    uint64_t n_str = n_prompts;
    if (scan) {
        enqueue_special_scan(b, sp, ws.w, sw, 0);
        const SpecialScanResult r = special_scan_result(ss, n_prompts, static_cast<uint32_t>(mp));
        if (!r.fits) return CFBPE_EINVAL;
        n_str = r.n_stretches;
    }
    int* prof = nullptr;
    const IdBases* bp = bases ? &ib : nullptr;
    *spliced = n_str != n_prompts;
    uint64_t n_tokens;
    if (!*spliced) {
        enqueue_encode(b, vs, uc_tables(), ws.w, out_ids, out_cap, out_offsets, counts.data(), 4u, 0, 0, 0, 0, 0, 0, prof);
        enqueue_rebase(b, bp, out_ids, out_offsets, out_cap, ws.w.status, 0);
        n_tokens = ws.st.n_tokens;
    } else {
        enqueue_encode_special(b, sp, vs, uc_tables(), ws.w, sw, static_cast<uint32_t>(n_str), ord_ids.data(), total + 1, ord_offsets.data(),
                               ord_counts.data(), out_ids, out_cap, out_offsets, counts.data(), 4u, 0, 0, 0, 0, 0, 0, prof, bp);
        n_tokens = ss.fin.n_tokens;
    }
    if (const int rc = status_error(ws.st).code) return rc;
    return n_tokens > out_cap ? CFBPE_ENOSPC : 0;
}

// the decode path with id bases (bases: every slot's base, NULL: none) and special tables (special_tables); returns 0, CFBPE_EINVAL
// for an id that is neither an ordinary token under its base nor a special token, or CFBPE_ENOSPC
__attribute__((visibility("default"))) int sim_decode_based(const uint8_t* const* blobs, uint32_t n_vocabs, const uint32_t* bases, const uint32_t* n_sp,
                                                            const uint8_t* sp_bytes, const uint64_t* sp_offsets, const uint32_t* sp_ids, uint32_t n_seqs,
                                                            const uint32_t* ids, const uint64_t* id_offsets, const uint8_t* vocab_ids, uint8_t* out,
                                                            uint64_t out_cap, uint64_t* out_offsets) {
    const VocabSet vs = vocab_set(blobs, n_vocabs);
    IdBases ib{};
    for (uint32_t v = 0; bases && v < kMaxVocabs; ++v) ib.v[v] = bases[v < n_vocabs ? v : 0];
    const std::vector<std::vector<uint32_t>> tables = special_tables(n_vocabs, n_sp, sp_bytes, sp_offsets, sp_ids);
    SpecialSet sp{};
    for (uint32_t v = 0; v < kMaxVocabs; ++v) if (!tables[v].empty()) sp.v[v] = make_special_view(tables[v].data(), tables[v]);
    const uint64_t n_ids = id_offsets[n_seqs];
    const DecodeView d{ids, id_offsets, vocab_ids, n_seqs, n_ids};
    const uint32_t n_tiles = static_cast<uint32_t>((n_ids + kDecodeTile - 1) / kDecodeTile);
    std::vector<uint32_t> lens(n_ids + 1), sums(n_tiles + 1);
    std::vector<uint64_t> base(n_tiles + 1);
    DeviceStatus st{};
    if (n_tiles) cusim::launch(n_tiles, 256, [&] { decode_len_kernel(d, vs, lens.data(), sums.data(), &st, sp, ib); });
    cusim::launch(1u, n_tiles ? 1024u : 32u, [&] { tile_scan_kernel(sums.data(), n_tiles, base.data(), &st, nullptr); });
    if (st.bad_utf8) return CFBPE_EINVAL;
    if (n_tiles) cusim::launch(n_tiles, 256, [&] { decode_copy_kernel(d, vs, lens.data(), base.data(), out, out_cap, sp, ib); });
    cusim::launch(static_cast<unsigned>((static_cast<uint64_t>(n_seqs) + 1 + 255) / 256), 256, [&] { decode_offsets_kernel(d, lens.data(), base.data(), out_offsets, &st); });
    return st.tok_end > out_cap ? CFBPE_ENOSPC : 0;
}

// the check cfbpe_vocab_set_id_base and cfbpe_vocab_set_specials make (special_in_id_range) on a table of n specials
__attribute__((visibility("default"))) int sim_special_in_id_range(uint32_t n, const uint8_t* bytes, const uint64_t* offsets, const uint32_t* ids,
                                                                   uint32_t base, uint32_t n_ranks) {
    std::vector<uint32_t> words;
    std::string e;
    if (build_special_table(n, bytes, offsets, ids, words, e)) return -2;
    return special_in_id_range(words, base, n_ranks);
}

}  // extern "C"
