// sim_harness.cpp -- runs the product's CUDA kernels on the CPU SIMT emulator (tests/simt/cusim.h).
// TEST INFRASTRUCTURE: built by tests/simt/build.py into tests/simt/_build/libcfbpe_sim.so and
// loaded only by the non-GPU tests, through tests/simt/simlib.py.  The table builder (csrc/vocab.cpp), the kernels
// (csrc/bpe_kernels.cuh, csrc/pipeline.cuh, csrc/specials.cuh) and the special-token host code (csrc/specials.h) are the
// product sources, compiled unchanged.
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
#include <memory>
#include <string>
#include <type_traits>
#include <vector>

template <typename T> inline T atomicAnd(T* p, T v) { T o = *p; *p = o & v; return o; }   // (specials.cuh's; not in cusim.h)

#include "../../cyberfabric-core_b200/csrc/pipeline.cuh"
#include "../../cyberfabric-core_b200/csrc/specials.cuh"
#include "../../cyberfabric-core_b200/csrc/pretok_ctx.h"
#include "../../cyberfabric-core_b200/csrc/subbatch.h"
#include "../../cyberfabric-core_b200/csrc/unicode_tables.h"
#include "../../cyberfabric-core_b200/csrc/vocab.h"
#include "../../include/cfbpe.h"

using namespace cfbpe;

struct SimVocab {
    std::vector<uint8_t> blob;
    TablesHeader hdr;
};
struct SimSpecials { std::vector<uint32_t> words; };

static UcTables uc_tables() {
    static uint16_t fsm[kNumPatterns * kPretokTableSize];
    static uint8_t ascii[128];
    static SplitTablesHost st;
    static bool init = false;
    if (!init) { build_pretok_tables(fsm); build_ascii_classes(ascii); build_split_tables(&st); init = true; }
    return UcTables{cfbpe_uc_stage1, cfbpe_uc_stage2, ascii, fsm, st.cls256, st.fsm16, st.ctx16, st.prod, st.prod_info, st.prod_skip, st.prod_start};
}

// The workspace of one pass over `total` bytes on host memory: workspace_extent(total) elements of every buffer, as a one-shot
// call needs.  ids_by_pos, by_piece and extras start as 0xDEADBEEF (a slot the kernels never wrote shows), the rest as zero.
struct SimWorkspace {
    std::vector<std::vector<uint64_t>> store;
    DeviceStatus st{};
    Workspace w{};
    explicit SimWorkspace(uint64_t total) {
        const WsSizes s = workspace_extent(total);
        for_each_ws_buffer(w, [&](auto*& p, WsKind kind) {
            store.emplace_back((s.n[kind] * sizeof(*p) + 7) / 8);
            p = reinterpret_cast<std::remove_reference_t<decltype(*p)>*>(store.back().data());
        });
        set_workspace_caps(w, s);
        w.status = &st;
        for (uint32_t* p : {w.ids_by_pos, w.dense.by_piece, w.dense.extras}) std::fill_n(p, s.n[kWsPerByte], 0xDEADBEEFu);
    }
    SimWorkspace(const SimWorkspace&) = delete;
    SimWorkspace& operator=(const SimWorkspace&) = delete;
};

// Where every call puts its batch's bytes (sim_batch_layout; process-wide): the first prompt byte at an address = misalign
// (mod 16), the fill repeated over the mapped bytes before it and over the padding after the last prompt byte, and a guard:
//   kGuardNone    64 bytes of padding
//   kGuardAfter   exactly 32 bytes of padding (what include/cfbpe.h asks of a caller), then a PROT_NONE page; the start
//                 follows from the batch length, misalign is not used
//   kGuardBefore  the first byte misalign bytes into a page whose predecessor is PROT_NONE; 64 bytes of padding
// The default (misalign 0, fill one zero byte, no guard) is the layout every test had before layouts could be chosen.
enum : uint32_t { kGuardNone = 0, kGuardAfter = 1, kGuardBefore = 2 };
struct SimByteLayout {
    uint32_t misalign = 0, guard = kGuardNone;
    std::vector<uint8_t> fill{0};
};
static SimByteLayout g_layout;

// a batch's bytes placed by g_layout, unmapped on destruction (an access to a guard page stops the process with SIGSEGV)
struct SimBytes {
    uint8_t* p = nullptr;              // the first prompt byte
    void* map = nullptr;
    size_t map_len = 0;
    SimBytes(const uint8_t* bytes, uint64_t total) {
        const size_t page = static_cast<size_t>(sysconf(_SC_PAGESIZE));
        const SimByteLayout& L = g_layout;
        const uint64_t pad = L.guard == kGuardAfter ? 32 : 64;
        const uint64_t lead = L.guard == kGuardAfter ? 0 : L.misalign;
        const size_t readable = (lead + total + pad + page - 1) / page * page;
        map_len = readable + (L.guard == kGuardNone ? 0 : page);
        map = mmap(nullptr, map_len, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
        if (map == MAP_FAILED) { std::perror("mmap"); std::abort(); }
        uint8_t* r = static_cast<uint8_t*>(map);                  // the readable region [r, r + readable)
        if (L.guard == kGuardBefore) r += page;
        p = L.guard == kGuardAfter ? r + readable - pad - total : r + lead;
        const size_t n_fill = L.fill.size();
        for (uint8_t* q = r; q < p; ++q) *q = L.fill[static_cast<size_t>(q - r) % n_fill];
        if (total) std::memcpy(p, bytes, total);
        for (uint64_t i = 0; i < pad; ++i) p[total + i] = L.fill[i % n_fill];
        if (L.guard == kGuardAfter && mprotect(r + readable, page, PROT_NONE)) { std::perror("mprotect"); std::abort(); }
        if (L.guard == kGuardBefore && mprotect(map, page, PROT_NONE)) { std::perror("mprotect"); std::abort(); }
    }
    ~SimBytes() { munmap(map, map_len); }
    SimBytes(const SimBytes&) = delete;
    SimBytes& operator=(const SimBytes&) = delete;
};

// The VocabSet of a call over built vocabularies, unloaded slots aliasing slot 0 as the library's install_blob makes them, and,
// when the call has prompts (offsets != nullptr), its batch: the bytes placed by the current layout (SimBytes).
struct SimBatch {
    VocabSet vs{};
    std::unique_ptr<SimBytes> bytes;
    BatchView b{};
    SimBatch(void* const* vocabs, uint32_t n_vocabs, uint32_t n_prompts, const uint8_t* bytes, const uint64_t* offsets, const uint8_t* vocab_ids) {
        for (uint32_t i = 0; i < n_vocabs && i < kMaxVocabs; ++i) {
            SimVocab* v = static_cast<SimVocab*>(vocabs[i]);
            vs.v[i] = make_view(v->blob.data(), v->hdr);
        }
        for (uint32_t i = n_vocabs; i < kMaxVocabs && n_vocabs; ++i) vs.v[i] = vs.v[0];
        vs.loaded_mask = n_vocabs >= 32 ? 0xFFFFFFFFu : ((1u << n_vocabs) - 1u);
        if (!offsets) return;
        const uint64_t total = offsets[n_prompts];
        this->bytes = std::make_unique<SimBytes>(bytes, total);
        b = BatchView{this->bytes->p, offsets, vocab_ids, n_prompts, total};
    }
    SimBatch(const SimBatch&) = delete;
    SimBatch& operator=(const SimBatch&) = delete;
};

extern "C" __attribute__((visibility("default"))) uint32_t sim_ctx_count(uint32_t cased) { static SplitTablesHost st; build_split_tables(&st); return st.n_ctx[cased & 1]; }
extern "C" __attribute__((visibility("default"))) uint32_t sim_prod_count(uint32_t pat) { static SplitTablesHost st; build_split_tables(&st); return st.n_prod[pat & 3]; }

extern "C" {

// the layout of every later call's batch (SimBytes): 0, or CFBPE_EINVAL for misalign > 15, an empty fill or an unknown guard
__attribute__((visibility("default"))) int sim_batch_layout(uint32_t misalign, const uint8_t* fill, uint32_t fill_len, uint32_t guard) {
    if (misalign > 15 || !fill || !fill_len || guard > kGuardBefore) return CFBPE_EINVAL;
    g_layout.misalign = misalign;
    g_layout.guard = guard;
    g_layout.fill.assign(fill, fill + fill_len);
    return 0;
}

__attribute__((visibility("default"))) void* sim_vocab_build(const uint8_t* file, size_t len, uint32_t format,
                                                             uint32_t pattern, uint32_t max_ranks, char* err, size_t errcap) {
    std::vector<std::string> toks;
    std::string e;
    int rc = (format == CFBPE_FORMAT_TEKKEN_JSON) ? parse_tekken_json(file, len, max_ranks, toks, e)
                                                  : parse_tiktoken(file, len, max_ranks, toks, e);
    SimVocab* v = nullptr;
    if (rc == 0) {
        v = new SimVocab();
        rc = build_tables(toks, pattern, v->blob, e);
        if (rc == 0) rc = validate_tables(v->blob.data(), v->blob.size(), e);
        if (rc != 0) { delete v; v = nullptr; }
        else std::memcpy(&v->hdr, v->blob.data(), sizeof(TablesHeader));
    }
    if (!v && err && errcap) { std::snprintf(err, errcap, "%s", e.c_str()); }
    return v;
}
// the packed tables of a built vocabulary (what cfbpe_vocab_export hands out) and the check cfbpe_vocab_import runs on a blob
__attribute__((visibility("default"))) uint64_t sim_vocab_blob(void* vp, uint8_t* out, uint64_t cap) {
    SimVocab* v = static_cast<SimVocab*>(vp);
    if (out && cap >= v->blob.size()) std::memcpy(out, v->blob.data(), v->blob.size());
    return v->blob.size();
}
__attribute__((visibility("default"))) int sim_validate_blob(const uint8_t* blob, uint64_t size, char* err, size_t errcap) {
    std::string e;
    const int rc = validate_tables(blob, size, e);
    if (err && errcap) std::snprintf(err, errcap, "%s", e.c_str());
    return rc;
}
__attribute__((visibility("default"))) unsigned long long sim_dbg_counter(uint32_t i, int reset) {
    unsigned long long* c = cfbpe::dbg_counters();
    const unsigned long long v = c[i & 15];
    if (reset) c[i & 15] = 0;
    return v;
}
__attribute__((visibility("default"))) void sim_vocab_free(void* v) { delete static_cast<SimVocab*>(v); }
__attribute__((visibility("default"))) void sim_vocab_info(void* vp, cfbpe_vocab_info* out) {
    SimVocab* v = static_cast<SimVocab*>(vp);
    out->n_ranks = v->hdr.n_ranks; out->pattern_id = v->hdr.pattern_id; out->max_token_len = v->hdr.max_token_len;
    out->n_pair_entries = v->hdr.n_pair_entries; out->table_bytes = v->hdr.total_bytes;
}
// host-side lookups through the packed tables (table-builder tests)
__attribute__((visibility("default"))) uint32_t sim_piece_lookup(void* vp, const uint8_t* p, uint32_t n) {
    SimVocab* v = static_cast<SimVocab*>(vp);
    std::vector<uint8_t> tmp(p, p + n); tmp.resize(n + 16);
    return piece_lookup(make_view(v->blob.data(), v->hdr), tmp.data(), n);
}
__attribute__((visibility("default"))) uint32_t sim_pair_lookup(void* vp, uint32_t l, uint32_t r) {
    SimVocab* v = static_cast<SimVocab*>(vp);
    return pair_lookup(make_view(v->blob.data(), v->hdr), l, r);
}

// K1's bulk run scanners on n bytes placed by the current layout: ascii_digit_run_end (digits != 0) or same_byte_run_end(c) from
// pos, bounded by pe
__attribute__((visibility("default"))) uint64_t sim_run_end(uint32_t digits, const uint8_t* bytes, uint64_t n, uint64_t pos, uint64_t pe, uint32_t c) {
    const SimBytes placed(bytes, n);
    return digits ? ascii_digit_run_end(placed.p, pos, pe) : same_byte_run_end(placed.p, pos, pe, c);
}

// K1 only: piece-start bits (n_words+2 words) for a packed batch; patterns[] per vocab id
static unsigned long long fixups_seen = 0, resumes_seen = 0;
__attribute__((visibility("default"))) unsigned long long sim_split_fixups(int reset) { const unsigned long long v = fixups_seen; if (reset) fixups_seen = 0; return v; }
__attribute__((visibility("default"))) int sim_split(const uint32_t* patterns, uint32_t n_patterns, uint32_t n_prompts,
                                                     const uint8_t* bytes, const uint64_t* offsets, const uint8_t* vocab_ids,
                                                     uint32_t* piece_bits) {
    const uint64_t total = offsets[n_prompts];
    const SimBytes placed(bytes, total);
    BatchView b{placed.p, offsets, vocab_ids, n_prompts, total};
    VocabSet vs{};
    for (uint32_t i = 0; i < n_patterns && i < kMaxVocabs; ++i) vs.v[i].pattern_id = patterns[i];
    DeviceStatus st{};
    const uint64_t nw = n_flag_words(total);
    std::memset(piece_bits, 0, (nw + 2) * 4);
    vs.loaded_mask = n_patterns >= 32 ? 0xFFFFFFFFu : ((1u << n_patterns) - 1u);
    if (total) {
        UcTables uc = uc_tables();
        std::vector<SplitFix> fix(total / 16 + 2);
        const uint32_t fix_cap = static_cast<uint32_t>(fix.size());
        std::vector<uint32_t> pstart(nw + 2), bprompt((total >> kPromptBlockShift) + 2);
        cusim::launch(static_cast<unsigned>((static_cast<uint64_t>(n_prompts) + 1 + 255) / 256), 256, [&] { prompt_map_kernel(b, vs, pstart.data(), bprompt.data(), &st); });
        const uint64_t n_blocks16 = (total + 15) / 16;
        const uint32_t n_tiles = static_cast<uint32_t>((n_blocks16 + kSplitWarpOwned - 1) / kSplitWarpOwned);
        const uint32_t n_tabs = vocab_ids ? kNumPatterns : 1u;
        cusim::launch(n_tiles < 17 ? 1u : 2u, kSplitCta,      // fewer warps than tiles: the persistent loop runs
                      [&] { pretok_split16_kernel(b, vs, uc, pstart.data(), bprompt.data(), piece_bits, &st, fix.data(), fix_cap, n_tabs, n_tiles); });
        cusim::launch(2u, 256, [&] { pretok_fixup_kernel(b, vs, uc, piece_bits, &st, fix.data(), fix_cap); });
        fixups_seen += st.fix_n;
        resumes_seen += cfbpe::dbg_counters()[3] + cfbpe::dbg_counters()[4];
    }
    return st.bad_utf8 ? CFBPE_EILSEQ : 0;
}

// the whole path (K1..K3) on host memory, one pass as run_lane without pipelining: cfbpe_encode_batch, or with a non-NULL
// out_starts (room for out_cap entries) cfbpe_encode_batch_starts
__attribute__((visibility("default"))) int sim_encode_batch(void* const* vocabs, uint32_t n_vocabs, uint32_t n_prompts,
                                                            const uint8_t* bytes, const uint64_t* offsets, const uint8_t* vocab_ids,
                                                            uint32_t* out_ids, uint32_t* out_starts, uint64_t out_cap, uint64_t* out_offsets,
                                                            uint32_t* out_counts, uint64_t* n_long_out) {
    SimBatch c(vocabs, n_vocabs, n_prompts, bytes, offsets, vocab_ids);
    SimWorkspace ws(c.b.total_bytes);
    int* prof = nullptr;
    enqueue_encode(c.b, c.vs, uc_tables(), ws.w, out_ids, out_cap, out_offsets, out_counts, 4u, 0, 0, 0, 0, 0, 0, prof, nullptr, out_starts);
    if (n_long_out) *n_long_out = static_cast<uint64_t>(ws.st.n_long) + ws.st.n_big;
    if (const int rc = status_error(ws.st).code) return rc;
    if (out_ids && ws.st.n_tokens > out_cap) { out_offsets[n_prompts] = ws.st.n_tokens; return CFBPE_ENOSPC; }
    return 0;
}

// Where a pipelined host call puts sub-batch k (len bytes from byte o0, prompts from p0) in a lane of max_bytes / max_prompts
// that holds max_chunks sub-batches; per workspace buffer in for_each_ws_buffer's order: its kind, element size, the slice's
// first element and the lane's allocation
struct SimLayout {
    uint64_t n_buffers;
    uint64_t kind[32], elem[32], start[32], alloc[32];
    uint64_t extent[kWsKinds];             // workspace_extent(len)
    uint64_t long_cap, fix_cap, extras_cap, miss_cap[3];   // the slice's caps
    uint64_t bytes_at, bytes_alloc, offsets_at, offsets_alloc;
};
__attribute__((visibility("default"))) void sim_workspace_layout(uint64_t o0, uint64_t len, uint32_t k, uint32_t p0, uint64_t max_bytes,
                                                                 uint64_t max_prompts, uint32_t max_chunks, SimLayout* out) {
    Workspace base{};
    for_each_ws_buffer(base, [](auto*& p, WsKind) { p = reinterpret_cast<std::remove_reference_t<decltype(*p)>*>(uintptr_t(1) << 40); });
    Workspace sl = slice_workspace(base, o0, len, k);
    const WsSizes ext = workspace_extent(len), all = workspace_alloc(max_bytes, max_chunks);
    uintptr_t b0[32], s0[32];
    uint64_t n = 0;
    for_each_ws_buffer(base, [&](auto*& p, WsKind kind) { b0[n] = reinterpret_cast<uintptr_t>(p); out->kind[n] = kind; out->elem[n] = sizeof(*p); out->alloc[n] = all.n[kind]; ++n; });
    n = 0;
    for_each_ws_buffer(sl, [&](auto*& p, WsKind) { s0[n++] = reinterpret_cast<uintptr_t>(p); });
    out->n_buffers = n;
    for (uint64_t i = 0; i < n; ++i) out->start[i] = (s0[i] - b0[i]) / out->elem[i];
    for (uint32_t i = 0; i < kWsKinds; ++i) out->extent[i] = ext.n[i];
    out->long_cap = sl.long_cap; out->fix_cap = sl.fix_cap; out->extras_cap = sl.dense.extras_cap;
    for (uint32_t c = 0; c < 3; ++c) out->miss_cap[c] = sl.miss.cap[c];
    out->bytes_at = sub_batch_bytes_at(o0, k); out->bytes_alloc = lane_bytes_alloc(max_bytes, max_chunks);
    out->offsets_at = sub_batch_offsets_at(p0, k); out->offsets_alloc = lane_offsets_alloc(max_prompts, max_chunks);
}

// the sub-batch plan of a pipelined host call (host code of the product, csrc/subbatch.h)
__attribute__((visibility("default"))) int sim_plan_sub_batches(const uint64_t* offsets, uint32_t n, uint64_t chunk, int max_chunks, uint32_t* cut) {
    return plan_sub_batches(offsets, n, offsets[n], chunk, max_chunks, cut);
}

// the decode path (ids -> bytes) on host memory, with the vocabularies' special tables when specials is not NULL (a NULL
// entry: no table); returns the number of decoded bytes in out_offsets[n_seqs]
__attribute__((visibility("default"))) int sim_decode_batch(void* const* vocabs, void* const* specials, uint32_t n_vocabs, uint32_t n_seqs,
                                                            const uint32_t* ids, const uint64_t* id_offsets, const uint8_t* vocab_ids,
                                                            uint8_t* out, uint64_t out_cap, uint64_t* out_offsets) {
    const SimBatch c(vocabs, n_vocabs, 0, nullptr, nullptr, nullptr);
    SpecialSet sp{};
    for (uint32_t i = 0; specials && i < n_vocabs && i < kMaxVocabs; ++i)
        if (const SimSpecials* t = static_cast<const SimSpecials*>(specials[i])) sp.v[i] = make_special_view(t->words.data(), t->words);
    const uint64_t n_ids = id_offsets[n_seqs];
    DecodeView d{ids, id_offsets, vocab_ids, n_seqs, n_ids};
    const uint32_t n_tiles = static_cast<uint32_t>((n_ids + kDecodeTile - 1) / kDecodeTile);
    std::vector<uint32_t> lens(n_ids + 1), sums(n_tiles + 1);
    std::vector<uint64_t> base(n_tiles + 1);
    DeviceStatus st{};
    if (n_tiles) cusim::launch(n_tiles, 256, [&] { decode_len_kernel(d, c.vs, lens.data(), sums.data(), &st, sp); });
    cusim::launch(1u, n_tiles ? 1024u : 32u, [&] { tile_scan_kernel(sums.data(), n_tiles, base.data(), &st, nullptr); });
    if (st.bad_utf8) return CFBPE_EINVAL;
    if (n_tiles) cusim::launch(n_tiles, 256, [&] { decode_copy_kernel(d, c.vs, lens.data(), base.data(), out, out_cap, sp); });
    cusim::launch(static_cast<unsigned>((static_cast<uint64_t>(n_seqs) + 1 + 255) / 256), 256, [&] { decode_offsets_kernel(d, lens.data(), base.data(), out_offsets, &st); });
    return st.tok_end > out_cap ? CFBPE_ENOSPC : 0;
}

// the table cfbpe_vocab_set_specials builds (rc 0 or CFBPE_EINVAL with a message); n == 0 gives an empty table
__attribute__((visibility("default"))) void* sim_specials_build(uint32_t n, const uint8_t* bytes, const uint64_t* offsets, const uint32_t* ids,
                                                                int* rc, char* err, size_t errcap) {
    SimSpecials* t = new SimSpecials();
    std::string e;
    *rc = build_special_table(n, bytes, offsets, ids, t->words, e);
    if (*rc) { if (err && errcap) std::snprintf(err, errcap, "%s", e.c_str()); delete t; return nullptr; }
    return t;
}
__attribute__((visibility("default"))) void sim_specials_free(void* t) { delete static_cast<SimSpecials*>(t); }

// the special set of a call (fill_special_set, as the library's special_set) over the host tables
static int sim_special_set(void* const* specials, uint32_t n_vocabs, const uint8_t* const* modes, SpecialSet* sp, bool* scan) {
    const uint32_t* words[kMaxVocabs] = {};
    SpecialView views[kMaxVocabs] = {};
    for (uint32_t v = 0; v < n_vocabs && v < kMaxVocabs; ++v) {
        const SimSpecials* t = static_cast<const SimSpecials*>(specials[v]);
        if (!t || t->words.empty()) continue;
        words[v] = t->words.data();
        views[v] = make_special_view(t->words.data(), t->words);
    }
    uint32_t bad[2];
    return fill_special_set(words, views, modes, sp, scan, bad);
}

// cfbpe_encode_batch_special on host memory: the special set (fill_special_set) and the reading of the scan
// (special_scan_result) are the library's host code; between them the scan, then the ordinary path on the prompts as they are
// (no kept match) or on the stretches followed by the splice, as enqueue_special_call in csrc/cfbpe.cu runs them.  out_bad[2];
// *n_stretches_out: the stretches of the ordinary pass (n_prompts when the call took the fast path)
__attribute__((visibility("default"))) int sim_encode_batch_special(void* const* vocabs, void* const* specials, uint32_t n_vocabs,
                                                                    const uint8_t* const* modes, uint32_t n_prompts, const uint8_t* bytes,
                                                                    const uint64_t* offsets, const uint8_t* vocab_ids, uint32_t* out_ids,
                                                                    uint64_t out_cap, uint64_t* out_offsets, uint32_t* out_counts,
                                                                    uint32_t max_prompts, uint32_t* out_bad, uint64_t* n_stretches_out) {
    SimBatch c(vocabs, n_vocabs, n_prompts, bytes, offsets, vocab_ids);
    const uint64_t total = c.b.total_bytes, mp = max_prompts;
    SimWorkspace ws(total);
    std::vector<uint32_t> kept_n(mp + 1), st_id(mp + 1), ord_ids(total + 1), ord_counts(mp + 1);
    std::vector<uint64_t> kept_base(mp + 1), st_off(mp + 2), st_base(mp + 1), ord_offsets(mp + 2);
    std::vector<uint8_t> st_vocab(mp + 1);
    SpecialStatus ss{};
    const SpecialWork sw{kept_n.data(), kept_base.data(), st_off.data(), st_vocab.data(), st_id.data(), st_base.data(), &ss};
    SpecialSet sp;
    bool scan = false;
    if (const int rc = sim_special_set(specials, n_vocabs, modes, &sp, &scan)) return rc;
    uint64_t n_str = n_prompts;
    if (scan) {
        enqueue_special_scan(c.b, sp, ws.w, sw, 0);
        const SpecialScanResult r = special_scan_result(ss, n_prompts, max_prompts);
        if (r.disallowed) {
            if (out_bad) { out_bad[0] = r.prompt; out_bad[1] = r.index; }
            return CFBPE_EBADMSG;
        }
        if (!r.fits) return CFBPE_EINVAL;
        n_str = r.n_stretches;
    }
    if (n_stretches_out) *n_stretches_out = n_str;
    int* prof = nullptr;
    uint64_t n_tokens;
    if (n_str == n_prompts) {
        enqueue_encode(c.b, c.vs, uc_tables(), ws.w, out_ids, out_cap, out_offsets, out_counts, 4u, 0, 0, 0, 0, 0, 0, prof);
        n_tokens = ws.st.n_tokens;
    } else {
        enqueue_encode_special(c.b, sp, c.vs, uc_tables(), ws.w, sw, static_cast<uint32_t>(n_str), ord_ids.data(), total + 1, ord_offsets.data(),
                               ord_counts.data(), out_ids, out_cap, out_offsets, out_counts, 4u, 0, 0, 0, 0, 0, 0, prof);
        n_tokens = ss.fin.n_tokens;
    }
    if (const int rc = status_error(ws.st).code) return rc;
    if (out_ids && n_tokens > out_cap) { out_offsets[n_prompts] = n_tokens; return CFBPE_ENOSPC; }
    return 0;
}

// cfbpe_truncate_batch on host memory (one pass, as run_lane without pipelining): the ids go to a scratch buffer of one id a
// byte, as they go to the lane's buffer; out_counts may be NULL
__attribute__((visibility("default"))) int sim_truncate_batch(void* const* vocabs, uint32_t n_vocabs, uint32_t n_prompts,
                                                              const uint8_t* bytes, const uint64_t* offsets, const uint8_t* vocab_ids,
                                                              const uint32_t* budgets, uint32_t mode, uint32_t* out_cut, uint32_t* out_kept,
                                                              uint32_t* out_counts) {
    if (truncate_args_error(budgets, mode, out_cut, out_kept)) return CFBPE_EINVAL;
    SimBatch c(vocabs, n_vocabs, n_prompts, bytes, offsets, vocab_ids);
    const uint64_t total = c.b.total_bytes;
    SimWorkspace ws(total);
    std::vector<uint32_t> ids(total + 1, 0xDEADBEEF);
    std::vector<uint64_t> offs(static_cast<uint64_t>(n_prompts) + 1);
    std::vector<uint32_t> counts(static_cast<uint64_t>(n_prompts) + 1);
    const TruncateView tv{budgets, mode == CFBPE_TRUNCATE_TAIL ? 1u : 0u, out_cut, out_kept};
    int* prof = nullptr;
    enqueue_encode(c.b, c.vs, uc_tables(), ws.w, ids.data(), total + 1, offs.data(), counts.data(), 4u, 0, 0, 0, 0, 0, 0, prof, nullptr, nullptr, &tv);
    if (const int rc = status_error(ws.st).code) return rc;
    if (out_counts) std::copy(counts.begin(), counts.begin() + n_prompts, out_counts);
    return 0;
}

// cfbpe_chunk_batch on host memory (one pass, as run_lane without pipelining): the ids and starts go to scratch buffers of one
// entry a byte, as they go to the lane's buffers.  device_form = 0: the spans stage in the workspace's ids_by_pos / dense.by_piece
// and are copied out when they fit, as a host call does; 1: they go straight to out_spans (pairs, chunks at or past chunk_cap not
// written), as cfbpe_chunk_batch_device does.  out_counts may be NULL.
__attribute__((visibility("default"))) int sim_chunk_batch(void* const* vocabs, uint32_t n_vocabs, uint32_t n_prompts, const uint8_t* bytes,
                                                           const uint64_t* offsets, const uint8_t* vocab_ids, uint32_t chunk_tokens,
                                                           uint32_t overlap_tokens, uint32_t* out_spans, uint64_t chunk_cap,
                                                           uint64_t* out_chunk_offsets, uint32_t* out_counts, int device_form) {
    if (chunk_args_error(chunk_tokens, overlap_tokens, out_spans, out_chunk_offsets)) return CFBPE_EINVAL;
    SimBatch c(vocabs, n_vocabs, n_prompts, bytes, offsets, vocab_ids);
    const uint64_t total = c.b.total_bytes;
    SimWorkspace ws(total);
    std::vector<uint32_t> ids(total + 1, 0xDEADBEEF), starts(total + 1, 0xDEADBEEF);
    std::vector<uint64_t> offs(static_cast<uint64_t>(n_prompts) + 1);
    std::vector<uint32_t> counts(static_cast<uint64_t>(n_prompts) + 1);
    const uint32_t step = chunk_tokens - overlap_tokens;
    const ChunkView cv = device_form ? ChunkView{chunk_tokens, step, out_chunk_offsets, nullptr, out_spans, out_spans + 1, 2u, chunk_cap}
                                     : ChunkView{chunk_tokens, step, out_chunk_offsets, nullptr, ws.w.ids_by_pos, ws.w.dense.by_piece, 1u, UINT64_MAX};
    int* prof = nullptr;
    enqueue_encode(c.b, c.vs, uc_tables(), ws.w, ids.data(), total + 1, offs.data(), counts.data(), 4u, 0, 0, 0, 0, 0, 0, prof, nullptr, starts.data(),
                   nullptr, &cv);
    if (const int rc = status_error(ws.st).code) return rc;
    if (out_counts) std::copy(counts.begin(), counts.begin() + n_prompts, out_counts);
    if (ws.st.chunk_end != out_chunk_offsets[n_prompts] || ws.st.n_chunks != ws.st.chunk_end) return CFBPE_EIO;
    if (ws.st.chunk_end > chunk_cap) return CFBPE_ENOSPC;
    if (!device_form)
        for (uint64_t q = 0; q < ws.st.chunk_end; ++q) { out_spans[2 * q] = ws.w.ids_by_pos[q]; out_spans[2 * q + 1] = ws.w.dense.by_piece[q]; }
    return 0;
}

}  // extern "C"
