// pipeline.cuh -- the launch sequence of one encode pass (shared by libcfbpe.so and the
// non-GPU SIMT-emulator tests so that both run the same kernels in the same order).
//
// The including translation unit supplies three macros:
//   CFBPE_LAUNCH(kernel, grid, block, stream, ...)   launch
//   CFBPE_LAUNCH_SMEM(kernel, grid, block, smem, stream, ...)   launch with dynamic shared memory
//   CFBPE_ZERO(ptr, bytes, stream)                   asynchronous zero fill
//   CFBPE_MARK(prof, idx, stream, begin)             optional per-kernel event record
//   CFBPE_FORK(main, aux, ev) / CFBPE_JOIN(main, aux, ev)   make aux wait for main / main wait for aux
#pragma once
#include "../../include/cfbpe.h"
#include "bpe_kernels.cuh"

namespace cfbpe {

struct Workspace {
    uint32_t* piece_bits;   // 1 bit per byte: a piece starts here          [n_words + 2]
    uint32_t* tok_bits;     // 1 bit per byte: a token id lives here        [n_words + 2]
    uint32_t* ids_by_pos;   // token id at the byte position of its first byte [total]
    LongScratch lscratch;   // K2b per-byte state                            [total] each
    LongPiece* long_list;
    uint32_t long_cap;
    uint32_t* tile_counts;  // [n_tiles]
    uint64_t* tile_base;    // [n_tiles]
    DeviceStatus* status;
    MissLists miss;         // K2a -> K2m: short pieces that need the merge loop, by length class
    SplitFix* fix_list;     // K1 -> fixup: walkers that stopped in an undecided state (at most one per 16-byte block)   [total / 16 + 2]
    uint32_t fix_cap;
    DenseIds dense;         // ids of the short pieces, one word per piece; extras; piece counts / bases per 2 KiB tile
    uint32_t* pstart_bits;  // 1 bit per byte: a prompt starts here (and one at the end of the data)   [n_words + 2]
    uint32_t* block_prompt; // the prompt that holds the first byte of every 512-byte block           [total / 512 + 2]
};

// ---------------------------------------------------------------------------------------
// The workspace layout.  Every sized buffer of a Workspace follows one rule of the byte count: a pass over `len` bytes touches
// extent = len / unit (rounded up or down) + add elements of it.  A pipelined host call runs its sub-batches side by side in
// one lane's workspace: sub-batch k (first byte o0) starts at o0 / unit + per_k * k, which leaves room for the extent of every
// sub-batch before it, and the lane allocates the extent of max_bytes + per_k per sub-batch + spare.
// ---------------------------------------------------------------------------------------
enum WsKind : uint32_t {
    kWsFlagWords,     // piece_bits, tok_bits, pstart_bits: a bit per byte
    kWsPerByte,       // ids_by_pos, lscratch.*, dense.by_piece, dense.extras: at most one piece, token or part per byte
    kWsLongList,      // a long piece holds more than 32 bytes
    kWsScanTiles,     // tile_counts, tile_base: a K3 tile per 8 KiB
    kWsMiss0, kWsMiss1, kWsMiss2,   // miss lists: class c holds pieces of >= 13 | 7 | 2 bytes (no one-byte piece is ever a miss)
    kWsFixList,       // K1 walkers that stopped undecided: at most one per 16-byte block
    kWsPieceTiles,    // dense.tile_pieces, dense.piece_base: a piece tile per 2 KiB
    kWsBlockPrompt,   // a prompt per 512-byte block
    kWsKinds
};
struct WsRule { uint32_t unit; bool round_up; uint32_t add, per_k, spare; };
constexpr WsRule kWsRules[kWsKinds] = {
    {32, true, 2, 4, 2}, {1, false, 0, 0, 1}, {32, false, 1, 1, 0}, {kScanTileWords * 32, true, 1, 2, 0},
    {13, false, 2, 2, 62}, {7, false, 2, 2, 62}, {2, false, 2, 2, 62},
    {16, false, 2, 2, 0}, {kPieceTileBytes, false, 2, 2, 0}, {1u << kPromptBlockShift, false, 2, 2, 0},
};

// element counts, one per kind
struct WsSizes { uint64_t n[kWsKinds]; };

// what one pass over len bytes may touch: a one-shot call on its own buffers needs exactly this
inline WsSizes workspace_extent(uint64_t len) {
    WsSizes s;
    for (uint32_t i = 0; i < kWsKinds; ++i) {
        const WsRule& r = kWsRules[i];
        s.n[i] = (r.round_up ? (len + r.unit - 1) / r.unit : len / r.unit) + r.add;
    }
    return s;
}
// what a lane allocates: room for up to max_chunks sub-batches of a pipelined call over max_bytes
inline WsSizes workspace_alloc(uint64_t max_bytes, uint32_t max_chunks) {
    WsSizes s = workspace_extent(max_bytes);
    for (uint32_t i = 0; i < kWsKinds; ++i) s.n[i] += static_cast<uint64_t>(kWsRules[i].per_k) * max_chunks + kWsRules[i].spare;
    return s;
}

// the 64-bit entries of miss list c in a workspace with room for max_chunks sub-batches of max_bytes (a hand-built workspace,
// such as the emulator harnesses', sizes its miss lists with it)
inline uint64_t miss_list_words(uint64_t max_bytes, uint32_t c, uint32_t max_chunks) {
    return workspace_alloc(max_bytes, max_chunks).n[kWsMiss0 + c];
}

// every sized buffer of w with its kind: f(pointer&, kind).  One list for allocation, release, slicing and the emulator.
template <typename F>
inline void for_each_ws_buffer(Workspace& w, F&& f) {
    f(w.piece_bits, kWsFlagWords); f(w.tok_bits, kWsFlagWords); f(w.pstart_bits, kWsFlagWords);
    f(w.ids_by_pos, kWsPerByte); f(w.lscratch.rank, kWsPerByte); f(w.lscratch.aux0, kWsPerByte); f(w.lscratch.aux1, kWsPerByte);
    f(w.dense.by_piece, kWsPerByte); f(w.dense.extras, kWsPerByte);
    f(w.long_list, kWsLongList);
    f(w.tile_counts, kWsScanTiles); f(w.tile_base, kWsScanTiles);
    f(w.miss.list[0], kWsMiss0); f(w.miss.list[1], kWsMiss1); f(w.miss.list[2], kWsMiss2);
    f(w.fix_list, kWsFixList);
    f(w.dense.tile_pieces, kWsPieceTiles); f(w.dense.piece_base, kWsPieceTiles);
    f(w.block_prompt, kWsBlockPrompt);
}

// the capacities the kernels check, for buffers of the given sizes
inline void set_workspace_caps(Workspace& w, const WsSizes& s) {
    w.long_cap = static_cast<uint32_t>(s.n[kWsLongList]);
    w.fix_cap = static_cast<uint32_t>(s.n[kWsFixList]);
    w.dense.extras_cap = static_cast<uint32_t>(s.n[kWsPerByte]);
    for (uint32_t c = 0; c < 3; ++c) w.miss.cap[c] = static_cast<uint32_t>(s.n[kWsMiss0 + c]);
}

// sub-batch k's view of a lane's workspace `all`: the sub-batch holds len bytes from byte o0 of the call (status: set by the caller)
inline Workspace slice_workspace(const Workspace& all, uint64_t o0, uint64_t len, uint32_t k) {
    Workspace w = all;
    for_each_ws_buffer(w, [&](auto*& p, WsKind kind) { p += o0 / kWsRules[kind].unit + static_cast<uint64_t>(kWsRules[kind].per_k) * k; });
    set_workspace_caps(w, workspace_extent(len));
    return w;
}

// The lane's inputs and outputs of a pipelined host call.  Sub-batch k's bytes start on a 16-byte boundary (K1 reads 16 bytes a
// lane with one load); its n_k + 1 offsets start at p0 + k.  Between the end of sub-batch k and the start of k + 1 lie 1 to 31
// bytes (1 when o0 = 1 and o0 + len = 0 mod 16), so k's kernels read up to 32 bytes past its end into k + 1's bytes -- stale
// data from an earlier call, or an upload in flight -- which no result depends on; the allocation leaves more than 32 bytes after
// the last sub-batch.
inline uint64_t sub_batch_bytes_at(uint64_t o0, uint32_t k) { return ((o0 + 15) & ~15ull) + 16ull * k; }
inline uint64_t lane_bytes_alloc(uint64_t max_bytes, uint32_t max_chunks) { return max_bytes + 256 + 16ull * (max_chunks + 1); }
inline uint64_t sub_batch_offsets_at(uint32_t p0, uint32_t k) { return static_cast<uint64_t>(p0) + k; }
inline uint64_t lane_offsets_alloc(uint64_t max_prompts, uint32_t max_chunks) { return max_prompts + 1 + max_chunks; }

// the error a pass's status reports (overflow before vocabulary before UTF-8), or code CFBPE_OK
struct StatusError { int code; const char* msg; };
inline StatusError status_error(const DeviceStatus& st) {
    if (st.long_overflow || st.miss_overflow) return {CFBPE_EIO, "internal: long-piece list overflow"};
    if (st.bad_vocab) return {CFBPE_ENOENT, "a prompt names a vocabulary that is not loaded"};
    if (st.bad_utf8) return {CFBPE_EILSEQ, "a prompt holds malformed UTF-8"};
    return {CFBPE_OK, nullptr};
}

// the checks of a truncate call's own arguments (cfbpe_truncate_batch and its device form): the error, or nullptr
inline const char* truncate_args_error(const uint32_t* budgets, uint32_t mode, const uint32_t* cut, const uint32_t* kept) {
    if (mode != CFBPE_TRUNCATE_HEAD && mode != CFBPE_TRUNCATE_TAIL) return "mode is not a CFBPE_TRUNCATE_* value";
    if (!budgets || !cut || !kept) return "budgets, out_cut and out_kept are required";
    return nullptr;
}

// the checks of a chunk call's own arguments (cfbpe_chunk_batch and its device form): the error, or nullptr
inline const char* chunk_args_error(uint32_t chunk_tokens, uint32_t overlap_tokens, const uint32_t* spans, const uint64_t* chunk_offsets) {
    if (chunk_tokens == 0) return "chunk_tokens must be at least 1";
    if (overlap_tokens >= chunk_tokens) return "overlap_tokens must be less than chunk_tokens";
    if (!spans || !chunk_offsets) return "out_spans and out_chunk_offsets are required";
    return nullptr;
}

// the checks of a unit-starts call's own arguments (cfbpe_encode_batch_char_starts and its device form): the error, or nullptr
inline const char* unit_args_error(uint32_t unit, const uint32_t* ids, const uint32_t* starts) {
    if (unit != CFBPE_UNIT_CODEPOINT && unit != CFBPE_UNIT_UTF16) return "unit is not a CFBPE_UNIT_* value";
    if (!ids || !starts) return "out_ids and out_starts are required";
    return nullptr;
}

// K2b CTAs per SM (long_grid = 4 x SM count).  8 x 128 threads x 64 registers is the whole register file of an SM: the
// short-piece kernels on the other stream then wait for K2b instead of running beside it.
#ifndef CFBPE_LONG_CTAS
#define CFBPE_LONG_CTAS 8
#endif
constexpr uint32_t kLongCtasPerSm = CFBPE_LONG_CTAS;
#ifndef CFBPE_LIST_CTAS
#define CFBPE_LIST_CTAS 3      // (H100, 3 vs 2: the kernel alone 0.63 vs 0.80 ms, the step unchanged)
#endif
constexpr uint32_t kListCtasPerSm = CFBPE_LIST_CTAS;   // K2c CTAs (64 KB of shared memory each) per SM

enum KernelIdx { K_SPLIT = 0, K_ENCODE = 1, K_LONG = 2, K_COUNT = 3, K_SCAN = 4, K_EMIT = 5, K_LIST = 6, K_LONGSCAN = 7, K_MERGE = 8 };

inline uint64_t n_flag_words(uint64_t total_bytes) { return (total_bytes + 31) >> 5; }
inline uint32_t n_scan_tiles(uint64_t total_bytes) {
    return static_cast<uint32_t>((n_flag_words(total_bytes) + kScanTileWords - 1) / kScanTileWords);
}

// The path in stages, so that a caller with more than one stream can overlap the latency-bound long-piece kernel with
// the throughput-bound short-piece kernel (and, in a pipelined host call, with the next sub-batch):
//   split   zero the flags, K1 split, find the long pieces (K2 in scan mode)
//   long    K2b (+ K2c): pieces longer than 32 bytes               } independent of each other:
//   short   K2: whole-piece lookups and in-lane merges (<= 32 B)   } may run on two streams
//   back    flag_count, tile_scan (chained on the previous sub-batch's token total), emit, prompt offsets
template <typename Stream, typename Prof>
inline void enqueue_split(const BatchView& b, const VocabSet& vs, const UcTables& uc, const Workspace& w, Stream stream, Prof* prof,
                          uint32_t sm_count) {
    const uint64_t nw = n_flag_words(b.total_bytes);
    CFBPE_ZERO(w.status, sizeof(DeviceStatus), stream);
    if (!b.total_bytes) return;
    CFBPE_ZERO(w.piece_bits, (nw + 2) * sizeof(uint32_t), stream);
    CFBPE_ZERO(w.tok_bits, (nw + 2) * sizeof(uint32_t), stream);
    CFBPE_MARK(prof, K_SPLIT, stream, true);
#ifdef CFBPE_SPLIT_LEGACY      // A/B build: the first form of K1, one thread per 64-byte chunk
    const uint64_t n_chunks = (b.total_bytes + kSplitChunk - 1) / kSplitChunk;
    CFBPE_LAUNCH(pretok_split_kernel, static_cast<unsigned>((n_chunks + 255) / 256), 256, stream, b, vs, uc, w.piece_bits, w.status, w.fix_list, w.fix_cap);
#else
    CFBPE_ZERO(w.pstart_bits, (nw + 2) * sizeof(uint32_t), stream);
    CFBPE_LAUNCH(prompt_map_kernel, static_cast<unsigned>((static_cast<uint64_t>(b.n_prompts) + 1 + 255) / 256), 256, stream, b, vs, w.pstart_bits, w.block_prompt, w.status);
    {   // K1: persistent CTAs (the product tables are loaded once per CTA); a warp takes tiles of kSplitWarpOwned 16-byte blocks
        const uint64_t n_blocks16 = (b.total_bytes + 15) / 16;
        const uint32_t n_tiles = static_cast<uint32_t>((n_blocks16 + kSplitWarpOwned - 1) / kSplitWarpOwned);
        const uint32_t n_tabs = b.vocab_ids ? kNumPatterns : 1u;
        const uint32_t cap = sm_count * CFBPE_SPLIT_CTAS;      // resident CTAs: SMs x CTAs per SM (launch bounds)
        const uint32_t n_ctas = (n_tiles + kSplitCta / 32 - 1) / (kSplitCta / 32);
        CFBPE_LAUNCH_SMEM(pretok_split16_kernel, n_ctas < cap ? n_ctas : cap, kSplitCta, n_tabs * kProdTableBytes, stream,
                          b, vs, uc, w.pstart_bits, w.block_prompt, w.piece_bits, w.status, w.fix_list, w.fix_cap, n_tabs, n_tiles);
    }
#endif
    CFBPE_LAUNCH(pretok_fixup_kernel, 2 * sm_count, 256, stream, b, vs, uc, w.piece_bits, w.status, w.fix_list, w.fix_cap);   // almost always empty
    CFBPE_MARK(prof, K_SPLIT, stream, false);
    const uint64_t n_warps = (b.total_bytes + kPieceRange - 1) / kPieceRange;
    CFBPE_MARK(prof, K_LONGSCAN, stream, true);
    CFBPE_LAUNCH(long_scan_kernel, static_cast<unsigned>((n_warps + kPieceWarps - 1) / kPieceWarps), kPieceWarps * 32, stream,
                 b, w.piece_bits, w.long_list, w.long_cap, w.status, w.dense.tile_pieces);
    CFBPE_MARK(prof, K_LONGSCAN, stream, false);
}

template <typename Stream, typename Prof>
inline void enqueue_short(const BatchView& b, const VocabSet& vs, const Workspace& w, uint32_t long_grid, Stream stream, Prof* prof) {
    if (!b.total_bytes) return;
    const uint64_t n_warps = (b.total_bytes + kPieceRange - 1) / kPieceRange;
    CFBPE_MARK(prof, K_ENCODE, stream, true);
    const uint32_t n_tiles2k = static_cast<uint32_t>((n_warps + kLookupWarps - 1) / kLookupWarps);
    CFBPE_LAUNCH(tile_scan_kernel, 1u, 1024, stream, w.dense.tile_pieces, n_tiles2k, w.dense.piece_base, static_cast<DeviceStatus*>(nullptr),
                 static_cast<const uint64_t*>(nullptr));      // piece ranks: exclusive scan of K2s's per-tile counts
    CFBPE_LAUNCH(bpe_lookup_kernel, n_tiles2k, kLookupWarps * 32, stream, b, vs, w.piece_bits, w.dense, w.miss, w.status);
    CFBPE_MARK(prof, K_ENCODE, stream, false);
    CFBPE_MARK(prof, K_MERGE, stream, true);
    CFBPE_LAUNCH(bpe_merge_kernel, long_grid + long_grid / 2, kPieceWarps * 32, stream,      // 6 CTAs of 32 KB per SM
                 b, vs, w.piece_bits, w.dense, w.tok_bits, w.miss, w.status);
    CFBPE_MARK(prof, K_MERGE, stream, false);
}

// K2b: the pieces of 33 .. kBigPiece bytes (and the rare giants the list kernel cannot hold), one warp each
template <typename Stream, typename Prof>
inline void enqueue_long(const BatchView& b, const VocabSet& vs, const Workspace& w, uint32_t long_grid, Stream stream, Prof* prof) {
    if (!b.total_bytes) return;
    CFBPE_MARK(prof, K_LONG, stream, true);
    CFBPE_LAUNCH(bpe_long_kernel, (long_grid / 4) * kLongCtasPerSm, kLongWarps * 32, stream, b, vs, w.long_list, w.status, w.long_cap, w.ids_by_pos, w.lscratch, w.tok_bits);
    CFBPE_MARK(prof, K_LONG, stream, false);
}
// K2c: the big pieces, one CTA each, from their bytes -- independent of K2b (its own stream where the caller has one): two 64 KB
// CTAs per SM (long_grid = 4 x SM count), so that the short-piece kernels on the other stream keep ~100 KB of shared memory per SM
template <typename Stream, typename Prof>
inline void enqueue_list(const BatchView& b, const VocabSet& vs, const Workspace& w, uint32_t long_grid, Stream stream, Prof* prof) {
    if (!b.total_bytes) return;
#ifndef CFBPE_NO_DEFER
    CFBPE_MARK(prof, K_LIST, stream, true);
    CFBPE_LAUNCH_SMEM(bpe_list_kernel, (long_grid / 4) * kListCtasPerSm, kListWarps * 32, kListSmemBytes, stream, b, vs, w.long_list, w.status, w.long_cap, w.ids_by_pos, w.lscratch, w.tok_bits);
    CFBPE_MARK(prof, K_LIST, stream, false);
#endif
}

// back = count | scan | emit.  Only the scan reads what the previous sub-batch of a pipelined call produced (token_base), so
// a caller that chains sub-batches waits between count and scan and can let the emits of consecutive sub-batches overlap.
template <typename Stream, typename Prof>
inline void enqueue_count(const BatchView& b, const Workspace& w, Stream stream, Prof* prof) {
    if (!b.total_bytes) return;
    CFBPE_MARK(prof, K_COUNT, stream, true);
    CFBPE_LAUNCH(flag_count_kernel, n_scan_tiles(b.total_bytes), 256, stream, w.tok_bits, w.piece_bits, n_flag_words(b.total_bytes), w.tile_counts);
    CFBPE_MARK(prof, K_COUNT, stream, false);
}
template <typename Stream, typename Prof>
inline void enqueue_scan(const BatchView& b, const Workspace& w, Stream stream, Prof* prof, const uint64_t* token_base) {
    if (b.total_bytes) {
        CFBPE_MARK(prof, K_SCAN, stream, true);
        CFBPE_LAUNCH(tile_scan_kernel, 1u, 1024, stream, w.tile_counts, n_scan_tiles(b.total_bytes), w.tile_base, w.status, token_base);
        CFBPE_MARK(prof, K_SCAN, stream, false);
    } else {
        CFBPE_LAUNCH(tile_scan_kernel, 1u, 32, stream, w.tile_counts, 0u, w.tile_base, w.status, token_base);   // tok_end = base
    }
}
// out_starts (nullable; only with out_ids, and then vs too): each token's byte offset within its prompt, at the token's rank.  The
// token flags inside a multi-token piece are not at the tokens' first bytes (the long-piece kernels flag compacted slots), so the
// starts come from the ids: the tokens tile the text, so a token's byte position is the sum of the byte lengths of the tokens
// before it.  Lengths and their per-tile sums, a scan of the tile sums, then the scan inside every tile minus the prompt's offset.
// The dense-id tile arrays are free once the ids are out (the tiles of 2048 tokens are no more than the 2 KiB piece tiles).
// trunc (nullable; only with out_ids, and then vs too): every prompt's cut to its token budget, from the ids where they are
// (truncate_kernel, and truncate_long_kernel for the prompts with more ids to sum than one warp takes).
// chunk (nullable; only with out_starts): every prompt's chunks of chunk->n tokens, from the starts (chunk_scan, then chunk_emit
// over a grid of at most kChunkEmitCtas CTAs; a (sub-)batch has no more chunks than bytes).
// unit (nullable; only with out_starts): the starts in code points or UTF-16 units instead of bytes, and every prompt's length in
// them (unit_len, unit_tile_scan, unit_emit: a scan of the tokens' units that restarts at every prompt, over the byte starts).
constexpr uint32_t kChunkEmitCtas = 1024;
template <typename Stream, typename Prof>
inline void enqueue_emit(const BatchView& b, const Workspace& w, uint32_t* out_ids, uint64_t out_cap, uint64_t* out_offsets,
                         uint32_t* out_counts, Stream stream, Prof* prof, uint32_t* out_starts = nullptr, const VocabSet* vs = nullptr,
                         const TruncateView* trunc = nullptr, const ChunkView* chunk = nullptr, const UnitView* unit = nullptr) {
    CFBPE_MARK(prof, K_EMIT, stream, true);
    if (b.total_bytes && out_ids) {
        CFBPE_LAUNCH(emit_compact_kernel, n_scan_tiles(b.total_bytes), 256, stream, w.tok_bits, w.piece_bits, n_flag_words(b.total_bytes), w.tile_base,
                     w.dense, w.ids_by_pos, out_ids, out_cap);
    }
    CFBPE_LAUNCH(prompt_offsets_kernel, static_cast<unsigned>((static_cast<uint64_t>(b.n_prompts) + 1 + 7) / 8), 256, stream,      // a warp per prompt boundary
                 b, w.tok_bits, w.tile_base, out_offsets, out_counts, w.status);
    CFBPE_MARK(prof, K_EMIT, stream, false);
    if (b.total_bytes && out_ids && out_starts) {
        const uint32_t n_tiles = static_cast<uint32_t>((b.total_bytes + kStartsTile - 1) / kStartsTile);   // (at most one token a byte)
        CFBPE_LAUNCH(starts_len_kernel, n_tiles, 256, stream, b, *vs, out_ids, out_offsets, out_cap, w.status, out_starts, w.dense.tile_pieces);
        CFBPE_LAUNCH(tile_scan_kernel, 1u, 1024, stream, w.dense.tile_pieces, n_tiles, w.dense.piece_base, static_cast<DeviceStatus*>(nullptr),
                     static_cast<const uint64_t*>(nullptr));
        CFBPE_LAUNCH(starts_emit_kernel, n_tiles, 256, stream, b, out_offsets, out_cap, w.status, w.dense.piece_base, out_starts);
    }
    if (out_ids && out_starts && unit) {
        if (unit->lens && b.n_prompts) CFBPE_ZERO(unit->lens, static_cast<uint64_t>(b.n_prompts) * sizeof(uint32_t), stream);   // (an empty prompt has no token)
        if (b.total_bytes) {
            const uint32_t n_tiles = static_cast<uint32_t>((b.total_bytes + kStartsTile - 1) / kStartsTile);
            CFBPE_LAUNCH(unit_len_kernel, n_tiles, 256, stream, b, *vs, static_cast<const uint32_t*>(out_ids), out_offsets, out_cap, w.status,
                         static_cast<const uint32_t*>(out_starts), unit->utf16, w.dense.tile_pieces);
            CFBPE_LAUNCH(unit_tile_scan_kernel, 1u, 1024, stream, static_cast<const uint32_t*>(w.dense.tile_pieces), n_tiles, w.dense.piece_base);
            CFBPE_LAUNCH(unit_emit_kernel, n_tiles, 256, stream, b, *vs, static_cast<const uint32_t*>(out_ids), out_offsets, out_cap, w.status,
                         static_cast<const uint64_t*>(w.dense.piece_base), *unit, out_starts);
        }
    }
    if (out_ids && trunc && b.n_prompts) {
        CFBPE_LAUNCH(truncate_kernel, static_cast<unsigned>((static_cast<uint64_t>(b.n_prompts) + 7) / 8), 256, stream,    // a warp per prompt
                     b, *vs, out_ids, out_offsets, *trunc);
        if (b.total_bytes > kTruncChunkBytes) {       // (else no prompt has more than kTruncPartIds ids to sum)
            const uint64_t n_chunks = (b.total_bytes + kTruncChunkBytes - 1) / kTruncChunkBytes;
            CFBPE_LAUNCH(truncate_long_kernel, static_cast<unsigned>((n_chunks + 7) / 8), 256, stream, b, *vs, out_ids, out_offsets, *trunc);
        }
    }
    if (out_ids && out_starts && chunk) {
        CFBPE_LAUNCH(chunk_scan_kernel, 1u, 1024, stream, b, out_offsets, *chunk, w.status);
        if (b.total_bytes) {
            const uint64_t ctas = (b.total_bytes + 255) / 256;
            CFBPE_LAUNCH(chunk_emit_kernel, static_cast<unsigned>(ctas < kChunkEmitCtas ? ctas : kChunkEmitCtas), 256, stream,
                         b, out_offsets, static_cast<const uint32_t*>(out_starts), *chunk, static_cast<const DeviceStatus*>(w.status));
        }
    }
}
template <typename Stream, typename Prof>
inline void enqueue_back(const BatchView& b, const Workspace& w, uint32_t* out_ids, uint64_t out_cap, uint64_t* out_offsets,
                         uint32_t* out_counts, Stream stream, Prof* prof, const uint64_t* token_base, uint32_t* out_starts = nullptr,
                         const VocabSet* vs = nullptr, const TruncateView* trunc = nullptr, const ChunkView* chunk = nullptr,
                         const UnitView* unit = nullptr) {
    enqueue_count(b, w, stream, prof);
    enqueue_scan(b, w, stream, prof, token_base);
    enqueue_emit(b, w, out_ids, out_cap, out_offsets, out_counts, stream, prof, out_starts, vs, trunc, chunk, unit);
}

// The ids of a (sub-)batch from its ranks (id_rebase_kernel), once every kernel that reads them as ranks has run.  bases: the id bases
// of the vocabularies, or nullptr when none the call can touch has a base above 0 (nothing is launched).  status, out_offsets and
// out_cap: those of the pass that emitted the ranks into ids.
template <typename Stream>
inline void enqueue_rebase(const BatchView& b, const IdBases* bases, uint32_t* ids, const uint64_t* out_offsets, uint64_t out_cap,
                           const DeviceStatus* status, Stream stream) {
    if (!bases || !ids || !b.total_bytes) return;
    const uint32_t n_tiles = static_cast<uint32_t>((b.total_bytes + kStartsTile - 1) / kStartsTile);   // (at most one id a byte)
    CFBPE_LAUNCH(id_rebase_kernel, n_tiles, 256, stream, b, *bases, ids, out_offsets, out_cap, status);
}

// The whole path.  `aux` / `aux2` are streams of their own for the two long-piece kernels (pass the main stream to run everything
// in order); CFBPE_FORK / CFBPE_JOIN order them.  out_ids may be nullptr (count only); out_starts (nullable, with out_ids): the
// tokens' byte offsets within their prompts; trunc (nullable, with out_ids): the prompts' cuts to their token budgets; chunk
// (nullable, with out_starts): the prompts' chunks; unit (nullable, with out_starts): the starts in code points or UTF-16 units.
// Everything is asynchronous.
template <typename Stream, typename Prof, typename Ev>
inline void enqueue_encode(const BatchView& b, const VocabSet& vs, const UcTables& uc, const Workspace& w,
                           uint32_t* out_ids, uint64_t out_cap, uint64_t* out_offsets, uint32_t* out_counts,
                           uint32_t long_grid, Stream stream, Stream aux, Stream aux2, Ev ev_fork, Ev ev_join, Ev ev_join2, Prof* prof,
                           const uint64_t* token_base = nullptr, uint32_t* out_starts = nullptr, const TruncateView* trunc = nullptr,
                           const ChunkView* chunk = nullptr, const UnitView* unit = nullptr) {
    enqueue_split(b, vs, uc, w, stream, prof, long_grid / 4);
    CFBPE_FORK(stream, aux2, ev_fork);
    enqueue_list(b, vs, w, long_grid, aux2, prof);
    CFBPE_FORK(stream, aux, ev_fork);
    enqueue_long(b, vs, w, long_grid, aux, prof);
    enqueue_short(b, vs, w, long_grid, stream, prof);
    CFBPE_JOIN(stream, aux, ev_join);
    CFBPE_JOIN(stream, aux2, ev_join2);
    enqueue_back(b, w, out_ids, out_cap, out_offsets, out_counts, stream, prof, token_base, out_starts, &vs, trunc, chunk, unit);
}

}  // namespace cfbpe
