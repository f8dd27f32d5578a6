// pretok_lanes.cuh -- K1, second form: the pre-tokenizer split with ONE LANE PER 16 BYTES.
//
// The first form (split_thread in bpe_kernels.cuh: a thread per 64-byte chunk, byte loads, a ~170-instruction loop body
// per character, half the lanes idle) was bound by instruction issue at a small fraction of the
// HBM roofline.  Here a warp reads 512 contiguous bytes with one 16-byte load per lane, every lane classifies its 16
// bytes in registers (class table in shared memory), and the automaton of pretok_fsm.h runs in LOCK-STEP over byte
// indices: iteration k of the unrolled loop handles byte k of every lane's window, so all byte extraction is static and
// the loop body is ~35 instructions with no divergence in the common (ASCII) case.
//
// How a lane knows its state without the lanes to its left: the context automaton of pretok_ctx.h.  A lane gets the exact
// context at the start of its block from its left neighbour (the context after any 16 bytes depends on those bytes only),
// walks its block, and at the first position the context table calls a sync point it adopts the state named there.  From
// there it runs the split automaton to the end of its block AND ON into the next block (whose class bytes it has from its
// right neighbour through shared memory) until it stands on the first sync point of that block -- the very position where
// the right neighbour started, found through the same table lookup on the same context.  Every byte is covered by exactly
// one walker.  A walker that crosses the whole next block without meeting a sync point is in a long run (one whitespace byte
// repeated, digits, CJK under a cased pattern): the per-character walker of the first form takes over from its state
// (bulk run handling, undecided states and the fix-up kernel stay as they were).
//
// A CTA of 256 threads owns 254 blocks; threads 0 and 255 classify the blocks on either side and do not walk (ghosts), so
// neighbours never cross a CTA.  Prompt starts come as a bit array (prompt_map_kernel, one thread per prompt), so no lane
// searches the offsets; multi-vocabulary batches find their prompt through one u32 per 512 bytes.
#pragma once
#include "pretok_ctx.h"

namespace cfbpe {

constexpr uint32_t kSplitCta = 256;                 // threads per CTA
constexpr uint32_t kPromptBlockShift = 9;           // block_prompt: one entry per 512 bytes
constexpr uint32_t kNoRow = 0xFFFFu;

__device__ __forceinline__ uint32_t bit_at(const uint32_t* __restrict__ bits, uint64_t pos) { return (bits[pos >> 5] >> (pos & 31)) & 1u; }

// the prompt that holds byte pos (< total): block_prompt names the one holding the first byte of pos's 512-byte block
__device__ __forceinline__ uint32_t prompt_at(const BatchView& b, const uint32_t* __restrict__ block_prompt, uint64_t pos) {
    uint32_t p = block_prompt[pos >> kPromptBlockShift];
    while (b.offsets[p + 1] <= pos) ++p;
    return p;
}

// One thread per prompt (and one for the end of the data): the prompt-start bit array K1 reads instead of searching the
// offsets, the prompt of every 512-byte block (multi-vocabulary batches), and the check of the vocabulary ids (a device-path
// caller's ids were never seen by the host).
__global__ void __launch_bounds__(256)
prompt_map_kernel(BatchView b, VocabSet vs, uint32_t* __restrict__ pstart_bits, uint32_t* __restrict__ block_prompt, DeviceStatus* status) {
    const uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i > b.n_prompts) return;
    if (i == b.n_prompts) { atomicOr(&pstart_bits[b.total_bytes >> 5], 1u << (b.total_bytes & 31)); return; }   // "a prompt starts" at the end of the data
    const uint64_t s = b.offsets[i], e = b.offsets[i + 1];
    if (b.vocab_ids) {
        const uint32_t v = b.vocab_ids[i];
        if (v >= kMaxVocabs || !((vs.loaded_mask >> v) & 1u)) atomicOr(&status->bad_vocab, 1u);
    }
    if (e <= s) return;
    atomicOr(&pstart_bits[s >> 5], 1u << (s & 31));
    for (uint64_t blk = (s + (1u << kPromptBlockShift) - 1) >> kPromptBlockShift; (blk << kPromptBlockShift) < e; ++blk)
        block_prompt[blk] = static_cast<uint32_t>(i);
}

// A block with bytes >= 0x80: decode every character that starts in it (class | (len - 1) << 4 replaces X_LEAD) and check
// the UTF-8: lead byte ranges, continuation bytes present and in range, no overlongs, no surrogates, nothing above U+10FFFF,
// no character cut by the end of its prompt, and every continuation byte inside a character (pretok.cuh::get_char, restated on
// the block's bytes in registers: a 20-byte window -- the block and the four bytes after it).
// P: prompt-start bits of [base, base + 32).
__device__ __noinline__ uint4 classify_non_ascii(const uint8_t* __restrict__ s, uint64_t base, uint64_t total, const uint32_t* __restrict__ pstart_bits,
                                                 const UcTables uc, uint4 raw, uint4 cwv, uint32_t P, DeviceStatus* status) {
    uint32_t bad = 0;
    uint32_t need = 0;     // continuation bytes the block should start with: a character that began in the block before
    if ((raw.x & 0xC0u) == 0x80u && !(P & 1u)) {
        for (uint32_t j = 1; j <= 3 && j <= base; ++j) {
            if (j > 1 && bit_at(pstart_bits, base - j + 1)) break;        // a prompt starts between that byte and my block
            const uint32_t c = s[base - j];
            if ((c & 0xC0u) == 0x80u) continue;
            if (c >= 0xC0u) { const uint32_t len = c < 0xE0u ? 2u : (c < 0xF0u ? 3u : 4u); if (len > j) need = len - j; }
            break;
        }
    }
    // one trip per LEAD byte (a CJK block has five), not per byte
    const uint64_t lo = raw.x | (static_cast<uint64_t>(raw.y) << 32), hi = raw.z | (static_cast<uint64_t>(raw.w) << 32);
    const uint64_t ext = load_u32_any(s + base + 16);                      // (the buffer is readable 32 bytes past its end)
    uint64_t clo = cwv.x | (static_cast<uint64_t>(cwv.y) << 32), chi = cwv.z | (static_cast<uint64_t>(cwv.w) << 32);
    const uint32_t n = total - base < 16 ? static_cast<uint32_t>(total - base) : 16u;
    const uint32_t valid = n >= 16 ? 0xFFFFu : ((1u << n) - 1u);
    auto byte_mask = [](uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3, uint32_t v) -> uint32_t {      // bit k: class byte k == v
        uint32_t m = 0;
        const uint32_t ws[4] = {w0, w1, w2, w3};
#pragma unroll
        for (uint32_t j = 0; j < 4; ++j) {
            const uint32_t nz = (((ws[j] ^ (v * 0x01010101u)) & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | (ws[j] ^ (v * 0x01010101u));    // bit 7 of a byte: byte != v
            m |= (((((~nz) & 0x80808080u) >> 7) * 0x01020408u) >> 24 & 15u) << (4u * j);
        }
        return m;
    };
    const uint32_t conts = byte_mask(cwv.x, cwv.y, cwv.z, cwv.w, X_CONT) & valid;
    uint32_t leads = byte_mask(cwv.x, cwv.y, cwv.z, cwv.w, X_LEAD) & valid;
    uint32_t expected = (1u << need) - 1u;         // continuation bytes that belong to a character
    while (leads) {
        const uint32_t k = static_cast<uint32_t>(__ffs(leads)) - 1u;
        leads &= leads - 1u;
        // bytes k .. k+3 of the 20-byte window
        const uint32_t w = k < 8 ? static_cast<uint32_t>(k ? ((lo >> (8u * k)) | (hi << (64u - 8u * k))) : lo)
                                 : static_cast<uint32_t>(k > 8 ? ((hi >> (8u * (k - 8u))) | (ext << (64u - 8u * (k - 8u)))) : hi);
        const uint32_t b0 = w & 0xFFu, b1 = (w >> 8) & 0xFFu, b2 = (w >> 16) & 0xFFu, b3 = w >> 24;
        uint32_t len, cp;
        bool ok;
        if (b0 >= 0xC2u && b0 <= 0xDFu) { len = 2; cp = ((b0 & 0x1Fu) << 6) | (b1 & 0x3Fu); ok = (b1 & 0xC0u) == 0x80u; }
        else if (b0 >= 0xE0u && b0 <= 0xEFu) {
            len = 3; cp = ((b0 & 0x0Fu) << 12) | ((b1 & 0x3Fu) << 6) | (b2 & 0x3Fu);
            ok = (b1 & 0xC0u) == 0x80u && (b2 & 0xC0u) == 0x80u && cp >= 0x800u && !(cp >= 0xD800u && cp <= 0xDFFFu);
        } else if (b0 >= 0xF0u && b0 <= 0xF4u) {
            len = 4; cp = ((b0 & 0x07u) << 18) | ((b1 & 0x3Fu) << 12) | ((b2 & 0x3Fu) << 6) | (b3 & 0x3Fu);
            ok = (b1 & 0xC0u) == 0x80u && (b2 & 0xC0u) == 0x80u && (b3 & 0xC0u) == 0x80u && cp >= 0x10000u && cp <= 0x10FFFFu;
        } else { len = 1; cp = 0; ok = false; }
        // the character must end inside its prompt: no prompt start (nor the end of the data) among its continuation bytes
        ok = ok && k + len <= n + (total - base > 16 ? 4u : 0u) && !((P >> (k + 1)) & ((1u << (len - 1u)) - 1u));
        uint32_t cb;
        if (!ok) { bad = 1; len = 1; cb = X_OTHER; }               // (consumed as one byte of class OTHER, like get_char)
        else cb = uc_class(uc, cp) | ((len - 1u) << 4);
        expected |= ((1u << (len - 1u)) - 1u) << (k + 1u);
        if (k < 8) clo = (clo & ~(0xFFull << (8u * k))) | (static_cast<uint64_t>(cb) << (8u * k));
        else chi = (chi & ~(0xFFull << (8u * (k - 8u)))) | (static_cast<uint64_t>(cb) << (8u * (k - 8u)));
    }
    if ((conts & ~expected) != 0u) bad = 1;          // a continuation byte that no character claims
    if (bad) atomicOr(&status->bad_utf8, 1u);
    return make_uint4(static_cast<uint32_t>(clo), static_cast<uint32_t>(clo >> 32), static_cast<uint32_t>(chi), static_cast<uint32_t>(chi >> 32));
}

// the pattern of the prompt that holds byte pos (multi-vocabulary batches, at prompt starts only)
// (pats: the pattern ids of the eight vocabulary slots, four bits each -- a VocabSet by reference would be copied to the stack)
__device__ __noinline__ uint32_t pattern_at(const uint64_t* __restrict__ offsets, const uint8_t* __restrict__ vocab_ids, uint32_t pats,
                                            const uint32_t* __restrict__ block_prompt, uint64_t pos) {
    uint32_t p = block_prompt[pos >> kPromptBlockShift];
    while (offsets[p + 1] <= pos) ++p;
    return (pats >> (4u * (vocab_ids[p] & 7u))) & 15u;
}

// What the out-of-line paths need, in shared memory: a call then carries a pointer and the walker's few registers instead of
// a dozen arguments (the marshalling code sat in the hot loop four times and pushed it out of the 6 KB L0 instruction cache:
// most stall samples were instruction fetches).
struct SplitEnv {
    const uint8_t* s; const uint32_t* pstart_bits; const uint32_t* block_prompt; const uint64_t* offsets; const uint8_t* vocab_ids;
    DeviceStatus* status; SplitFix* fix_list;
    uint64_t total; uint32_t fix_cap, pats, n_tabs;
    const uint16_t* fsm; const uint16_t* ctx; const ProdInfo* info; const uint8_t* skip; const uint8_t* start; const uint8_t* tabs;
    const uint8_t* cls; uint32_t* piece_bits;
};

// The rare actions of a step: an undecided state that has to be resolved (the fix-up kernel goes on from here: the walker
// stops), or a contraction that may start at this apostrophe.  st: row of the state BEFORE the step; lo: its table entry for
// class byte cb at window byte k.  Returns the entry to go on with: unchanged when there is no contraction; else its next state
// replaced by SKIPn (and A_B_NOW cleared when the contraction is the suffix of the word that just ended); 0 (= DONE, no flags)
// when the walker stops.
__device__ __noinline__ uint32_t split_rare(const SplitEnv* env, uint32_t lo, uint32_t st, uint32_t cb, uint32_t k, uint32_t pat, uint64_t base) {
    const ProdInfo pi = env->info[pat * kProdMax + (st >> PE_NEXT_SHIFT)];
    const uint32_t x = cb & 15u;
    const uint32_t q = pi.q == PQ_NOSYNC ? (env->ctx[(pat & 1u) * kCtx16Size + (pi.ctx << 4) + x] >> 8) : pi.q;   // (first sync point: the state the context names)
    const uint32_t a = q < S_COUNT ? env->fsm[pat * kFsm16Size + q * 16 + x] : 0u;
    if (a & A_RESOLVE) {
        const uint32_t n = atomicAdd(&env->status->fix_n, 1u);
        if (n < env->fix_cap) { SplitFix f; f.pos = static_cast<uint32_t>(base + k); f.ce = static_cast<uint32_t>(base + 16); env->fix_list[n] = f; }
        else atomicOr(&env->status->long_overflow, 1u);
        return 0u;
    }
    if (!(a & A_CONTR)) return lo;
    const uint64_t pos = base + k, total = env->total;
    uint64_t pe = pos + 3 < total ? pos + 3 : total;          // a contraction does not cross the end of its prompt
    if (pos + 2 < total && bit_at(env->pstart_bits, pos + 2)) pe = pos + 2;
    if (pos + 1 < total && bit_at(env->pstart_bits, pos + 1)) pe = pos + 1;
    const uint32_t skip = contraction_bytes(env->s, pos, pe);
    if (!skip) return lo;
    const uint32_t chars = (skip == 3 && env->s[pos + 1] < 0x80u) ? 2u : 1u;     // 'll 've 're: two characters follow the apostrophe; 's ... and U+017F: one
    if (a & A_CONTR_SUFFIX) lo &= ~PE_B_NOW;                  // the contraction belongs to the piece that just ended
    const uint32_t next_ctx = env->info[pat * kProdMax + ((lo & PE_NEXT_MASK) >> PE_NEXT_SHIFT)].ctx;
    return (lo & ~PE_NEXT_MASK) | (static_cast<uint32_t>(env->skip[(pat * 2 + chars - 1u) * kCtxMax + next_ctx]) << PE_NEXT_SHIFT);
}

// Four bytes of the window with a prompt start (or the end of the data) among them, one byte at a time, everything handled:
// the prompt before the start ends (its last state meets X_EOT), the walker stops there if that is the next block's affair, else
// goes on in the new prompt with the new prompt's pattern.  Out of line: one group in five hundred.
// Returns {state row, marks (window bits), remembered positions, pattern}.
__device__ __noinline__ uint4 split_prompt_group(const SplitEnv* env, uint32_t word, uint32_t Pw, uint32_t kb, uint32_t st, uint32_t pat,
                                                 uint32_t rem, uint64_t base, uint32_t sync_mask) {
    uint32_t marks = 0;
    for (uint32_t i = 0; i < 4; ++i, word >>= 8) {
        const uint32_t k = kb + i;
        if (((Pw >> i) & 1u) && st != 0u) {
            const ProdInfo pi = env->info[pat * kProdMax + (st >> PE_NEXT_SHIFT)];
            bool stop = k >= 16 || base + k >= env->total;                    // (the owner of that block starts there)
            if (pi.q < S_COUNT) {
                const uint32_t a = env->fsm[pat * kFsm16Size + pi.q * 16 + X_EOT];
                if (a & A_EMIT_ALC) marks |= 1u << (rem & 31u);
                if (a & A_EMIT_LAST) marks |= 1u << ((rem >> 8) & 31u);
                if (a & A_EMIT_LBE) marks |= 1u << ((rem >> 16) & 31u);
                if (a & A_RESOLVE) { split_rare(env, 0, st, X_EOT, k, pat, base); stop = true; }
            }
            if (env->vocab_ids && !stop) pat = pattern_at(env->offsets, env->vocab_ids, env->pats, env->block_prompt, base + k);
            st = stop ? 0u : (static_cast<uint32_t>(env->start[pat]) << PE_NEXT_SHIFT);
        }
        const uint32_t cb = word & 0xFFu;
        const uint8_t* tab = env->tabs + (env->n_tabs == 1 ? 0u : pat) * kProdTableBytes;
        const uint2 e = *reinterpret_cast<const uint2*>(tab + st + ((cb & 15u) << 3));
        uint32_t lo = e.x, hi = e.y;
        if (lo & PE_EMIT_ALC) marks |= 1u << (rem & 31u);
        if (lo & PE_EMIT_LAST) marks |= 1u << ((rem >> 8) & 31u);
        if (lo & PE_EMIT_LBE) marks |= 1u << ((rem >> 16) & 31u);
        if (lo & PE_RARE) { lo = split_rare(env, lo, st, cb, k, pat, base); if (lo == 0u) hi = 0u; }
        if (lo & sync_mask) { lo = 0u; hi = 0u; }
        marks |= (lo & PE_B_NOW) << k;
        const uint32_t kk = k * 0x010101u + ((cb >> 4) + 1u) * 0x010001u;
        rem = (rem & ~hi) | (kk & hi);
        st = lo & PE_NEXT_MASK;
    }
    return make_uint4(st, marks, rem, pat);
}

// A walker that crossed its whole 32-byte window (every second tile has one: sixteen spaces of indentation, a nine-digit number) and
// needs, on average, three or four characters more.  It goes on with the product automaton over the next blocks of 16 bytes, loaded
// here -- ASCII only, no prompt start inside: anything else is left to the per-character walker, whose set-up alone (prompt
// search, the classes of the last three characters from memory) dwarfs the few characters it walks.
// Marks at window positions >= 32 go to the flag words directly.  Returns {state row, marks at window positions < 32,
// remembered positions, blocks done}; state row != 0: the per-character walker goes on at base + 32 + 16 * blocks.
constexpr uint32_t kSplitExtBlocks = 8;      // window positions stay below 160 (the remembered positions are bytes)
__device__ __noinline__ uint4 split_extend(const SplitEnv* env, uint32_t st, uint32_t rem, uint32_t pat, uint64_t base) {
    const uint8_t* tab = env->tabs + (env->n_tabs == 1 ? 0u : pat) * kProdTableBytes;
    uint32_t marks_lo = 0, blocks = 0;
    while (st != 0u && blocks < kSplitExtBlocks) {
        const uint64_t p0 = base + 32u + 16u * blocks;
        if (p0 + 16u > env->total) break;
        uint32_t ww[4];
        load16(env->s + p0, ww[0], ww[1], ww[2], ww[3]);
        if ((ww[0] | ww[1] | ww[2] | ww[3]) & 0x80808080u) break;                                  // a character of several bytes
        if ((env->pstart_bits[p0 >> 5] >> (p0 & 31u)) & 0xFFFFu) break;                            // a prompt starts in these 16 bytes
        uint32_t out = 0;                                                                          // marks of this block (bit = byte in it) ...
        auto mark_at = [&](uint32_t k) {                                                           // ... and at remembered positions (anywhere before)
            if (k < 32u) marks_lo |= 1u << k;
            else if (k >= 32u + 16u * blocks) out |= 1u << (k - 32u - 16u * blocks);
            else atomicOr(&env->piece_bits[(base + k) >> 5], 1u << ((base + k) & 31u));
        };
#pragma unroll 1
        for (uint32_t i = 0; i < 16u && st != 0u; ++i) {
            const uint32_t k = 32u + 16u * blocks + i;
            const uint32_t cb = env->cls[(ww[i >> 2] >> (8u * (i & 3u))) & 0xFFu];
            const uint2 e = *reinterpret_cast<const uint2*>(tab + st + ((cb & 15u) << 3));
            uint32_t lo = e.x, hi = e.y;
            if (lo & (PE_EMIT_ANY | PE_RARE)) {
                if (lo & PE_EMIT_ALC) mark_at(rem & 0xFFu);
                if (lo & PE_EMIT_LAST) mark_at((rem >> 8) & 0xFFu);
                if (lo & PE_EMIT_LBE) mark_at((rem >> 16) & 0xFFu);
                if (lo & PE_RARE) { lo = split_rare(env, lo, st, cb, k, pat, base); if (lo == 0u) hi = 0u; }
            }
            if (lo & PE_SYNC) { lo = 0u; hi = 0u; }           // the owner of this block started exactly here
            if (lo & PE_B_NOW) out |= 1u << i;
            const uint32_t kk = k * 0x010101u + 0x010001u;     // (ASCII: every character is one byte)
            rem = (rem & ~hi) | (kk & hi);
            st = lo & PE_NEXT_MASK;
        }
        if (out) atomicOr(&env->piece_bits[p0 >> 5], out << (p0 & 31u));
        ++blocks;
    }
    return make_uint4(st, marks_lo, rem, blocks);
}

// the per-character walker of the first form, out of line (it is large, and rare: long runs without a sync point)
__device__ __noinline__ void split_resume(const BatchView b, uint32_t pats, const UcTables uc, const uint16_t* s_fsm, const uint8_t* s_cls,
                                         uint32_t* __restrict__ piece_bits, DeviceStatus* status, SplitFix* fix_list, uint32_t fix_cap,
                                         uint64_t pos, uint32_t pidx, uint32_t q, uint64_t alc, uint64_t last, uint64_t lbe) {
    const VocabSet* none = nullptr;      // (mode 2 never reads it: the patterns come packed)
    split_thread<2, 16, kFsm16Size>(b, *none, uc, s_fsm, s_cls, piece_bits, status, fix_list, fix_cap, 0, pos, pos, pidx, q, alc, last, lbe, pats);
}

// ---- TMA bulk copies (cp.async.bulk global -> shared, completion on an mbarrier): how K1 stages its tables.  One thread arms the
//      barrier with the byte count and issues the copies; everybody waits on the barrier's phase.  (The emulator copies in a loop.)
#ifndef CFBPE_SPLIT_TMA
#define CFBPE_SPLIT_TMA 1          // A/B: 0 = cooperative load loop (ld.global + st.shared by all threads)
#endif

constexpr uint32_t kSplitWarpOwned = 30;            // blocks of 16 bytes a WARP owns: lanes 1..30; lanes 0 and 31 classify the blocks on
                                                    // either side and do not walk (ghosts), so neighbours are one shuffle away and no
                                                    // warp ever waits for another (a CTA-wide exchange spent 39 % of the time in barriers)

// n_tabs: product tables in shared memory -- 1 (single-vocabulary batch: the table of pattern pat0) or kNumPatterns
#ifndef CFBPE_SPLIT_CTAS
#define CFBPE_SPLIT_CTAS 4
#endif
#ifndef CFBPE_SPLIT_TICKETS
#define CFBPE_SPLIT_TICKETS 1      // 1: warps draw tiles from a counter; 0: fixed stride (A/B: the ticket is faster)
#endif
#ifndef CFBPE_SPLIT_UNROLL
#define CFBPE_SPLIT_UNROLL 1       // copies of the step in the hot loop (1 | 2 | 4); 2 and 4 measured slower (instruction cache)
#endif
__global__ void __launch_bounds__(kSplitCta, CFBPE_SPLIT_CTAS)
pretok_split16_kernel(BatchView b, VocabSet vs, UcTables uc, const uint32_t* __restrict__ pstart_bits,
                      const uint32_t* __restrict__ block_prompt, uint32_t* __restrict__ piece_bits, DeviceStatus* status,
                      SplitFix* fix_list, uint32_t fix_cap, uint32_t n_tabs, uint32_t n_tiles) {
    CFBPE_DYN_SMEM(s_dyn);                                   // n_tabs product tables of kProdTableBytes
    __shared__ __align__(16) uint16_t s_fsm[kNumPatterns * kFsm16Size];    // for the end-of-prompt transition and the per-character walker
    __shared__ __align__(16) uint16_t s_ctx[2 * kCtx16Size];
    __shared__ __align__(16) uint8_t s_cls[256];
    __shared__ __align__(16) ProdInfo s_info[kNumPatterns * kProdMax];
    __shared__ __align__(16) uint8_t s_skip[kNumPatterns * 2 * kCtxMax];
    __shared__ __align__(16) uint8_t s_start[16];
    __shared__ __align__(8) uint64_t s_bar;
    __shared__ SplitEnv s_env;
    const uint32_t t = threadIdx.x, lane = t & 31u;
    const bool multi = b.vocab_ids != nullptr;
    const uint32_t pat0 = vs.v[0].pattern_id;
    {   // tables: once per CTA (its warps walk many tiles) -- staged by TMA: seven bulk copies, one mbarrier
        const uint64_t* src = uc.prod + (n_tabs == 1 ? static_cast<uint64_t>(pat0) * kProdMax * 16 : 0);
#if CFBPE_SPLIT_TMA && !defined(CUSIM_EMULATOR)
        if (t == 0) mbar_init(&s_bar, 1);
        __syncthreads();
        if (t == 0) {
            const uint32_t b_prod = n_tabs * kProdTableBytes, b_fsm = sizeof(uint16_t) * kNumPatterns * kFsm16Size, b_ctx = sizeof(uint16_t) * 2 * kCtx16Size,
                           b_info = sizeof(ProdInfo) * kNumPatterns * kProdMax, b_skip = kNumPatterns * 2 * kCtxMax;
            mbar_expect_tx(&s_bar, b_prod + b_fsm + b_ctx + b_info + b_skip + 16u + 256u);
            bulk_g2s(s_dyn, src, b_prod, &s_bar);
            bulk_g2s(s_fsm, uc.fsm16, b_fsm, &s_bar);
            bulk_g2s(s_ctx, uc.ctx16, b_ctx, &s_bar);
            bulk_g2s(s_info, uc.prod_info, b_info, &s_bar);
            bulk_g2s(s_skip, uc.prod_skip, b_skip, &s_bar);
            bulk_g2s(s_start, uc.prod_start, 16u, &s_bar);
            bulk_g2s(s_cls, uc.cls256, 256u, &s_bar);
        }
        mbar_wait(&s_bar, 0);
#else
        uint64_t* dst = reinterpret_cast<uint64_t*>(s_dyn);
        for (uint32_t i = t; i < n_tabs * kProdMax * 16; i += kSplitCta) dst[i] = src[i];
        for (uint32_t i = t; i < kNumPatterns * kFsm16Size; i += kSplitCta) s_fsm[i] = uc.fsm16[i];
        for (uint32_t i = t; i < 2 * kCtx16Size; i += kSplitCta) s_ctx[i] = uc.ctx16[i];
        for (uint32_t i = t; i < kNumPatterns * kProdMax; i += kSplitCta) s_info[i] = uc.prod_info[i];
        for (uint32_t i = t; i < kNumPatterns * 2 * kCtxMax; i += kSplitCta) s_skip[i] = uc.prod_skip[i];
        if (t < kNumPatterns) s_start[t] = uc.prod_start[t];
        s_cls[t] = uc.cls256[t];
        (void)s_bar;
#endif
    }
    uint32_t pats = 0;
#pragma unroll
    for (uint32_t i = 0; i < kMaxVocabs; ++i) pats |= (vs.v[i].pattern_id & 15u) << (4u * i);
    if (t == 0) {
        SplitEnv e;
        e.s = b.bytes; e.pstart_bits = pstart_bits; e.block_prompt = block_prompt; e.offsets = b.offsets; e.vocab_ids = b.vocab_ids;
        e.status = status; e.fix_list = fix_list; e.total = b.total_bytes; e.fix_cap = fix_cap; e.pats = pats; e.n_tabs = n_tabs;
        e.fsm = s_fsm; e.ctx = s_ctx; e.info = s_info; e.skip = s_skip; e.start = s_start; e.tabs = reinterpret_cast<const uint8_t*>(s_dyn);
        e.cls = s_cls; e.piece_bits = piece_bits;
        s_env = e;
    }
    __syncthreads();
    const uint8_t* __restrict__ s = b.bytes;
    const uint64_t total = b.total_bytes;
    const bool aligned = (reinterpret_cast<uintptr_t>(s) & 15u) == 0u;
    const uint8_t* const tabs = reinterpret_cast<const uint8_t*>(s_dyn);

    // tiles by ticket (CFBPE_SPLIT_TICKETS, A/B) or by stride: a tile that enters a long run (the per-character walker, one lane)
    // costs ten average tiles.  The next ticket is drawn while the current tile is worked on.
#if CFBPE_SPLIT_TICKETS
    uint32_t tile = 0;
    if (lane == 0) tile = atomicAdd(&status->split_next, 1u);
    tile = __shfl_sync(kFull, tile, 0);
#else
    const uint32_t warps_total = gridDim.x * (kSplitCta / 32u);
    uint32_t tile = blockIdx.x * (kSplitCta / 32u) + (t >> 5);
#endif
#pragma unroll 1
    while (tile < n_tiles) {
#if CFBPE_SPLIT_TICKETS
        uint32_t next_tile = 0;
        if (lane == 0) next_tile = atomicAdd(&status->split_next, 1u);
#else
        const uint32_t next_tile = tile + warps_total;
#endif
        CFBPE_DBG_COUNT(10);
#if defined(CFBPE_TILE_CLOCK) && !defined(CUSIM_EMULATOR)
        const long long tile_t0 = clock64();         // measurement build: which tiles take long (printf from the device)
        const uint32_t tile_dbg = tile;
#endif
        const int64_t blk = static_cast<int64_t>(tile) * kSplitWarpOwned + static_cast<int64_t>(lane) - 1;
        const uint64_t base = blk > 0 ? static_cast<uint64_t>(blk) * 16u : 0u;
        const bool have = blk >= 0 && base < total;
        const bool owner = have && lane >= 1 && lane <= kSplitWarpOwned;

        // ---- my 16 bytes -> 16 class bytes
        uint32_t cw[4] = {0, 0, 0, 0};
        uint32_t P = 0;                 // prompt-start bits of [base, base + 32)
        uint32_t pat = pat0;
        bool nonascii = false;
        if (have) {
            uint32_t ww[4];
            if (aligned) { const uint4 w = *reinterpret_cast<const uint4*>(s + base); ww[0] = w.x; ww[1] = w.y; ww[2] = w.z; ww[3] = w.w; }
            else load16(s + base, ww[0], ww[1], ww[2], ww[3]);       // a device-path caller's buffer that is not 16-byte aligned
#pragma unroll
            for (uint32_t j = 0; j < 4; ++j)
                cw[j] = s_cls[ww[j] & 0xFFu] | (static_cast<uint32_t>(s_cls[(ww[j] >> 8) & 0xFFu]) << 8) |
                        (static_cast<uint32_t>(s_cls[(ww[j] >> 16) & 0xFFu]) << 16) | (static_cast<uint32_t>(s_cls[ww[j] >> 24]) << 24);
            const uint64_t wi = base >> 5;
            P = (base & 16u) ? ((pstart_bits[wi] >> 16) | (pstart_bits[wi + 1] << 16)) : pstart_bits[wi];
            nonascii = ((ww[0] | ww[1] | ww[2] | ww[3]) & 0x80808080u) != 0u;
            if (nonascii) {
                const uint4 r = classify_non_ascii(s, base, total, pstart_bits, uc, make_uint4(ww[0], ww[1], ww[2], ww[3]),
                                                   make_uint4(cw[0], cw[1], cw[2], cw[3]), P, status);
                cw[0] = r.x; cw[1] = r.y; cw[2] = r.z; cw[3] = r.w;
            }
        }
        if (multi) {    // the pattern at my block's first byte: one query per warp, repeated only by lanes behind a prompt start
            const uint32_t starts_before = __ballot_sync(kFull, have && (P & 0xFFFFu)) & ((2u << lane) - 1u);
            uint32_t p0 = 0;
            if (lane == 0 && have) p0 = pattern_at(b.offsets, b.vocab_ids, pats, block_prompt, base);
            else if (lane == 0 && blk < 0 && total) p0 = pattern_at(b.offsets, b.vocab_ids, pats, block_prompt, 0);
            p0 = __shfl_sync(kFull, p0, 0);
            pat = (have && starts_before) ? pattern_at(b.offsets, b.vocab_ids, pats, block_prompt, base) : p0;
        }
        // ---- the exact context at the end of my block: the context automaton over its last three characters
        uint32_t endc = kCtxStart;
        if (have) {
            uint32_t cased = pat & 1u;
            // (a prompt of another casedness may have started before the bytes looked at)
            if (multi && (P & 0xFFFFu)) { const uint64_t q = base + (nonascii ? 4u : 13u); if (q < total) cased = pattern_at(b.offsets, b.vocab_ids, pats, block_prompt, q) & 1u; }
            auto ctx_step = [&](uint32_t k) {
                if ((P >> k) & 1u) {
                    endc = kCtxStart;
                    if (multi && base + k < total) cased = pattern_at(b.offsets, b.vocab_ids, pats, block_prompt, base + k) & 1u;
                }
                const uint32_t x = (cw[k >> 2] >> (8u * (k & 3u))) & 15u;
                endc = s_ctx[cased * kCtx16Size + (endc << 4) + x] & 0xFFu;
            };
            if (!nonascii) { ctx_step(13); ctx_step(14); ctx_step(15); }       // three ASCII bytes are three characters
            else if (!(P & 0xFFFFu)) {                                         // the last three characters that START in my block
                uint32_t starts = 0;                                            // bit k: byte k is not a continuation byte
#pragma unroll
                for (uint32_t j = 0; j < 4; ++j) {
                    const uint32_t nz = (((cw[j] ^ 0x0C0C0C0Cu) & 0x0F0F0F0Fu) + 0x0F0F0F0Fu) & 0x10101010u;     // low nibble != X_CONT
                    starts |= ((((nz >> 4) * 0x01020408u) >> 24) & 15u) << (4u * j);
                }
                const uint32_t c1 = 31u - static_cast<uint32_t>(__clz(starts)); starts &= ~(1u << c1);
                const uint32_t c2 = 31u - static_cast<uint32_t>(__clz(starts)); starts &= ~(1u << c2);
                const uint32_t c3 = starts ? 31u - static_cast<uint32_t>(__clz(starts)) : c2;
                auto cls_at = [&](uint32_t k) { const uint32_t w = k < 8 ? (k < 4 ? cw[0] : cw[1]) : (k < 12 ? cw[2] : cw[3]); return (w >> (8u * (k & 3u))) & 15u; };
                endc = s_ctx[cased * kCtx16Size + (endc << 4) + cls_at(c3)] & 0xFFu;
                endc = s_ctx[cased * kCtx16Size + (endc << 4) + cls_at(c2)] & 0xFFu;
                endc = s_ctx[cased * kCtx16Size + (endc << 4) + cls_at(c1)] & 0xFFu;
            } else {                                                            // a prompt starts inside: twelve bytes hold at least three characters
#pragma unroll 1
                for (uint32_t k = 4; k < 16; ++k) ctx_step(k);
            }
        }
#if defined(CFBPE_TILE_CLOCK) && !defined(CUSIM_EMULATOR)
        __syncwarp(); const long long tile_t1 = clock64();
#endif
        // ---- neighbours: the class bytes of the block to my right, the context at the end of the block to my left
        const uint32_t left_ctx = __shfl_up_sync(kFull, endc, 1);
        uint32_t w0 = cw[0], w1 = cw[1], w2 = cw[2], w3 = cw[3];
        uint32_t w4 = __shfl_down_sync(kFull, w0, 1), w5 = __shfl_down_sync(kFull, w1, 1), w6 = __shfl_down_sync(kFull, w2, 1), w7 = __shfl_down_sync(kFull, w3, 1);

        // ---- walk: from my first sync point to the first sync point of the next block.  One lookup in the product table per
        //      byte; the eight class words of the window in a shift register; ONE copy of the step in the instruction stream
        //      (unrolled it overflowed the instruction cache: the warps of an SM are all at different places of the kernel)
        uint32_t mine = 0;              // bit k: a piece starts at base + k (every mark of the 32 steps lies inside the window: a remembered
                                        // position is emitted at a later character than the one that set it)
        uint32_t rem = 0;               // remembered positions, relative to base: alc | last << 8 | lbe << 16
        uint32_t st = owner ? ((1u + left_ctx) << PE_NEXT_SHIFT) : 0u;     // row of my state in the product table; 0 = DONE; NOSYNC(context to my left)
        const uint8_t* tab = tabs + (n_tabs == 1 ? 0u : pat) * kProdTableBytes;
        // one byte: ONE lookup in the product table.  kb = first byte index of the group of four, i = index in the group.  The
        // hot loop is these ~20 instructions four times over, plus the three conditional marks; everything else is a call.
        auto step = [&](const uint32_t i, const uint32_t cb, const uint32_t kb, const uint32_t kb3, const uint32_t sync_mask, uint32_t& gm) {
            const uint2 e = *reinterpret_cast<const uint2*>(tab + st + ((cb & 15u) << 3));
            uint32_t lo = e.x, hi = e.y;
            if (lo & (PE_EMIT_ANY | PE_RARE)) {      // boundaries at remembered positions (indentation, cased words); contractions
                if (lo & PE_EMIT_ALC) mine |= 1u << (rem & 31u);
                if (lo & PE_EMIT_LAST) mine |= 1u << ((rem >> 8) & 31u);
                if (lo & PE_EMIT_LBE) mine |= 1u << ((rem >> 16) & 31u);
                if (lo & PE_RARE) { lo = split_rare(&s_env, lo, st, cb, kb + i, pat, base); if (lo == 0u) hi = 0u; }
            }
            if (lo & sync_mask) { lo = 0u; hi = 0u; }               // hand-over: the next block's owner started exactly here
            gm |= (lo & PE_B_NOW) << i;
            const uint32_t kk = kb3 + i * 0x010101u + ((cb >> 4) + 1u) * 0x010001u;    // alc, lbe: the position after this character; last: this one
            rem = (rem & ~hi) | (kk & hi);
            st = lo & PE_NEXT_MASK;
        };
#pragma unroll 1
        for (uint32_t j = 0; j < 8; ++j) {
            if (j == 4 && s_info[pat * kProdMax + (st >> PE_NEXT_SHIFT)].q == PQ_NOSYNC) st = 0;   // no sync point in my own block: the walker from the left covers it
            if (j >= 4 && __all_sync(kFull, st == 0u)) break;
            const uint32_t word = w0;
            w0 = w1; w1 = w2; w2 = w3; w3 = w4; w4 = w5; w5 = w6; w6 = w7;
            const uint32_t kb = 4u * j, kb3 = kb * 0x010101u;
            const uint32_t Pw = (P >> kb) & 15u;
            const uint32_t sync_mask = j >= 4 ? static_cast<uint32_t>(PE_SYNC) : 0u;
            if (Pw && st != 0u) {       // a prompt starts inside these four bytes (or the data ends): rare
                const uint4 r = split_prompt_group(&s_env, word, Pw, kb, st, pat, rem, base, sync_mask);
                st = r.x; mine |= r.y; rem = r.z; pat = r.w;
                tab = tabs + (n_tabs == 1 ? 0u : pat) * kProdTableBytes;
            } else {
                uint32_t gm = 0;            // the group's A_B_NOW marks
#if CFBPE_SPLIT_UNROLL == 4
#pragma unroll
                for (uint32_t i = 0; i < 4; ++i) step(i, (word >> (8u * i)) & 0xFFu, kb, kb3, sync_mask, gm);
#elif CFBPE_SPLIT_UNROLL == 2
#pragma unroll 1
                for (uint32_t i = 0; i < 4; i += 2) { step(i, (word >> (8u * i)) & 0xFFu, kb, kb3, sync_mask, gm); step(i + 1, (word >> (8u * i + 8u)) & 0xFFu, kb, kb3, sync_mask, gm); }
#else
#pragma unroll 1
                for (uint32_t i = 0; i < 4; ++i) step(i, (word >> (8u * i)) & 0xFFu, kb, kb3, sync_mask, gm);
#endif
                mine |= gm << kb;
            }
        }
#if defined(CFBPE_TILE_CLOCK) && !defined(CUSIM_EMULATOR)
        __syncwarp(); const long long tile_t2 = clock64(); const uint32_t n_resume = __popc(__ballot_sync(kFull, st != 0u));
#endif
        // ---- a walker that crossed the whole next block: the per-character walker goes on from its state
        uint32_t ext_blocks = 0;
        if (st != 0u) {         // a few characters more, mostly: go on with the product automaton (split_extend)
            const uint4 r = split_extend(&s_env, st, rem, pat, base);
            st = r.x; mine |= r.y; rem = r.z; ext_blocks = r.w;
        }
        if (st != 0u) {
            const ProdInfo pi = s_info[pat * kProdMax + (st >> PE_NEXT_SHIFT)];
            uint64_t pos = base + 32u + 16u * ext_blocks;
            while (pos < total && (s[pos] & 0xC0u) == 0x80u) ++pos;          // byte 32 may lie inside the character that began at byte 29..31
            uint32_t q = pi.q;
            if (q == PQ_SKIP1 || q == PQ_SKIP2) {                            // inside a contraction: step over what is left of it
                for (uint32_t n = (q == PQ_SKIP2 ? 2u : 1u); n && pos < total; --n) { ++pos; while (pos < total && (s[pos] & 0xC0u) == 0x80u) ++pos; }
                q = S_START;
            }
            split_resume(b, pats, uc, s_fsm, s_cls, piece_bits, status, fix_list, fix_cap, pos, prompt_at(b, block_prompt, pos - 1),
                         q, base + (rem & 0xFFu), base + ((rem >> 8) & 0xFFu), base + ((rem >> 16) & 0xFFu));
        }

#if defined(CFBPE_TILE_CLOCK) && !defined(CUSIM_EMULATOR)
        __syncwarp(); const long long tile_t3 = clock64();
#endif
        // ---- flags out: my 16 bits + what the lane to my left marked in my block; two lanes share a 32-bit word
        //      (30 blocks a warp: odd lanes hold even blocks)
        uint32_t v = mine & 0xFFFFu;
        const uint32_t spill = mine >> 16;
        const uint32_t incoming = __shfl_up_sync(kFull, spill, 1);
        if (lane) v |= incoming;
        const uint32_t nv = __shfl_down_sync(kFull, v, 1);
        if (blk >= 0) {
            const uint64_t wi = base >> 5;
            if (lane & 1u) {            // even block: low half; the odd block to my right is lane + 1 (lane 31, the ghost, has none in this warp)
                const uint32_t word = v | (lane == 31u ? 0u : (nv << 16));
                if (word) atomicOr(&piece_bits[wi], word);
            } else if (lane == 0u) {    // the ghost to the left owns nothing here
            }
        }
#if CFBPE_SPLIT_TICKETS
        tile = __shfl_sync(kFull, next_tile, 0);
#else
        tile = next_tile;
#endif
#if defined(CFBPE_TILE_CLOCK) && !defined(CUSIM_EMULATOR)
        __syncwarp();
        { const long long dt = clock64() - tile_t0; if (lane == 0 && dt > CFBPE_TILE_CLOCK) printf("slow tile %u: %lld cycles (classify %lld walk %lld resume %lld [%u lanes] out %lld)\n", tile_dbg, dt, tile_t1 - tile_t0, tile_t2 - tile_t1, tile_t3 - tile_t2, n_resume, clock64() - tile_t3); }
#endif
    }   // tiles
}

}  // namespace cfbpe
