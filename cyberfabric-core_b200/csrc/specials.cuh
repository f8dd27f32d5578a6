// specials.cuh -- encode with special tokens (tiktoken's Encoding.encode with allowed / disallowed specials) on the device.
//
//   special_scan      a lane per 16 bytes: positions whose first byte starts some special are probed (specials.h); the longest
//                     ALLOWED match of a position is marked (a bit per byte + its length and index), a DISALLOWED occurrence of
//                     any length is reported (the leftmost wins)
//   special_resolve   a warp per prompt: keeps the non-overlapping leftmost-longest matches (a match is dropped iff a kept one
//                     before it covers it), counts them (m_i), names the prompt of the reported disallowed occurrence
//   tile_scan         exclusive scan of m_i
//   special_layout    a warp per prompt: prompt i becomes 2 m_i + 1 stretches, text / special / text / ... / text, at stretch
//                     index i + 2 (m_0 + .. + m_{i-1}); a stretch's bytes, vocabulary and id (kSpText for text)
//   (the ordinary path, enqueue_encode, on the stretches as prompts: each text stretch ends where tiktoken's slice ends)
//   special_mark      a special stretch counts one token (the ordinary ids of its bytes are thrown away)
//   tile_scan         exclusive scan of the stretch counts: where each stretch's ids go
//   special_splice    a warp per stretch: a text stretch's ids, copied with coalesced warp loads and stores; a special's id
//   special_offsets   the prompts' offsets and counts
// The scan, the resolve and the first scan come first (enqueue_special_scan); the host learns the number of kept matches from
// the status they leave and then either runs the ordinary path on the prompts as they are (no match, nothing disallowed) or
// the rest (enqueue_encode_special).
#pragma once
#include "pipeline.cuh"
#include "specials.h"

namespace cfbpe {

struct SpecialStatus {
    unsigned long long bad_inv;   // ~(position << 15 | vocab << 12 | special index) of the leftmost DISALLOWED occurrence (0: none): atomicMax
    uint32_t bad_prompt;          // the prompt that holds it (special_resolve)
    uint32_t pad;
    DeviceStatus kept;            // tile_scan of the kept matches per prompt: kept.n_tokens = matches in all
    DeviceStatus fin;             // tile_scan of the stretch counts: fin.n_tokens = ids of the call
};

// the buffers of a special call beside the workspace (the candidate marks live in the workspace's tok_bits / ids_by_pos: they
// are dead until the ordinary pass starts)
struct SpecialWork {
    uint32_t* kept_n;       // [n_prompts]       kept matches per prompt
    uint64_t* kept_base;    // [n_prompts]       their exclusive scan
    uint64_t* st_off;       // [n_stretches + 1] stretch byte offsets
    uint8_t* st_vocab;      // [n_stretches]     stretch vocabulary (when the call has per-prompt vocabularies)
    uint32_t* st_id;        // [n_stretches]     special id, or kSpText
    uint64_t* st_base;      // [n_stretches]     first id of each stretch in the output
    SpecialStatus* status;
};

__global__ void __launch_bounds__(256)
special_scan_kernel(BatchView b, SpecialSet sp, uint32_t* __restrict__ cand_bits, uint32_t* __restrict__ cand_info, SpecialStatus* status) {
    __shared__ uint32_t s_first[8];
    if (threadIdx.x < 8) s_first[threadIdx.x] = sp.first_bytes[threadIdx.x];
    __syncthreads();
    const uint64_t base = (static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x) * 16ull;
    if (base >= b.total_bytes) return;
    uint32_t ww[4];
    if ((reinterpret_cast<uintptr_t>(b.bytes) & 15u) == 0) {
        const uint4 v = *reinterpret_cast<const uint4*>(b.bytes + base); ww[0] = v.x; ww[1] = v.y; ww[2] = v.z; ww[3] = v.w;
    } else {
        load16(b.bytes + base, ww[0], ww[1], ww[2], ww[3]);      // a device-path caller's buffer that is not 16-byte aligned
    }
    const uint64_t left = b.total_bytes - base;
    uint32_t hits = 0;
#pragma unroll
    for (uint32_t j = 0; j < 16; ++j) {
        const uint32_t c = (ww[j >> 2] >> (8 * (j & 3))) & 0xFFu;
        if (j < left && ((s_first[c >> 5] >> (c & 31)) & 1u)) hits |= 1u << j;
    }
    if (!hits) return;
    uint32_t prompt = find_prompt(b.offsets, b.n_prompts, base + (__ffs(hits) - 1));
    uint64_t pend = b.offsets[prompt + 1];
    for (; hits; hits &= hits - 1) {
        const uint64_t q = base + (__ffs(hits) - 1);
        while (q >= pend) { ++prompt; pend = b.offsets[prompt + 1]; }      // (empty prompts are skipped over)
        const uint32_t vid = b.vocab_ids ? b.vocab_ids[prompt] : 0u;
        if (vid >= kMaxVocabs) continue;                                 // reported by the ordinary pass (bad_vocab)
        const SpecialView& V = sp.v[vid];
        if (!V.w || !V.n) continue;
        const uint8_t* p = b.bytes + q;
        const uint32_t pair = p[0] | (q + 1 < pend ? static_cast<uint32_t>(p[1]) << 8 : 0u);
        const uint32_t bits2 = __ldg(V.w + V.o_bm2 + (pair >> 5));
        if (q + 1 < pend && !((bits2 >> (pair & 31)) & 1u)) continue;
        // every prefix of the bytes at q whose length is a special's: one hash probe each, ascending
        const uint64_t room = pend - q;
        const uint32_t maxlen = room < kMaxSpecialLen ? static_cast<uint32_t>(room) : kMaxSpecialLen;
        const uint8_t* lens = reinterpret_cast<const uint8_t*>(V.w + V.o_lens);
        const uint8_t* modes = sp.modes[vid];
        int allow = -1, bad = -1;
        uint32_t allow_len = 0, li = 0, h = sp_hash_init();
        for (uint32_t k = 0; k < maxlen && li < V.n_lens; ++k) {
            h = sp_hash_step(h, p[k]);
            if (lens[li] != k + 1) continue;
            ++li;
            const int idx = sp_find(V, sp_hash_final(h, k + 1), k + 1, p);
            if (idx < 0) continue;
            const uint32_t mode = modes ? modes[idx] : static_cast<uint32_t>(kSpDisallow);
            if (mode == kSpAllow) { allow = idx; allow_len = k + 1; }
            else if (mode == kSpDisallow) bad = idx;
        }
        if (bad >= 0) atomicMax(&status->bad_inv, ~((static_cast<unsigned long long>(q) << 15) | (vid << 12) | static_cast<uint32_t>(bad)));
        if (allow >= 0) {
            atomicOr(&cand_bits[q >> 5], 1u << (q & 31));
            cand_info[q] = (allow_len << 16) | static_cast<uint32_t>(allow);
        }
    }
}

// The marks of prompt i, a warp at a time over its bit words (32 words = 1 KiB a trip); visit(pos, info) for every mark in
// order, warp-uniform.  keep(pos, info) decides; the marks it drops are cleared (atomically: a word may hold two prompts).
template <bool kResolve, typename F>
__device__ __forceinline__ void special_walk(uint32_t* __restrict__ cand_bits, const uint32_t* __restrict__ cand_info, uint64_t lo, uint64_t hi, F&& visit) {
    if (lo >= hi) return;
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t wlo = lo >> 5, whi = (hi - 1) >> 5;
    for (uint64_t w0 = wlo; w0 <= whi; w0 += 32) {
        const uint64_t w = w0 + lane;
        uint32_t bits = w <= whi ? cand_bits[w] : 0u;
        if (w == wlo) bits &= ~0u << (lo & 31);
        if (w == whi && ((hi & 31) != 0)) bits &= (1u << (hi & 31)) - 1u;
        for (uint32_t nz = __ballot_sync(kFull, bits != 0); nz; nz &= nz - 1) {
            const uint32_t src = __ffs(nz) - 1;
            const uint32_t wb = __shfl_sync(kFull, bits, src);
            uint32_t dropped = 0;
            for (uint32_t rest = wb; rest; rest &= rest - 1) {
                const uint32_t bit = __ffs(rest) - 1;
                const uint64_t pos = ((w0 + src) << 5) + bit;
                if (!visit(pos, cand_info[pos])) dropped |= 1u << bit;
            }
            if (kResolve && lane == src && dropped) atomicAnd(&cand_bits[w], ~dropped);
        }
    }
}

__global__ void __launch_bounds__(256)
special_resolve_kernel(BatchView b, uint32_t* __restrict__ cand_bits, const uint32_t* __restrict__ cand_info, uint32_t* __restrict__ kept_n,
                       SpecialStatus* status) {
    const uint64_t i = (static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    if (i >= b.n_prompts) return;
    const uint64_t lo = b.offsets[i], hi = b.offsets[i + 1];
    const unsigned long long bad = status->bad_inv;
    if (bad && (threadIdx.x & 31) == 0) {
        const uint64_t pos = (~bad) >> 15;
        if (pos >= lo && pos < hi) status->bad_prompt = static_cast<uint32_t>(i);
    }
    uint64_t last_end = lo;
    uint32_t m = 0;
    special_walk<true>(cand_bits, cand_info, lo, hi, [&](uint64_t pos, uint32_t info) {
        if (pos < last_end) return false;
        last_end = pos + (info >> 16);
        ++m;
        return true;
    });
    if ((threadIdx.x & 31) == 0) kept_n[i] = m;
}

__global__ void __launch_bounds__(256)
special_layout_kernel(BatchView b, SpecialSet sp, uint32_t* __restrict__ cand_bits, const uint32_t* __restrict__ cand_info, SpecialWork sw,
                      uint32_t n_stretches) {
    const uint64_t i = (static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    if (i >= b.n_prompts) return;
    const bool lead = (threadIdx.x & 31) == 0;
    const uint64_t lo = b.offsets[i], hi = b.offsets[i + 1];
    const uint32_t vid = b.vocab_ids ? b.vocab_ids[i] : 0u;
    uint64_t s = i + 2 * sw.kept_base[i];
    auto put = [&](uint64_t k, uint64_t off, uint32_t id) {
        sw.st_off[k] = off; sw.st_id[k] = id;
        if (b.vocab_ids) sw.st_vocab[k] = static_cast<uint8_t>(vid);
    };
    if (lead) put(s, lo, kSpText);
    const SpecialView& V = sp.v[vid < kMaxVocabs ? vid : 0u];
    special_walk<false>(cand_bits, cand_info, lo, hi, [&](uint64_t pos, uint32_t info) {
        if (lead) { put(s + 1, pos, V.w[V.o_ids + (info & 0xFFFFu)]); put(s + 2, pos + (info >> 16), kSpText); }
        s += 2;
        return true;
    });
    if (lead && i + 1 == b.n_prompts) sw.st_off[n_stretches] = b.total_bytes;
}

__global__ void __launch_bounds__(256)
special_mark_kernel(const uint32_t* __restrict__ st_id, uint32_t n_stretches, uint32_t* __restrict__ counts) {
    const uint64_t s = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (s < n_stretches && st_id[s] != kSpText) counts[s] = 1;
}

__global__ void __launch_bounds__(256)
special_splice_kernel(SpecialWork sw, uint32_t n_stretches, const uint32_t* __restrict__ ord_ids, const uint64_t* __restrict__ ord_offsets,
                      const uint32_t* __restrict__ counts, uint32_t* __restrict__ out_ids, uint64_t out_cap) {
    const uint64_t s = (static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    if (s >= n_stretches) return;
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t dst = sw.st_base[s];
    const uint32_t id = sw.st_id[s];
    if (id != kSpText) { if (lane == 0 && dst < out_cap) out_ids[dst] = id; return; }
    const uint64_t src = ord_offsets[s];
    const uint32_t cnt = counts[s];
    for (uint32_t k = lane; k < cnt; k += 32) if (dst + k < out_cap) out_ids[dst + k] = __ldg(ord_ids + src + k);
}

__global__ void __launch_bounds__(256)
special_offsets_kernel(BatchView b, SpecialWork sw, uint64_t* __restrict__ out_offsets, uint32_t* __restrict__ out_counts) {
    const uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i > b.n_prompts) return;
    auto first_id = [&](uint64_t p) -> uint64_t {       // rank of the first id of prompt p (p == n_prompts: the total)
        return p < b.n_prompts ? sw.st_base[p + 2 * sw.kept_base[p]] : sw.status->fin.n_tokens;
    };
    const uint64_t r = first_id(i);
    out_offsets[i] = r;
    if (i < b.n_prompts && out_counts) out_counts[i] = static_cast<uint32_t>(first_id(i + 1) - r);
}

// the first half of a special call: marks, kept matches, their scan (status->kept.n_tokens, status->bad_inv / bad_prompt)
template <typename Stream>
inline void enqueue_special_scan(const BatchView& b, const SpecialSet& sp, const Workspace& w, const SpecialWork& sw, Stream stream) {
    CFBPE_ZERO(sw.status, sizeof(SpecialStatus), stream);
    if (!b.n_prompts) return;
    CFBPE_ZERO(w.tok_bits, (n_flag_words(b.total_bytes) + 2) * sizeof(uint32_t), stream);
    if (b.total_bytes)
        CFBPE_LAUNCH(special_scan_kernel, static_cast<unsigned>((b.total_bytes + 16ull * 256 - 1) / (16ull * 256)), 256, stream, b, sp, w.tok_bits, w.ids_by_pos, sw.status);
    CFBPE_LAUNCH(special_resolve_kernel, static_cast<unsigned>((static_cast<uint64_t>(b.n_prompts) + 7) / 8), 256, stream, b, w.tok_bits, w.ids_by_pos, sw.kept_n, sw.status);
    CFBPE_LAUNCH(tile_scan_kernel, 1u, 1024, stream, sw.kept_n, b.n_prompts, sw.kept_base, &sw.status->kept, static_cast<const uint64_t*>(nullptr));
}

// The second half, once the host knows n_stretches = n_prompts + 2 x kept matches (> n_prompts): stretches, the ordinary path on
// them (its ids, offsets and counts go to the scratch buffers ord_*, which hold n_stretches prompts / total_bytes ids), the splice
// into out_ids (nullptr: counts only), out_offsets and out_counts.
template <typename Stream, typename Ev, typename Prof>
inline void enqueue_encode_special(const BatchView& b, const SpecialSet& sp, const VocabSet& vs, const UcTables& uc, const Workspace& w,
                                   const SpecialWork& sw, uint32_t n_stretches, uint32_t* ord_ids, uint64_t ord_cap, uint64_t* ord_offsets,
                                   uint32_t* ord_counts, uint32_t* out_ids, uint64_t out_cap, uint64_t* out_offsets, uint32_t* out_counts,
                                   uint32_t long_grid, Stream stream, Stream aux, Stream aux2, Ev ev_fork, Ev ev_join, Ev ev_join2, Prof* prof) {
    CFBPE_LAUNCH(special_layout_kernel, static_cast<unsigned>((static_cast<uint64_t>(b.n_prompts) + 7) / 8), 256, stream, b, sp, w.tok_bits, w.ids_by_pos, sw, n_stretches);
    const BatchView st{b.bytes, sw.st_off, b.vocab_ids ? sw.st_vocab : nullptr, n_stretches, b.total_bytes};
    enqueue_encode(st, vs, uc, w, out_ids ? ord_ids : nullptr, ord_cap, ord_offsets, ord_counts, long_grid, stream, aux, aux2, ev_fork, ev_join, ev_join2, prof);
    const unsigned g = static_cast<unsigned>((static_cast<uint64_t>(n_stretches) + 255) / 256);
    CFBPE_LAUNCH(special_mark_kernel, g, 256, stream, sw.st_id, n_stretches, ord_counts);
    CFBPE_LAUNCH(tile_scan_kernel, 1u, 1024, stream, ord_counts, n_stretches, sw.st_base, &sw.status->fin, static_cast<const uint64_t*>(nullptr));
    if (out_ids)
        CFBPE_LAUNCH(special_splice_kernel, static_cast<unsigned>((static_cast<uint64_t>(n_stretches) + 7) / 8), 256, stream, sw, n_stretches, ord_ids, ord_offsets,
                     ord_counts, out_ids, out_cap);
    CFBPE_LAUNCH(special_offsets_kernel, static_cast<unsigned>((static_cast<uint64_t>(b.n_prompts) + 1 + 255) / 256), 256, stream, b, sw, out_offsets, out_counts);
}

}  // namespace cfbpe
