// utf8_repair.cuh -- encode bytes that are not valid UTF-8 as if they had first been decoded with Python's
// bytes.decode("utf-8", errors="replace") and encoded again (cfbpe_encode_batch_lossy).
//
// The rule is the Unicode Standard's "substitution of maximal subparts" (chapter 3, U+FFFD substitution), which CPython,
// String::from_utf8_lossy and the WHATWG decoder follow: every byte that is not a continuation byte (80..BF) starts a unit; a unit
// takes the continuation bytes of the longest valid prefix of the sequence its lead byte starts, and is valid when that prefix is a
// whole character.  A continuation byte outside every unit is a unit of its own (a stray).  An invalid unit -- a maximal subpart or
// a stray -- becomes one U+FFFD (EF BF BD).  Prefixes stop at a prompt boundary: a sequence never spans two prompts.
//
// Since a lead byte's prefix is at most 4 bytes long, a byte's unit is decided by the 3 bytes before it and the 3 after it, so a
// lane of 16 bytes decides its own units from a window of 24 bytes (utf8_window):
//   utf8_scan           a lane per 16 bytes: the growth of its bytes (3 - length, summed over the invalid units that start in
//                       them) summed per 4 KiB tile, its invalid units added to their prompts' replaced counts, and one atomic
//                       per lane with an invalid unit on the status (lanes with one, total growth)
// The host reads the status (the call's one synchronisation).  No invalid unit: the ordinary path runs on the bytes as they are.
// Else the repaired batch R is written and the ordinary path runs on it:
//   tile_scan           exclusive scan of the tile growths
//   utf8_repair_emit    a lane per 16 bytes again: its place in R (the tile's base + a scan inside the tile), its bytes written
//                       there with EF BF BD for every invalid unit that starts in them, and the growth before it (lane_base)
//   utf8_repair_offsets a thread per prompt: its offset in R
#pragma once
#include "pipeline.cuh"

namespace cfbpe {

// what the scan leaves: lanes_growth = (lanes with an invalid unit) << kLossyLaneShift | (total growth).  A batch has fewer than
// 2^28 lanes (max_batch_bytes < 4 GiB) and grows by less than 2^33 bytes, so one 64-bit add per dirty lane carries both.
constexpr uint32_t kLossyLaneShift = 36;
struct LossyStatus {
    unsigned long long lanes_growth;
};

// what the host learns from a scan: whether some byte is not valid UTF-8, and the size of the repaired batch
struct LossyScanResult { bool dirty; uint64_t total; };
inline LossyScanResult lossy_scan_result(const LossyStatus& st, uint64_t total_bytes) {
    return LossyScanResult{(st.lanes_growth >> kLossyLaneShift) != 0,
                           total_bytes + (st.lanes_growth & ((1ull << kLossyLaneShift) - 1ull))};
}

// the buffers of a lossy call beside the workspace (the scan's scratch lives in the workspace: pstart_bits, the tile arrays of the
// dense ids and lscratch.aux0, all dead until the ordinary pass starts)
struct LossyWork {
    uint32_t* replaced;     // [n_prompts]     U+FFFD inserted per prompt
    uint64_t* offsets;      // [n_prompts + 1] the prompts' offsets in R
    LossyStatus* status;
};

constexpr uint32_t kUtf8Cta = 256;                    // lanes of 16 bytes per CTA: a tile of 4 KiB
constexpr uint64_t kUtf8Tile = 16ull * kUtf8Cta;

inline uint32_t n_utf8_tiles(uint64_t total_bytes) { return static_cast<uint32_t>((total_bytes + kUtf8Tile - 1) / kUtf8Tile); }

// bytes [p, p + 4) with aligned 32-bit loads (p may be unaligned; the furthest byte read is p + 7)
__device__ __forceinline__ uint32_t utf8_load4(const uint8_t* __restrict__ p) {
    const uintptr_t a = reinterpret_cast<uintptr_t>(p);
    const uint32_t* q = reinterpret_cast<const uint32_t*>(a & ~static_cast<uintptr_t>(3));
    const uint32_t sh = static_cast<uint32_t>(a & 3) * 8;
    return sh ? __funnelshift_r(q[0], q[1], sh) : q[0];
}

// The window of the lane at base (< total): byte t of q is byte base - 4 + t (t < 24; the 4 bytes before the batch read as 0), bit
// t of bnd says that a prompt starts (or the data ends) at base - 4 + t, and bit j of own that base + j is inside the batch.  The
// furthest byte read is base + 23, within the 32 readable bytes past the batch.
struct Utf8Window { uint64_t q[3]; uint32_t bnd, own; };
__device__ __forceinline__ Utf8Window utf8_window(const BatchView& b, const uint32_t* __restrict__ pstart_bits, uint64_t base) {
    uint32_t w0, w1, w2, w3;
    if ((reinterpret_cast<uintptr_t>(b.bytes) & 15u) == 0) {
        const uint4 v = *reinterpret_cast<const uint4*>(b.bytes + base); w0 = v.x; w1 = v.y; w2 = v.z; w3 = v.w;
    } else {
        load16(b.bytes + base, w0, w1, w2, w3);      // a device-path caller's buffer that is not 16-byte aligned
    }
    const uint32_t before = base ? utf8_load4(b.bytes + base - 4) : 0u;
    const uint32_t after = utf8_load4(b.bytes + base + 16);
    Utf8Window v;
    v.q[0] = before | (static_cast<uint64_t>(w0) << 32);
    v.q[1] = w1 | (static_cast<uint64_t>(w2) << 32);
    v.q[2] = w3 | (static_cast<uint64_t>(after) << 32);
    if (base) {
        const uint64_t p = base - 4, wi = p >> 5;
        const uint64_t bits = pstart_bits[wi] | (static_cast<uint64_t>(pstart_bits[wi + 1]) << 32);
        v.bnd = static_cast<uint32_t>(bits >> (p & 31)) & 0xFFFFFFu;
    } else {
        v.bnd = static_cast<uint32_t>((pstart_bits[0] | (static_cast<uint64_t>(pstart_bits[1]) << 32)) << 4) & 0xFFFFFFu;
    }
    const uint64_t left = b.total_bytes - base;
    v.own = left >= 16 ? 0xFFFFu : (1u << left) - 1u;
    return v;
}

__device__ __forceinline__ uint32_t utf8_byte(const Utf8Window& v, uint32_t t) { return static_cast<uint32_t>(v.q[t >> 3] >> (8 * (t & 7))) & 0xFFu; }

// the length (1 .. 4) of the maximal valid prefix of the sequence the lead byte at window position t starts, and whether it is a
// whole character.  A byte at a prompt boundary ends the prefix.
__device__ __forceinline__ uint32_t utf8_prefix(const Utf8Window& v, uint32_t t, bool& valid) {
    const uint32_t c0 = utf8_byte(v, t);
    const uint32_t need = c0 < 0x80u ? 1u : c0 < 0xC2u ? 0u : c0 < 0xE0u ? 2u : c0 < 0xF0u ? 3u : c0 < 0xF5u ? 4u : 0u;
    if (need <= 1) { valid = need == 1; return 1; }
    const uint32_t lo = c0 == 0xE0u ? 0xA0u : (c0 == 0xF0u ? 0x90u : 0x80u);      // no overlong
    const uint32_t hi = c0 == 0xEDu ? 0x9Fu : (c0 == 0xF4u ? 0x8Fu : 0xBFu);      // no surrogate, nothing above U+10FFFF
    const uint32_t c1 = utf8_byte(v, t + 1), c2 = utf8_byte(v, t + 2), c3 = utf8_byte(v, t + 3);
    uint32_t len = 1;
    if (!((v.bnd >> (t + 1)) & 1u) && c1 >= lo && c1 <= hi) {
        len = 2;
        if (need > 2 && !((v.bnd >> (t + 2)) & 1u) && (c2 & 0xC0u) == 0x80u) {
            len = 3;
            if (need > 3 && !((v.bnd >> (t + 3)) & 1u) && (c3 & 0xC0u) == 0x80u) len = 4;
        }
    }
    valid = len == need;
    return len;
}

// the invalid units among the lane's own bytes, bit j for base + j:
//   start   an invalid unit (a maximal subpart or a stray) starts here
//   inside  the byte is inside an invalid unit that started before it (in this lane or the one before)
//   cover   ... of one that started in this lane (bits up to 18: a unit may run 3 bytes past the lane)
struct Utf8Units { uint32_t start, inside, cover; };
__device__ __forceinline__ Utf8Units utf8_units(const Utf8Window& v) {
    uint32_t cont = 0;
#pragma unroll
    for (uint32_t t = 1; t < 20; ++t) if ((utf8_byte(v, t) & 0xC0u) == 0x80u) cont |= 1u << t;
    const uint32_t own = v.own << 4;
    uint32_t cov_valid = 0, cov_bad = 0, cov_own = 0, lead_bad = 0;
#pragma unroll
    for (uint32_t t = 1; t < 20; ++t) {          // a lead more than 3 bytes before the lane covers none of its bytes
        bool valid;
        const uint32_t len = utf8_prefix(v, t, valid);
        const uint32_t cov = (((1u << len) - 1u) << t) & ~(1u << t);
        const bool lead = !((cont >> t) & 1u);
        if (lead && valid) cov_valid |= cov;
        if (lead && !valid) {
            cov_bad |= cov;
            if ((own >> t) & 1u) { lead_bad |= 1u << t; cov_own |= cov; }
        }
    }
    const uint32_t stray = cont & ~(cov_valid | cov_bad) & own;
    return Utf8Units{(lead_bad | stray) >> 4, (cov_bad & own) >> 4, cov_own >> 4};
}
// bytes R gains over the lane's bytes before base + k (k <= 16): 3 - length for every invalid unit that starts there (k = 16:
// every unit of the lane, with the bytes past it that its last one covers)
__device__ __forceinline__ uint32_t utf8_growth(const Utf8Units& u, uint32_t k) {
    const uint32_t m = k >= 16 ? ~0u : (1u << k) - 1u;
    return 2u * __popc(u.start & m) - __popc(u.cover & m);
}
// the lane's 16 bytes are ASCII: each is a valid unit of its own (the common case; bytes past the batch may make it false)
__device__ __forceinline__ bool utf8_ascii(const Utf8Window& v) {
    return (((v.q[0] >> 32) | v.q[1] | (v.q[2] << 32)) & 0x8080808080808080ull) == 0;
}

__global__ void __launch_bounds__(kUtf8Cta)
utf8_scan_kernel(BatchView b, const uint32_t* __restrict__ pstart_bits, uint32_t* __restrict__ tile_growth, uint32_t* __restrict__ replaced,
                 LossyStatus* status) {
    __shared__ uint32_t s_warp[kUtf8Cta / 32];
    const uint64_t base = (static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x) * 16ull;
    uint32_t growth = 0;
    if (base < b.total_bytes) {
        const Utf8Window v = utf8_window(b, pstart_bits, base);
        const Utf8Units u = utf8_ascii(v) ? Utf8Units{0u, 0u, 0u} : utf8_units(v);
        if (u.start) {
            growth = utf8_growth(u, 16);
            atomicAdd(&status->lanes_growth, (1ull << kLossyLaneShift) | growth);
            uint32_t p = find_prompt(b.offsets, b.n_prompts, base + (__ffs(u.start) - 1));
            uint64_t pend = b.offsets[p + 1];
            uint32_t run = 0;
            for (uint32_t s = u.start; s; s &= s - 1) {
                const uint64_t q = base + (__ffs(s) - 1);
                if (q >= pend) {
                    atomicAdd(&replaced[p], run);
                    run = 0;
                    while (q >= pend) { ++p; pend = b.offsets[p + 1]; }      // (empty prompts are skipped over)
                }
                ++run;
            }
            atomicAdd(&replaced[p], run);
        }
    }
#pragma unroll
    for (uint32_t d = 16; d; d >>= 1) growth += __shfl_xor_sync(kFull, growth, d);
    if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = growth;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t sum = 0;
        for (uint32_t w = 0; w < kUtf8Cta / 32; ++w) sum += s_warp[w];
        tile_growth[blockIdx.x] = sum;
    }
}

// out: R, out + tile_base[tile] + (growth of the lanes before this one in the tile) is where the lane's first own byte goes;
// lane_base: that growth before every lane, for utf8_repair_offsets
__global__ void __launch_bounds__(kUtf8Cta)
utf8_repair_emit_kernel(BatchView b, const uint32_t* __restrict__ pstart_bits, const uint64_t* __restrict__ tile_base, uint8_t* __restrict__ out,
                        uint64_t* __restrict__ lane_base) {
    __shared__ uint32_t s_warp[kUtf8Cta / 32];
    const uint64_t lane_idx = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    const uint64_t base = lane_idx * 16ull;
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    Utf8Window v{};
    Utf8Units u{0u, 0u, 0u};
    if (base < b.total_bytes) {
        v = utf8_window(b, pstart_bits, base);
        if (!utf8_ascii(v)) u = utf8_units(v);
    }
    const uint32_t growth = utf8_growth(u, 16);
    uint32_t x = growth;
#pragma unroll
    for (uint32_t d = 1; d < 32; d <<= 1) { const uint32_t o = __shfl_up_sync(kFull, x, d); if (lane >= d) x += o; }
    if (lane == 31) s_warp[wid] = x;
    __syncthreads();
    uint32_t before = x - growth;
    for (uint32_t w = 0; w < wid; ++w) before += s_warp[w];
    if (base >= b.total_bytes) return;
    const uint64_t g = tile_base[blockIdx.x] + before;
    lane_base[lane_idx] = g;
    // base + g is where byte base goes: an invalid unit that starts here takes 3 bytes for its length, one that started in the
    // lane before has its growth in g already (its bytes here keep their places, unwritten)
    uint8_t* o = out + base + g;
#pragma unroll
    for (uint32_t j = 0; j < 16; ++j) {
        if (!((v.own >> j) & 1u)) break;
        if ((u.start >> j) & 1u) { o[0] = 0xEFu; o[1] = 0xBFu; o[2] = 0xBDu; o += 3; }
        else if (!((u.inside >> j) & 1u)) *o++ = static_cast<uint8_t>(utf8_byte(v, j + 4));
        else if (!((u.cover >> j) & 1u)) ++o;
    }
}

// out_offsets[i] = prompt i's offset in R (r_total for the end of the data)
__global__ void __launch_bounds__(256)
utf8_repair_offsets_kernel(BatchView b, const uint32_t* __restrict__ pstart_bits, const uint64_t* __restrict__ lane_base, uint64_t r_total,
                           uint64_t* __restrict__ out_offsets) {
    const uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i > b.n_prompts) return;
    const uint64_t x = b.offsets[i];
    if (x >= b.total_bytes) { out_offsets[i] = r_total; return; }
    const uint64_t base = x & ~15ull;
    const Utf8Window v = utf8_window(b, pstart_bits, base);
    const Utf8Units u = utf8_ascii(v) ? Utf8Units{0u, 0u, 0u} : utf8_units(v);
    out_offsets[i] = x + lane_base[x >> 4] + utf8_growth(u, static_cast<uint32_t>(x - base));    // (a prompt start starts a unit)
}

inline uint64_t* utf8_lane_base(const Workspace& w) { return reinterpret_cast<uint64_t*>(w.lscratch.aux0); }   // [total / 16] <= 4 B a byte

// The scan: lw.status and lw.replaced zeroed, the prompt-start bits of the batch (prompt_map_kernel, which the ordinary pass
// runs again), then utf8_scan.  The host reads lw.status next (lossy_scan_result).
template <typename Stream>
inline void enqueue_utf8_scan(const BatchView& b, const VocabSet& vs, const Workspace& w, const LossyWork& lw, Stream stream) {
    CFBPE_ZERO(lw.status, sizeof(LossyStatus), stream);
    if (b.n_prompts) CFBPE_ZERO(lw.replaced, static_cast<uint64_t>(b.n_prompts) * sizeof(uint32_t), stream);
    if (!b.total_bytes) return;
    CFBPE_ZERO(w.pstart_bits, (n_flag_words(b.total_bytes) + 2) * sizeof(uint32_t), stream);
    CFBPE_LAUNCH(prompt_map_kernel, static_cast<unsigned>((static_cast<uint64_t>(b.n_prompts) + 1 + 255) / 256), 256, stream, b, vs, w.pstart_bits,
                 w.block_prompt, w.status);
    CFBPE_LAUNCH(utf8_scan_kernel, n_utf8_tiles(b.total_bytes), kUtf8Cta, stream, b, static_cast<const uint32_t*>(w.pstart_bits), w.dense.tile_pieces,
                 lw.replaced, lw.status);
}

// The repair, after a scan of raw that found an invalid unit: R (r_total bytes) into out_bytes, which must not overlap raw's bytes
// and must hold r_total + 32 bytes, and the prompts' offsets in R into lw.offsets.  raw.bytes may be a copy of the scanned bytes.
template <typename Stream>
inline void enqueue_utf8_repair(const BatchView& raw, const Workspace& w, const LossyWork& lw, uint8_t* out_bytes, uint64_t r_total, Stream stream) {
    const uint32_t n_tiles = n_utf8_tiles(raw.total_bytes);
    CFBPE_LAUNCH(tile_scan_kernel, 1u, 1024, stream, static_cast<const uint32_t*>(w.dense.tile_pieces), n_tiles, w.dense.piece_base,
                 static_cast<DeviceStatus*>(nullptr), static_cast<const uint64_t*>(nullptr));
    CFBPE_LAUNCH(utf8_repair_emit_kernel, n_tiles, kUtf8Cta, stream, raw, static_cast<const uint32_t*>(w.pstart_bits),
                 static_cast<const uint64_t*>(w.dense.piece_base), out_bytes, utf8_lane_base(w));
    CFBPE_LAUNCH(utf8_repair_offsets_kernel, static_cast<unsigned>((static_cast<uint64_t>(raw.n_prompts) + 1 + 255) / 256), 256, stream, raw,
                 static_cast<const uint32_t*>(w.pstart_bits), static_cast<const uint64_t*>(utf8_lane_base(w)), r_total, lw.offsets);
}

}  // namespace cfbpe
