// specials.h -- a vocabulary's special-token table: host builder and the device view the kernels read.
//
// A vocabulary may register up to kMaxSpecials special tokens of 1..kMaxSpecialLen bytes each (cfbpe_vocab_set_specials).
// The table is a few KB, built here on the host and copied to every device of the context; it is NOT part of the packed
// vocabulary blob (export / import / broadcast are unchanged).  Layout, in 32-bit words:
//   header (kSpHeaderWords)   n, n_lens, hash_mask and the word offset of every section
//   bm1   256 bits            a special starts with this byte
//   bm2   64 Kbit             ... with these two bytes (b0 | b1 << 8); a one-byte special sets all 256 bits of its b0
//   lens  64 bytes            the distinct lengths, ascending
//   hash  pow2 >= 2n slots    open addressing on (length, bytes): special index + 1, 0 = empty
//   ids   n                   token id of each special
//   offs  n + 1               byte offsets of the specials' bytes
//   sid / sidx  n each        the ids sorted, and the special index of each (decode looks an id up by binary search)
//   bytes                     the specials' bytes back to back
// A position is probed only when its first two bytes pass the bitmaps; the probe walks the bytes once, hashing every prefix,
// and looks up the prefixes whose length is one of the distinct lengths -- one hash probe per distinct length, so a set of
// prefix-sharing tokens (<|reserved_special_token_N|>) costs no scan over its members.
#pragma once
#include <stdint.h>

#include <algorithm>
#include <string>
#include <vector>

namespace cfbpe {

constexpr uint32_t kMaxSpecials = 4096;
constexpr uint32_t kMaxSpecialLen = 64;
constexpr uint32_t kSpHeaderWords = 16;
constexpr uint32_t kSpText = 0xFFFFFFFFu;      // stretch id of a text stretch (no special token has this id)
enum SpecialMode : uint8_t { kSpOrdinary = 0, kSpAllow = 1, kSpDisallow = 2 };   // = CFBPE_SPECIAL_*

struct SpecialView {
    const uint32_t* w;     // nullptr / n == 0: the vocabulary has no special tokens (or none this call looks for)
    uint32_t n, n_lens, hash_mask;
    uint32_t o_bm2, o_lens, o_hash, o_ids, o_offs, o_sid, o_sidx, o_bytes;
};

// everything the special-token kernels of one call read: one view per vocabulary slot, the call's mode bytes per vocabulary
// (nullptr = every special DISALLOWED, tiktoken's default) and the union of the first-byte bitmaps of the vocabularies in play
struct SpecialSet {
    SpecialView v[8];
    const uint8_t* modes[8];
    uint32_t first_bytes[8];
};

__host__ __device__ inline uint32_t sp_hash_init() { return 2166136261u; }
__host__ __device__ inline uint32_t sp_hash_step(uint32_t h, uint32_t byte) { return (h ^ byte) * 16777619u; }
__host__ __device__ inline uint32_t sp_hash_final(uint32_t h, uint32_t len) {
    h ^= len * 0x9E3779B1u;
    h ^= h >> 15; h *= 0x2C1B3C6Du; h ^= h >> 12;
    return h;
}
__host__ __device__ inline const uint8_t* sp_bytes(const SpecialView& V) { return reinterpret_cast<const uint8_t*>(V.w + V.o_bytes); }
__host__ __device__ inline uint32_t sp_len(const SpecialView& V, uint32_t k) { return V.w[V.o_offs + k + 1] - V.w[V.o_offs + k]; }

// the special whose bytes are p[0, len) (hash = sp_hash_final of them), or -1
__host__ __device__ inline int sp_find(const SpecialView& V, uint32_t hash, uint32_t len, const uint8_t* p) {
    const uint8_t* sb = sp_bytes(V);
    for (uint32_t s = hash & V.hash_mask;; s = (s + 1) & V.hash_mask) {
        const uint32_t e = V.w[V.o_hash + s];
        if (!e) return -1;
        const uint32_t k = e - 1, o = V.w[V.o_offs + k];
        if (V.w[V.o_offs + k + 1] - o != len) continue;
        uint32_t j = 0;
        while (j < len && sb[o + j] == p[j]) ++j;
        if (j == len) return static_cast<int>(k);
    }
}

// the special index of token id `id`, or -1 (binary search over the sorted ids)
__host__ __device__ inline int sp_by_id(const SpecialView& V, uint32_t id) {
    if (!V.w || !V.n) return -1;
    uint32_t lo = 0, hi = V.n;
    while (lo < hi) { const uint32_t m = (lo + hi) >> 1; if (V.w[V.o_sid + m] < id) lo = m + 1; else hi = m; }
    return (lo < V.n && V.w[V.o_sid + lo] == id) ? static_cast<int>(V.w[V.o_sidx + lo]) : -1;
}

inline SpecialView make_special_view(const uint32_t* dev_words, const std::vector<uint32_t>& host_words) {
    SpecialView v{};
    if (host_words.empty()) return v;
    const uint32_t* h = host_words.data();
    v.w = dev_words; v.n = h[0]; v.n_lens = h[1]; v.hash_mask = h[2];
    v.o_bm2 = h[4]; v.o_lens = h[5]; v.o_hash = h[6]; v.o_ids = h[7]; v.o_offs = h[8]; v.o_sid = h[9]; v.o_sidx = h[10]; v.o_bytes = h[11];
    return v;
}

// strict UTF-8 (no overlong forms, no surrogates, nothing above U+10FFFF): what a Python str encodes to
inline bool sp_valid_utf8(const uint8_t* p, uint64_t n) {
    for (uint64_t i = 0; i < n;) {
        const uint32_t c = p[i];
        uint32_t need, cp;
        if (c < 0x80) { ++i; continue; }
        else if (c >= 0xC2 && c <= 0xDF) { need = 1; cp = c & 0x1F; }
        else if (c >= 0xE0 && c <= 0xEF) { need = 2; cp = c & 0x0F; }
        else if (c >= 0xF0 && c <= 0xF4) { need = 3; cp = c & 0x07; }
        else return false;
        for (uint32_t k = 1; k <= need; ++k) {
            if (i + k >= n || (p[i + k] & 0xC0) != 0x80) return false;
            cp = (cp << 6) | (p[i + k] & 0x3F);
        }
        if ((need == 2 && (cp < 0x800 || (cp >= 0xD800 && cp <= 0xDFFF))) || (need == 3 && (cp < 0x10000 || cp > 0x10FFFF))) return false;
        i += need + 1;
    }
    return true;
}

// Build the table of n special tokens (token k = bytes[offsets[k], offsets[k+1]), id ids[k]).  n == 0: an empty table (no
// special tokens).  Returns 0 or CFBPE_EINVAL (-22) with a message: more than kMaxSpecials tokens, a token of 0 or more than
// kMaxSpecialLen bytes, invalid UTF-8, two tokens with the same bytes or the same id, or the id 0xFFFFFFFF.
inline int build_special_table(uint32_t n, const uint8_t* bytes, const uint64_t* offsets, const uint32_t* ids,
                               std::vector<uint32_t>& words, std::string& err) {
    constexpr int kEinval = -22;
    words.clear();
    if (n == 0) return 0;
    if (n > kMaxSpecials) { err = "at most " + std::to_string(kMaxSpecials) + " special tokens per vocabulary"; return kEinval; }
    if (!bytes || !offsets || !ids) { err = "bytes, offsets or ids is NULL"; return kEinval; }
    std::vector<std::string> toks(n);
    bool has_len[kMaxSpecialLen + 1] = {};
    for (uint32_t k = 0; k < n; ++k) {
        if (offsets[k + 1] < offsets[k]) { err = "special-token offsets decrease at token " + std::to_string(k); return kEinval; }
        const uint64_t len = offsets[k + 1] - offsets[k];
        if (len < 1 || len > kMaxSpecialLen) { err = "special token " + std::to_string(k) + " has " + std::to_string(len) + " bytes (1.." + std::to_string(kMaxSpecialLen) + ")"; return kEinval; }
        if (!sp_valid_utf8(bytes + offsets[k], len)) { err = "special token " + std::to_string(k) + " is not valid UTF-8"; return kEinval; }
        if (ids[k] == kSpText) { err = "special token " + std::to_string(k) + " has the reserved id 0xFFFFFFFF"; return kEinval; }
        toks[k].assign(reinterpret_cast<const char*>(bytes + offsets[k]), len);
        has_len[len] = true;
    }
    {
        std::vector<uint32_t> order(n);
        for (uint32_t k = 0; k < n; ++k) order[k] = k;
        std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return toks[a] < toks[b]; });
        for (uint32_t k = 1; k < n; ++k) if (toks[order[k]] == toks[order[k - 1]]) { err = "special tokens " + std::to_string(order[k - 1]) + " and " + std::to_string(order[k]) + " are the same bytes"; return kEinval; }
    }
    std::vector<uint32_t> sid(n);
    for (uint32_t k = 0; k < n; ++k) sid[k] = k;
    std::sort(sid.begin(), sid.end(), [&](uint32_t a, uint32_t b) { return ids[a] < ids[b]; });
    for (uint32_t k = 1; k < n; ++k) if (ids[sid[k]] == ids[sid[k - 1]]) { err = "two special tokens have the id " + std::to_string(ids[sid[k]]); return kEinval; }
    uint32_t hsize = 16;
    while (hsize < 2 * n) hsize <<= 1;
    uint64_t total_bytes = 0;
    for (const auto& t : toks) total_bytes += t.size();
    const uint32_t o_bm1 = kSpHeaderWords, o_bm2 = o_bm1 + 8, o_lens = o_bm2 + 2048, o_hash = o_lens + kMaxSpecialLen / 4;
    const uint32_t o_ids = o_hash + hsize, o_offs = o_ids + n, o_sid = o_offs + n + 1, o_sidx = o_sid + n, o_bytes = o_sidx + n;
    const uint32_t n_words = o_bytes + static_cast<uint32_t>((total_bytes + 3) / 4);
    words.assign(n_words, 0u);
    uint32_t n_lens = 0;
    uint8_t* lens = reinterpret_cast<uint8_t*>(words.data() + o_lens);
    for (uint32_t L = 1; L <= kMaxSpecialLen; ++L) if (has_len[L]) lens[n_lens++] = static_cast<uint8_t>(L);
    uint32_t* h = words.data();
    h[0] = n; h[1] = n_lens; h[2] = hsize - 1; h[3] = o_bm1; h[4] = o_bm2; h[5] = o_lens; h[6] = o_hash; h[7] = o_ids;
    h[8] = o_offs; h[9] = o_sid; h[10] = o_sidx; h[11] = o_bytes; h[12] = n_words;
    uint8_t* sb = reinterpret_cast<uint8_t*>(words.data() + o_bytes);
    uint32_t off = 0;
    for (uint32_t k = 0; k < n; ++k) {
        const std::string& t = toks[k];
        const uint32_t b0 = static_cast<uint8_t>(t[0]);
        words[o_bm1 + (b0 >> 5)] |= 1u << (b0 & 31);
        for (uint32_t b1 = 0; b1 < 256; ++b1) {
            if (t.size() > 1 && b1 != static_cast<uint8_t>(t[1])) continue;
            const uint32_t pair = b0 | (b1 << 8);
            words[o_bm2 + (pair >> 5)] |= 1u << (pair & 31);
        }
        words[o_ids + k] = ids[k];
        words[o_offs + k] = off;
        std::copy(t.begin(), t.end(), sb + off);
        off += static_cast<uint32_t>(t.size());
        uint32_t hv = sp_hash_init();
        for (unsigned char c : t) hv = sp_hash_step(hv, c);
        hv = sp_hash_final(hv, static_cast<uint32_t>(t.size()));
        uint32_t s = hv & (hsize - 1);
        while (words[o_hash + s]) s = (s + 1) & (hsize - 1);
        words[o_hash + s] = k + 1;
    }
    words[o_offs + n] = off;
    for (uint32_t k = 0; k < n; ++k) { words[o_sid + k] = ids[sid[k]]; words[o_sidx + k] = sid[k]; }
    return 0;
}

}  // namespace cfbpe
