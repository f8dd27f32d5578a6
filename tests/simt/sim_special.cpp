// sim_special.cpp -- the special-token path (csrc/specials.h, csrc/specials.cuh) on the CPU SIMT emulator.
// TEST INFRASTRUCTURE: built by tests/simt/build_special.py into tests/simt/_build/libcfbpe_sim_special.so, next to
// everything sim_harness.cpp exports.  The special set (fill_special_set) and the reading of the scan (special_scan_result) are
// the library's host code; between them the scan, then the ordinary path on the prompts as they are (no kept match) or on the
// stretches followed by the splice, as enqueue_special_call in csrc/cfbpe.cu runs them.
#include "sim_harness.cpp"

template <typename T> inline T atomicAnd(T* p, T v) { T o = *p; *p = o & v; return o; }

#include "../../cyberfabric-core_b200/csrc/specials.cuh"

struct SimSpecials { std::vector<uint32_t> words; };

extern "C" {

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

// cfbpe_encode_batch_special on host memory; out_bad[2]; *n_stretches_out: the stretches of the ordinary pass (n_prompts when
// the call took the fast path)
__attribute__((visibility("default"))) int sim_encode_batch_special(void* const* vocabs, void* const* specials, uint32_t n_vocabs,
                                                                    const uint8_t* const* modes, uint32_t n_prompts, const uint8_t* bytes,
                                                                    const uint64_t* offsets, const uint8_t* vocab_ids, uint32_t* out_ids,
                                                                    uint64_t out_cap, uint64_t* out_offsets, uint32_t* out_counts,
                                                                    uint32_t max_prompts, uint32_t* out_bad, uint64_t* n_stretches_out) {
    const uint64_t total = offsets[n_prompts];
    std::vector<uint8_t> padded(bytes, bytes + total); padded.resize(total + 64);
    BatchView b{padded.data(), offsets, vocab_ids, n_prompts, total};
    VocabSet vs{};
    for (uint32_t i = 0; i < n_vocabs && i < kMaxVocabs; ++i) {
        SimVocab* v = static_cast<SimVocab*>(vocabs[i]);
        vs.v[i] = make_view(v->blob.data(), v->hdr);
    }
    vs.loaded_mask = n_vocabs >= 32 ? 0xFFFFFFFFu : ((1u << n_vocabs) - 1u);
    const uint64_t mp = max_prompts;
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
        enqueue_special_scan(b, sp, ws.w, sw, 0);
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
        enqueue_encode(b, vs, uc_tables(), ws.w, out_ids, out_cap, out_offsets, out_counts, 4u, 0, 0, 0, 0, 0, 0, prof);
        n_tokens = ws.st.n_tokens;
    } else {
        enqueue_encode_special(b, sp, vs, uc_tables(), ws.w, sw, static_cast<uint32_t>(n_str), ord_ids.data(), total + 1, ord_offsets.data(), ord_counts.data(),
                               out_ids, out_cap, out_offsets, out_counts, 4u, 0, 0, 0, 0, 0, 0, prof);
        n_tokens = ss.fin.n_tokens;
    }
    if (const int rc = status_error(ws.st).code) return rc;
    if (out_ids && n_tokens > out_cap) { out_offsets[n_prompts] = n_tokens; return CFBPE_ENOSPC; }
    return 0;
}

// the decode path with the vocabularies' special tables
__attribute__((visibility("default"))) int sim_decode_batch_special(void* const* vocabs, void* const* specials, uint32_t n_vocabs, uint32_t n_seqs,
                                                                    const uint32_t* ids, const uint64_t* id_offsets, const uint8_t* vocab_ids,
                                                                    uint8_t* out, uint64_t out_cap, uint64_t* out_offsets) {
    VocabSet vs{};
    SpecialSet sp{};
    for (uint32_t i = 0; i < n_vocabs && i < kMaxVocabs; ++i) {
        SimVocab* v = static_cast<SimVocab*>(vocabs[i]);
        vs.v[i] = make_view(v->blob.data(), v->hdr);
        const SimSpecials* t = static_cast<const SimSpecials*>(specials[i]);
        if (t) sp.v[i] = make_special_view(t->words.data(), t->words);
    }
    const uint64_t n_ids = id_offsets[n_seqs];
    DecodeView d{ids, id_offsets, vocab_ids, n_seqs, n_ids};
    const uint32_t n_tiles = static_cast<uint32_t>((n_ids + kDecodeTile - 1) / kDecodeTile);
    std::vector<uint32_t> lens(n_ids + 1), sums(n_tiles + 1);
    std::vector<uint64_t> base(n_tiles + 1);
    DeviceStatus st{};
    if (n_tiles) cusim::launch(n_tiles, 256, [&] { decode_len_kernel(d, vs, lens.data(), sums.data(), &st, sp); });
    cusim::launch(1u, n_tiles ? 1024u : 32u, [&] { tile_scan_kernel(sums.data(), n_tiles, base.data(), &st, nullptr); });
    if (st.bad_utf8) return CFBPE_EINVAL;
    if (n_tiles) cusim::launch(n_tiles, 256, [&] { decode_copy_kernel(d, vs, lens.data(), base.data(), out, out_cap, sp); });
    cusim::launch(static_cast<unsigned>((static_cast<uint64_t>(n_seqs) + 1 + 255) / 256), 256, [&] { decode_offsets_kernel(d, lens.data(), base.data(), out_offsets, &st); });
    return st.tok_end > out_cap ? CFBPE_ENOSPC : 0;
}

}  // extern "C"
