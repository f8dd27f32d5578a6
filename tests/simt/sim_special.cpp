// sim_special.cpp -- the special-token path (csrc/specials.h, csrc/specials.cuh) on the CPU SIMT emulator.
// TEST INFRASTRUCTURE: built by tests/simt/build_special.py into tests/simt/_build/libcfbpe_sim_special.so, next to
// everything sim_harness.cpp exports.  The host control flow mirrors run_lane_special in csrc/cfbpe.cu: scan, then the ordinary
// path on the prompts as they are (no kept match) or on the stretches followed by the splice.
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

static SpecialSet sim_special_set(void* const* specials, uint32_t n_vocabs, const uint8_t* const* modes, bool* scan) {
    SpecialSet sp{};
    *scan = false;
    for (uint32_t v = 0; v < n_vocabs && v < kMaxVocabs; ++v) {
        const SimSpecials* t = static_cast<const SimSpecials*>(specials[v]);
        if (!t || t->words.empty()) continue;
        const uint8_t* m = modes ? modes[v] : nullptr;
        if (m) {
            bool looks = false;
            for (uint32_t k = 0; k < t->words[0]; ++k) looks = looks || m[k] != kSpOrdinary;
            if (!looks) continue;
        }
        sp.v[v] = make_special_view(t->words.data(), t->words);
        sp.modes[v] = m;
        for (uint32_t j = 0; j < 8; ++j) sp.first_bytes[j] |= t->words[kSpHeaderWords + j];
        *scan = true;
    }
    return sp;
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
    const uint64_t nw = n_flag_words(total);
    const uint32_t nt = n_scan_tiles(total);
    const uint64_t mp = max_prompts;
    std::vector<uint32_t> piece_bits(nw + 2), tok_bits(nw + 2), ids(total + 1, 0xDEADBEEF), rk(total + 1), nx(total + 1), pv(total + 1);
    std::vector<uint32_t> tile_counts(nt + 1);
    std::vector<uint64_t> tile_base(nt + 1);
    std::vector<LongPiece> ll(total / 32 + 1);
    DeviceStatus st{};
    std::vector<SplitFix> fix(total / 16 + 2);
    std::vector<uint64_t> miss[3];
    MissLists ml;
    for (uint32_t c = 0; c < 3; ++c) {
        miss[c].resize(miss_list_words(total, c, 1));
        ml.list[c] = miss[c].data();
        ml.cap[c] = static_cast<uint32_t>(miss[c].size());
    }
    std::vector<uint32_t> pstart(nw + 2), bprompt((total >> kPromptBlockShift) + 2);
    std::vector<uint32_t> by_piece(total + 1, 0xDEADBEEF), extras(total + 1, 0xDEADBEEF), tile_pieces((total >> 11) + 2);
    std::vector<uint64_t> piece_base((total >> 11) + 2);
    Workspace w{piece_bits.data(), tok_bits.data(), ids.data(), LongScratch{rk.data(), nx.data(), pv.data()},
                ll.data(), static_cast<uint32_t>(ll.size()), tile_counts.data(), tile_base.data(), &st, ml, fix.data(), static_cast<uint32_t>(fix.size()),
                DenseIds{by_piece.data(), extras.data(), static_cast<uint32_t>(extras.size()), tile_pieces.data(), piece_base.data()},
                pstart.data(), bprompt.data()};
    std::vector<uint32_t> kept_n(mp + 1), st_id(mp + 1), ord_ids(total + 1), ord_counts(mp + 1);
    std::vector<uint64_t> kept_base(mp + 1), st_off(mp + 2), st_base(mp + 1), ord_offsets(mp + 2);
    std::vector<uint8_t> st_vocab(mp + 1);
    SpecialStatus ss{};
    const SpecialWork sw{kept_n.data(), kept_base.data(), st_off.data(), st_vocab.data(), st_id.data(), st_base.data(), &ss};
    bool scan = false;
    const SpecialSet sp = sim_special_set(specials, n_vocabs, modes, &scan);
    uint64_t n_str = n_prompts;
    if (scan) {
        enqueue_special_scan(b, sp, w, sw, 0);
        if (ss.bad_inv) {
            const unsigned long long key = ~ss.bad_inv;
            if (out_bad) { out_bad[0] = ss.bad_prompt; out_bad[1] = static_cast<uint32_t>(key & 0xFFFu); }
            return CFBPE_EBADMSG;
        }
        n_str = n_prompts + 2 * ss.kept.n_tokens;
        if (n_str > max_prompts) return CFBPE_EINVAL;
    }
    if (n_stretches_out) *n_stretches_out = n_str;
    int* prof = nullptr;
    uint64_t n_tokens;
    if (n_str == n_prompts) {
        enqueue_encode(b, vs, uc_tables(), w, out_ids, out_cap, out_offsets, out_counts, 4u, 0, 0, 0, 0, 0, 0, prof);
        n_tokens = st.n_tokens;
    } else {
        enqueue_encode_special(b, sp, vs, uc_tables(), w, sw, static_cast<uint32_t>(n_str), ord_ids.data(), total + 1, ord_offsets.data(), ord_counts.data(),
                               out_ids, out_cap, out_offsets, out_counts, 4u, 0, 0, 0, 0, 0, 0, prof);
        n_tokens = ss.fin.n_tokens;
    }
    if (st.bad_utf8) return CFBPE_EILSEQ;
    if (st.long_overflow || st.miss_overflow) return CFBPE_EIO;
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
