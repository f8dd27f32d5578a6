// sim_starts.cpp -- encode with token starts (starts_len / starts_emit of csrc/bpe_kernels.cuh) on the CPU SIMT emulator.
// TEST INFRASTRUCTURE: built by tests/simt/build_starts.py into tests/simt/_build/libcfbpe_sim_starts.so, next to everything
// sim_harness.cpp exports.  The whole path runs through enqueue_encode of csrc/pipeline.cuh, as a one-shot host call does.
#include "sim_harness.cpp"

extern "C" {

// cfbpe_encode_batch_starts on host memory (one pass, as run_lane without pipelining); out_starts has room for out_cap entries
__attribute__((visibility("default"))) int sim_encode_batch_starts(void* const* vocabs, uint32_t n_vocabs, uint32_t n_prompts,
                                                                   const uint8_t* bytes, const uint64_t* offsets, const uint8_t* vocab_ids,
                                                                   uint32_t* out_ids, uint32_t* out_starts, uint64_t out_cap,
                                                                   uint64_t* out_offsets, uint32_t* out_counts) {
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
    int* prof = nullptr;
    enqueue_encode(b, vs, uc_tables(), w, out_ids, out_cap, out_offsets, out_counts, 4u, 0, 0, 0, 0, 0, 0, prof, nullptr, out_starts);
    if (st.bad_utf8) return CFBPE_EILSEQ;
    if (st.long_overflow || st.miss_overflow) return CFBPE_EIO;
    if (st.n_tokens > out_cap) { out_offsets[n_prompts] = st.n_tokens; return CFBPE_ENOSPC; }
    return 0;
}

}  // extern "C"
