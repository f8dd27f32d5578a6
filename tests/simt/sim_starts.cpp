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
    SimWorkspace ws(total);
    int* prof = nullptr;
    enqueue_encode(b, vs, uc_tables(), ws.w, out_ids, out_cap, out_offsets, out_counts, 4u, 0, 0, 0, 0, 0, 0, prof, nullptr, out_starts);
    if (const int rc = status_error(ws.st).code) return rc;
    if (ws.st.n_tokens > out_cap) { out_offsets[n_prompts] = ws.st.n_tokens; return CFBPE_ENOSPC; }
    return 0;
}

}  // extern "C"
