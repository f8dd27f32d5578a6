// sim_truncate.cpp -- truncation to token budgets (truncate / truncate_long of csrc/bpe_kernels.cuh) on the CPU SIMT emulator.
// TEST INFRASTRUCTURE: built by tests/simt/build_truncate.py into tests/simt/_build/libcfbpe_sim_truncate.so, next to everything
// sim_harness.cpp exports.  The whole path runs through enqueue_encode of csrc/pipeline.cuh, as a one-shot host call does.
#include "sim_harness.cpp"

extern "C" {

// cfbpe_truncate_batch on host memory (one pass, as run_lane without pipelining): the ids go to a scratch buffer of one id a
// byte, as they go to the lane's buffer; out_counts may be NULL
__attribute__((visibility("default"))) int sim_truncate_batch(void* const* vocabs, uint32_t n_vocabs, uint32_t n_prompts,
                                                              const uint8_t* bytes, const uint64_t* offsets, const uint8_t* vocab_ids,
                                                              const uint32_t* budgets, uint32_t mode, uint32_t* out_cut, uint32_t* out_kept,
                                                              uint32_t* out_counts) {
    if (truncate_args_error(budgets, mode, out_cut, out_kept)) return CFBPE_EINVAL;
    const uint64_t total = offsets[n_prompts];
    std::vector<uint8_t> padded(bytes, bytes + total); padded.resize(total + 64);
    BatchView b{padded.data(), offsets, vocab_ids, n_prompts, total};
    VocabSet vs{};
    for (uint32_t i = 0; i < n_vocabs && i < kMaxVocabs; ++i) {
        SimVocab* v = static_cast<SimVocab*>(vocabs[i]);
        vs.v[i] = make_view(v->blob.data(), v->hdr);
    }
    for (uint32_t i = n_vocabs; i < kMaxVocabs && n_vocabs; ++i) vs.v[i] = vs.v[0];   // (as the library: unloaded slots alias a loaded one)
    vs.loaded_mask = n_vocabs >= 32 ? 0xFFFFFFFFu : ((1u << n_vocabs) - 1u);
    SimWorkspace ws(total);
    std::vector<uint32_t> ids(total + 1, 0xDEADBEEF);
    std::vector<uint64_t> offs(static_cast<uint64_t>(n_prompts) + 1);
    std::vector<uint32_t> counts(static_cast<uint64_t>(n_prompts) + 1);
    const TruncateView tv{budgets, mode == CFBPE_TRUNCATE_TAIL ? 1u : 0u, out_cut, out_kept};
    int* prof = nullptr;
    enqueue_encode(b, vs, uc_tables(), ws.w, ids.data(), total + 1, offs.data(), counts.data(), 4u, 0, 0, 0, 0, 0, 0, prof, nullptr, nullptr, &tv);
    if (const int rc = status_error(ws.st).code) return rc;
    if (out_counts) std::copy(counts.begin(), counts.begin() + n_prompts, out_counts);
    return 0;
}

}  // extern "C"
