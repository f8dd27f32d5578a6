// sim_chunk.cpp -- chunking (chunk_scan / chunk_emit of csrc/bpe_kernels.cuh) on the CPU SIMT emulator.
// TEST INFRASTRUCTURE: built by tests/simt/build_chunk.py into tests/simt/_build/libcfbpe_sim_chunk.so, next to everything
// sim_harness.cpp exports.  The whole path runs through enqueue_encode of csrc/pipeline.cuh, as a one-shot call does.
#include "sim_harness.cpp"

extern "C" {

// cfbpe_chunk_batch on host memory (one pass, as run_lane without pipelining): the ids and starts go to scratch buffers of one
// entry a byte, as they go to the lane's buffers.  device_form = 0: the spans stage in the workspace's ids_by_pos / dense.by_piece
// and are copied out when they fit, as a host call does; 1: they go straight to out_spans (pairs, chunks at or past chunk_cap not
// written), as cfbpe_chunk_batch_device does.  out_counts may be NULL.
__attribute__((visibility("default"))) int sim_chunk_batch(void* const* vocabs, uint32_t n_vocabs, uint32_t n_prompts, const uint8_t* bytes,
                                                           const uint64_t* offsets, const uint8_t* vocab_ids, uint32_t chunk_tokens,
                                                           uint32_t overlap_tokens, uint32_t* out_spans, uint64_t chunk_cap,
                                                           uint64_t* out_chunk_offsets, uint32_t* out_counts, int device_form) {
    if (chunk_args_error(chunk_tokens, overlap_tokens, out_spans, out_chunk_offsets)) return CFBPE_EINVAL;
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
    std::vector<uint32_t> ids(total + 1, 0xDEADBEEF), starts(total + 1, 0xDEADBEEF);
    std::vector<uint64_t> offs(static_cast<uint64_t>(n_prompts) + 1);
    std::vector<uint32_t> counts(static_cast<uint64_t>(n_prompts) + 1);
    const uint32_t step = chunk_tokens - overlap_tokens;
    const ChunkView cv = device_form ? ChunkView{chunk_tokens, step, out_chunk_offsets, nullptr, out_spans, out_spans + 1, 2u, chunk_cap}
                                     : ChunkView{chunk_tokens, step, out_chunk_offsets, nullptr, ws.w.ids_by_pos, ws.w.dense.by_piece, 1u, UINT64_MAX};
    int* prof = nullptr;
    enqueue_encode(b, vs, uc_tables(), ws.w, ids.data(), total + 1, offs.data(), counts.data(), 4u, 0, 0, 0, 0, 0, 0, prof, nullptr, starts.data(),
                   nullptr, &cv);
    if (const int rc = status_error(ws.st).code) return rc;
    if (out_counts) std::copy(counts.begin(), counts.begin() + n_prompts, out_counts);
    if (ws.st.chunk_end != out_chunk_offsets[n_prompts] || ws.st.n_chunks != ws.st.chunk_end) return CFBPE_EIO;
    if (ws.st.chunk_end > chunk_cap) return CFBPE_ENOSPC;
    if (!device_form)
        for (uint64_t q = 0; q < ws.st.chunk_end; ++q) { out_spans[2 * q] = ws.w.ids_by_pos[q]; out_spans[2 * q + 1] = ws.w.dense.by_piece[q]; }
    return 0;
}

}  // extern "C"
