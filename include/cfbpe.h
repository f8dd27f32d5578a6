/*
 * cfbpe.h -- C ABI of the H100-native batched BPE tokenizer (libcfbpe.so).
 *
 * This is the drop-in boundary for cyberfabric-core's LLM Gateway tokenizer /
 * usage-meter worker.  The reference tree has no tokenizer code to replace
 * (modules/llm-gateway/README.md:51-52 lists the implementation crate and plugins as
 * "planned"; SURVEY.md F1), so each entry point cites the *spec'd consumer* it serves and
 * the ModKit convention it follows instead of a replaced function:
 *
 *   cfbpe_create / cfbpe_destroy   plugin Module::init / stop: one-time device context,
 *                                  tables and staging buffers, created where a ModKit plugin
 *                                  registers its scoped client
 *                                  (modules/system/tenant-resolver/plugins/static-tr-plugin/src/module.rs:43-88).
 *   cfbpe_vocab_load / _export / _import
 *                                  the model-registry vocab loader that does not exist yet:
 *                                  `Model` has no tokenizer field
 *                                  (modules/model-registry/docs/PRD.md:196-209); rank-file format
 *                                  per tiktoken/load.py:160-172.  export/import move the packed
 *                                  device tables so one rank parses and the host layer broadcasts
 *                                  them (NCCL) to the other GPUs of the box.
 *   cfbpe_encode_batch             `TokenizerPluginClient::encode_batch` (llm-gateway::tokenizer):
 *                                  token ids for a packed multi-tenant prompt buffer.
 *   cfbpe_count_batch              `llm-gateway::usage::count_tokens`: feeds
 *                                  Usage.input_tokens (modules/llm-gateway/llm-gateway-sdk/schemas/core/usage.v1.schema.json:8-12)
 *                                  and check_budget / report_usage (modules/llm-gateway/docs/DESIGN.md:833-855).
 *   cfbpe_encode_batch_device      same path with inputs/outputs already resident in HBM
 *                                  (for callers that keep token ids on the GPU).
 *
 * Conventions (SURVEY.md section 8(b)): 0 = ok, negative errno-style code = error; the caller
 * owns every buffer it passes and the library never retains a caller pointer past return;
 * the library owns device memory, pinned staging and streams; nothing throws across the
 * ABI; entry points taking a ctx may be called from several host threads: a context holds
 * cfbpe_config.n_workspaces independent call lanes per device (calls wait only when all are
 * busy; vocabulary loads exclude running calls), the last error is kept per thread, and every
 * entry point leaves the caller's current CUDA device as it found it.  There is NO CPU fallback: cfbpe_create fails with
 * CFBPE_ENODEV when no sm_90 device is present.
 *
 * Results are bit-exact with tiktoken 0.12.0 CoreBPE.encode_ordinary for the same rank
 * file and pattern (see oracle/ and tests/).
 */
#ifndef CFBPE_H
#define CFBPE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define CFBPE_API __attribute__((visibility("default")))
#else
#define CFBPE_API
#endif

#define CFBPE_ABI_VERSION 1u

/* error codes (negative errno values) */
#define CFBPE_OK 0
#define CFBPE_ENOENT (-2)    /* unknown vocab id */
#define CFBPE_EIO (-5)       /* CUDA runtime failure; see cfbpe_last_error */
#define CFBPE_ENOMEM (-12)
#define CFBPE_ENODEV (-19)   /* no usable sm_90 device */
#define CFBPE_EINVAL (-22)   /* bad argument: null pointer, non-monotonic offsets, oversize batch, bad rank file */
#define CFBPE_ENOSPC (-28)   /* out_cap too small; required id count is in out_offsets[n_prompts] */
#define CFBPE_EILSEQ (-84)   /* a prompt holds malformed UTF-8 (tiktoken only accepts valid text) */
#define CFBPE_EBADMSG (-74)  /* a prompt spells a special token this call disallows */

/* what an occurrence of a registered special token means in one call (cfbpe_encode_batch_special) */
#define CFBPE_SPECIAL_ORDINARY 0u   /* its text is ordinary text */
#define CFBPE_SPECIAL_ALLOW 1u      /* an occurrence becomes its id */
#define CFBPE_SPECIAL_DISALLOW 2u   /* an occurrence anywhere fails the call */
#define CFBPE_MAX_SPECIALS 4096u    /* special tokens per vocabulary */
#define CFBPE_MAX_SPECIAL_LEN 64u   /* bytes per special token */

/* rank-file formats */
#define CFBPE_FORMAT_TIKTOKEN 0u     /* "<base64 token> <rank>\n" lines */
#define CFBPE_FORMAT_TEKKEN_JSON 1u  /* mistral_common tekken_*.json */

/* pre-tokenizer patterns */
#define CFBPE_PATTERN_CL100K 0u
#define CFBPE_PATTERN_O200K 1u
#define CFBPE_PATTERN_LLAMA3 2u
#define CFBPE_PATTERN_TEKKEN 3u
#define CFBPE_PATTERN_COUNT 4u

#define CFBPE_MAX_VOCABS 8u

typedef struct cfbpe_ctx cfbpe_ctx; /* opaque */

#define CFBPE_MAX_DEVICES 8

typedef struct cfbpe_config {
    uint32_t struct_size;     /* sizeof(cfbpe_config), for forward compatibility: a caller built against the five-field struct of
                                 ABI version 1 (24 bytes) still works, and gets one device and one workspace */
    int32_t device;           /* CUDA device ordinal (used when n_devices == 0) */
    uint64_t max_batch_bytes; /* largest packed prompt buffer one DEVICE takes in one call (0 = 256 MiB) */
    uint32_t max_prompts;     /* largest n_prompts of one call (0 = 1 Mi) */
    uint32_t flags;           /* reserved, 0 */
    /* SURVEY.md section 8(b): cfbpe_create(cfg: devices[], n_devices, ...) */
    int32_t devices[CFBPE_MAX_DEVICES]; /* CUDA ordinals of a multi-device context */
    uint32_t n_devices;       /* 0 = single device (`device`); > 1: the packed tables are broadcast with NCCL (libnccl.so.2 is
                                 dlopen'ed; without it cfbpe_create fails with CFBPE_EIO) and a host batch is spread over the
                                 devices -- its sub-batches round-robin, token ranks chained over NVLink peer memory, when
                                 every device can hold the whole batch (<= max_batch_bytes); else one contiguous shard of
                                 whole prompts a device, the shard totals gathered with NCCL */
    uint32_t n_workspaces;    /* independent workspaces per device (0 = 1, at most 16): that many calls run concurrently on the
                                 context; each costs ~33 bytes of device memory per byte of max_batch_bytes */
} cfbpe_config;

typedef struct cfbpe_vocab_info {
    uint32_t n_ranks;
    uint32_t pattern_id;
    uint32_t max_token_len;
    uint32_t n_pair_entries;  /* (left,right)->merged entries in the all-splits pair table */
    uint64_t table_bytes;     /* size of the packed device tables (= export size) */
} cfbpe_vocab_info;

/* per-call device timings, filled when profiling is on (cfbpe_profile_enable) */
#define CFBPE_NUM_KERNELS 10
typedef struct cfbpe_profile {
    float kernel_ms[CFBPE_NUM_KERNELS]; /* 0 pretok_split, 1 bpe_encode, 2 bpe_long, 3 flag_count, 4 tile_scan, 5 emit_compact (+ offsets), 6 bpe_list, 7 long_scan, 8 bpe_merge, 9 reserved */
    uint32_t kernel_launches[CFBPE_NUM_KERNELS];
    float h2d_ms, d2h_ms, total_ms;
    uint64_t n_tokens, n_bytes, n_long_pieces;
    uint64_t n_long_bytes, n_long_tokens; /* bytes in / ids out of the long-piece kernels */
    uint64_t n_miss_pieces;               /* short pieces that were not one token (merged by bpe_merge) */
    uint64_t n_list_pieces, n_list_parts; /* big pieces whose list phase ran in bpe_list, and their parts when it began */
    uint64_t n_extra_tokens;              /* tokens of the merged short pieces (the dense `extras` list of bpe_merge) */
} cfbpe_profile;

CFBPE_API int cfbpe_abi_version(void);
/* sha256 (hex, first 16 chars) of the sources this binary was built from; lets the host layer refuse a stale build */
CFBPE_API const char *cfbpe_build_id(void);

CFBPE_API int cfbpe_create(const cfbpe_config *cfg, cfbpe_ctx **out);
CFBPE_API void cfbpe_destroy(cfbpe_ctx *ctx);
/* NUL-terminated description of the last failure of the CALLING THREAD (valid until its next call): entry points run
 * concurrently on one context, so the message is kept per thread, not per context */
CFBPE_API const char *cfbpe_last_error(const cfbpe_ctx *ctx);

/* Parse a rank file, build the lookup tables on the host and upload them.
 * max_ranks: keep only ranks < max_ranks (0 = all). */
CFBPE_API int cfbpe_vocab_load(cfbpe_ctx *ctx, uint32_t vocab_id, const uint8_t *ranks_file, size_t len,
                     uint32_t format, uint32_t pattern_id, uint32_t max_ranks);
CFBPE_API int cfbpe_vocab_get_info(const cfbpe_ctx *ctx, uint32_t vocab_id, cfbpe_vocab_info *out);
/* Copy the packed tables out (size query: buf = NULL, cap = 0) / install packed tables
 * produced by cfbpe_vocab_export on another rank. */
CFBPE_API int cfbpe_vocab_export(const cfbpe_ctx *ctx, uint32_t vocab_id, uint8_t *buf, uint64_t cap, uint64_t *size);
CFBPE_API int cfbpe_vocab_import(cfbpe_ctx *ctx, uint32_t vocab_id, const uint8_t *buf, uint64_t size);

/* Encode n_prompts prompts.  bytes/offsets: packed UTF-8, prompt i = bytes[offsets[i] .. offsets[i+1]),
 * offsets[0] must be 0.  vocab_ids: per-prompt vocab id or NULL (all vocab 0).
 * out_ids: room for out_cap ids; out_offsets: n_prompts+1; out_counts: n_prompts (may be NULL).
 * Host pointers; pinned buffers from cfbpe_host_alloc are DMA'd directly, others are staged. */
CFBPE_API int cfbpe_encode_batch(cfbpe_ctx *ctx, uint32_t n_prompts, const uint8_t *bytes, const uint64_t *offsets,
                       const uint8_t *vocab_ids, uint32_t *out_ids, uint64_t out_cap, uint64_t *out_offsets,
                       uint32_t *out_counts);
/* cfbpe_encode_batch plus the byte offset of every token within its prompt: out_starts[k] (room for out_cap entries, as out_ids)
 * is where the k-th id of the stream starts in its prompt, so token k of prompt i covers
 * bytes[offsets[i] + out_starts[k] .. offsets[i] + end), end = out_starts[k + 1], or the prompt's length for its last token.
 * A prompt's first token starts at 0 and the starts strictly increase within a prompt.  Ids, offsets and counts are those of
 * cfbpe_encode_batch on the same inputs.  out_ids and out_starts are required (NULL: CFBPE_EINVAL); other arguments and errors
 * as cfbpe_encode_batch (CFBPE_ENOSPC: out_offsets[n_prompts] = ids needed).  Costs: 4 bytes of device memory per byte of
 * max_batch_bytes on each lane that runs such a call, allocated on its first one (CFBPE_ENOMEM if that fails), and three small
 * kernels after the ids (the byte lengths of the ids, scanned). */
CFBPE_API int cfbpe_encode_batch_starts(cfbpe_ctx *ctx, uint32_t n_prompts, const uint8_t *bytes, const uint64_t *offsets,
                                        const uint8_t *vocab_ids, uint32_t *out_ids, uint32_t *out_starts, uint64_t out_cap,
                                        uint64_t *out_offsets, uint32_t *out_counts);
/* what a unit start counts (cfbpe_encode_batch_char_starts); byte starts are cfbpe_encode_batch_starts */
#define CFBPE_UNIT_CODEPOINT 0u   /* Unicode code points: Python str indices, tiktoken's decode_with_offsets */
#define CFBPE_UNIT_UTF16 1u       /* UTF-16 code units (a code point >= U+10000 counts 2): JavaScript, Java and C# string indices */
/* cfbpe_encode_batch_starts with each token's start counted in `unit` instead of bytes.  For prompt p with bytes b and token k's
 * byte start x_k (cfbpe_encode_batch_starts), F(x) = the largest character start <= x (the snap of CFBPE_TRUNCATE_HEAD and of the
 * chunk spans) and U(s) = the units of the byte string s:
 *   out_starts[k] = U(b[0 .. F(x_k))): the unit index of the character that holds the token's first byte.  For
 *                   CFBPE_UNIT_CODEPOINT this is tiktoken 0.12.0 decode_with_offsets(ids)[1].
 *   out_lens[p]   = U(b) (n_prompts entries, may be NULL): closes the last token's span without walking the text.
 * Within a prompt the starts never decrease and the first is 0.  A character split into several byte tokens gives them all the
 * same start, so a span built from consecutive starts ([out_starts[k], out_starts[k + 1]), the last one closed by out_lens[p])
 * can be EMPTY; the spans of a prompt still tile [0, out_lens[p]).  Ids, offsets and counts are those of cfbpe_encode_batch on the
 * same inputs.  Errors: as cfbpe_encode_batch_starts (CFBPE_ENOSPC: out_offsets[n_prompts] = ids needed); an unknown unit, a NULL
 * out_ids or a NULL out_starts is CFBPE_EINVAL.  Costs: the lane's token-start buffer (as cfbpe_encode_batch_starts), 4 bytes
 * per prompt of max_prompts for the lengths on each lane that runs a host call with out_lens (allocated on its first one,
 * CFBPE_ENOMEM if that fails), and three small kernels after the byte starts: every token's units from the vocabulary's token
 * bytes, scanned within each prompt. */
CFBPE_API int cfbpe_encode_batch_char_starts(cfbpe_ctx *ctx, uint32_t n_prompts, const uint8_t *bytes, const uint64_t *offsets,
                                             const uint8_t *vocab_ids, uint32_t unit, uint32_t *out_ids, uint32_t *out_starts,
                                             uint64_t out_cap, uint64_t *out_offsets, uint32_t *out_counts, uint32_t *out_lens);
/* Token counts only (no id stream leaves the device). */
CFBPE_API int cfbpe_count_batch(cfbpe_ctx *ctx, uint32_t n_prompts, const uint8_t *bytes, const uint64_t *offsets,
                      const uint8_t *vocab_ids, uint32_t *out_counts);

/* which tokens a truncation keeps (cfbpe_truncate_batch) */
#define CFBPE_TRUNCATE_HEAD 0u   /* the first ones: a long document or retrieved context */
#define CFBPE_TRUNCATE_TAIL 1u   /* the last ones: a chat history */
/* Cut every prompt to a token budget: where its text must be cut so that it keeps budgets[i] tokens, as one byte position.
 * For prompt i with bytes b, ids t_0 .. t_{c-1} (cfbpe_encode_batch) and k = min(budgets[i], c):
 *   CFBPE_TRUNCATE_HEAD: x = the byte length of t_0 .. t_{k-1}; out_cut[i] = the largest character start <= x, and the kept text
 *                        is b[0 .. out_cut[i]).
 *   CFBPE_TRUNCATE_TAIL: x = len(b) - the byte length of t_{c-k} .. t_{c-1}; out_cut[i] = the smallest character start >= x, or
 *                        len(b), and the kept text is b[out_cut[i] .. len(b)).
 * A byte-level token may end inside a UTF-8 character; the cut always moves to a character boundary, so the kept text is valid
 * UTF-8 (a caller who needs the token boundary itself has cfbpe_encode_batch_starts).  out_kept[i] = the tokens of the encoding
 * that lie wholly inside the kept text: k, or fewer when the cut moved.  out_counts[i] = c, as cfbpe_count_batch (may be NULL).
 * A budget of 0 keeps nothing (head: cut 0, tail: cut len(b)); a budget >= c keeps the whole prompt.  Cuts and kept counts are
 * per prompt and relative to it.
 * The boundaries are those of the encoding of the WHOLE prompt, as decode(ids[:N]) of tiktoken or the id truncation of Hugging
 * Face tokenizers: BPE is not prefix-stable, so encoding the kept text again may give other ids (and another count).
 * mode: a CFBPE_TRUNCATE_* value.  budgets, out_cut, out_kept: n_prompts entries each, required.  Errors: an unknown mode or a
 * NULL budgets / out_cut / out_kept is CFBPE_EINVAL; the rest as cfbpe_count_batch.  The ids stay on the device: the cut is a
 * sum of token lengths over the nearer end of each prompt's ids, at most min(k, c - k) of them, and a prompt with c <= budget reads
 * none.  Costs: 12 bytes of device memory per prompt of max_prompts on each lane that runs a host call of it, allocated on its
 * first one (CFBPE_ENOMEM if that fails). */
CFBPE_API int cfbpe_truncate_batch(cfbpe_ctx *ctx, uint32_t n_prompts, const uint8_t *bytes, const uint64_t *offsets,
                                   const uint8_t *vocab_ids, const uint32_t *budgets, uint32_t mode, uint32_t *out_cut,
                                   uint32_t *out_kept, uint32_t *out_counts);

/* Cut every prompt into chunks of at most chunk_tokens = N tokens that overlap by overlap_tokens = S (N >= 1, S < N; step
 * s = N - S): the chunk_size / chunk_overlap windows of a RAG splitter or of an embedding endpoint's long inputs.  For prompt i with
 * bytes b, ids t_0 .. t_{c-1} (cfbpe_encode_batch) and token starts x_j (cfbpe_encode_batch_starts; x_c = len(b)):
 *   chunks: 0 if c = 0, 1 if c <= N, else 1 + ceil((c - N) / s) -- LangChain's split_text_on_tokens: windows start at token 0, s,
 *           2s, ... and stop at the first that reaches the last token;
 *   chunk k covers tokens [a, e), a = k x s, e = min(a + N, c), and its text is b[F(a) .. F(e)): F(j) = the largest character
 *           start <= x_j (the snap of CFBPE_TRUNCATE_HEAD), F(c) = len(b).
 * Both ends take the same snap, so every chunk is valid UTF-8; with S = 0 the chunks tile the prompt (each ends where the next
 * begins, the first begins at 0, the last ends at len(b)); chunk 0 ends where cfbpe_truncate_batch(HEAD, budget N) cuts.  A chunk
 * is empty only when N is smaller than the number of byte tokens one character was split into (so N <= 3).  The boundaries are
 * those of the WHOLE prompt's encoding, as for truncation: encoding a chunk again may give other ids.
 * out_spans: 2 entries a chunk (begin, end; relative to the prompt), room for chunk_cap chunks; prompt i's chunks are
 * out_chunk_offsets[i] .. out_chunk_offsets[i + 1] (n_prompts + 1 entries).  CFBPE_ENOSPC when the chunks exceed chunk_cap
 * (out_chunk_offsets[n_prompts] = the chunks needed; no span is written).  Sum over the prompts of the chunk formula with c = the
 * prompt's byte length always fits, because c <= len: a caller can size out_spans once and never retry.  out_counts[i] = c, as
 * cfbpe_count_batch (may be NULL).  Errors: chunk_tokens = 0, overlap_tokens >= chunk_tokens, a NULL out_spans or a NULL
 * out_chunk_offsets is CFBPE_EINVAL; the rest as cfbpe_count_batch.  The ids and starts stay on the device.  Costs: the lane's
 * token-start buffer (4 bytes per byte of max_batch_bytes, as cfbpe_encode_batch_starts) and 8 bytes per prompt of max_prompts
 * for the chunk offsets, allocated on the lane's first such call (CFBPE_ENOMEM if that fails). */
CFBPE_API int cfbpe_chunk_batch(cfbpe_ctx *ctx, uint32_t n_prompts, const uint8_t *bytes, const uint64_t *offsets,
                                const uint8_t *vocab_ids, uint32_t chunk_tokens, uint32_t overlap_tokens,
                                uint32_t *out_spans /* 2 per chunk: begin, end; prompt-relative */, uint64_t chunk_cap,
                                uint64_t *out_chunk_offsets /* n_prompts + 1 */, uint32_t *out_counts /* may be NULL */);

/* Decode (SURVEY.md section 8(f) item 2; tiktoken CoreBPE.decode_bytes): out_bytes = the concatenation of the tokens' bytes.
 * ids: the packed token ids of n_seqs sequences, id_offsets[n_seqs + 1] their boundaries (in ids), vocab_ids[n_seqs] or NULL.
 * out_offsets[n_seqs + 1]: byte boundaries of the decoded sequences in out_bytes.  CFBPE_ENOSPC if out_cap is too small
 * (out_offsets[n_seqs] = bytes needed), CFBPE_EINVAL for an id outside its vocabulary or a batch beyond the context's limits
 * (at most max_batch_bytes ids and max_batch_bytes decoded bytes).  Ids are ranks, or base + rank with an id base set
 * (cfbpe_vocab_set_id_base).  An id past the vocabulary's ranks that is one of its
 * registered special tokens (cfbpe_vocab_set_specials) decodes to that token's bytes.  Host buffers; no reference interface exists for it
 * (the reference ships no tokenizer: SURVEY.md F1). */
CFBPE_API int cfbpe_decode_batch(cfbpe_ctx* ctx, uint32_t n_seqs, const uint32_t* ids, const uint64_t* id_offsets,
                                 const uint8_t* vocab_ids, uint8_t* out_bytes, uint64_t out_cap, uint64_t* out_offsets);

/* Register the special tokens of a vocabulary (tiktoken's special_tokens): token k = bytes[offsets[k] .. offsets[k+1]), id ids[k];
 * offsets has n + 1 entries.  Replaces the vocabulary's earlier set; n = 0 clears it, and so do cfbpe_vocab_load and
 * cfbpe_vocab_import.  Tokens must be valid UTF-8 of 1 .. CFBPE_MAX_SPECIAL_LEN bytes, distinct, with distinct ids (not
 * 0xFFFFFFFF), at most CFBPE_MAX_SPECIALS of them: else CFBPE_EINVAL.  CFBPE_ENOENT for a slot that is not loaded.  The table
 * is copied to every device of the context; it is not part of the exported blob (a multi-process deployment registers the
 * specials on each rank).  Waits for running calls, as a vocabulary load does.  Decode then turns these ids into their bytes
 * (an id below the vocabulary's n_ranks is always the ordinary token; with an id base set, see cfbpe_vocab_set_id_base). */
CFBPE_API int cfbpe_vocab_set_specials(cfbpe_ctx *ctx, uint32_t vocab_id, uint32_t n, const uint8_t *bytes, const uint64_t *offsets,
                                       const uint32_t *ids);

/* Give the ordinary tokens of a vocabulary the ids base + rank (rank 0 .. n_ranks - 1) instead of their ranks: mistral_common's
 * Tekken numbers its ordinary tokens from 1000, after its control tokens (<unk> 0, <s> 1, </s> 2, [INST] 3, ...).  Every id an
 * encode call returns (cfbpe_encode_batch and its _starts, _char_starts, _special, _lossy and _device forms) is then
 * base(v) + rank for its prompt's vocabulary v; a special token's id (cfbpe_encode_batch_special) is written as registered.  Decode
 * takes an id in [base, base + n_ranks) as the ordinary token id - base; any other id must be a registered special token
 * (else CFBPE_EINVAL).  Counts, offsets, starts, truncation and chunks do not depend on the base.
 * The base is 0 until set, and cfbpe_vocab_load and cfbpe_vocab_import reset it to 0.  base + n_ranks must not exceed 0xFFFFFFFF
 * (CFBPE_EINVAL).  With a base above 0, no special token may have an id in [base, base + n_ranks): this call refuses a base that
 * would put a registered special there, and cfbpe_vocab_set_specials refuses such a special (CFBPE_EINVAL); with base 0 the rules
 * of cfbpe_vocab_set_specials are unchanged.  CFBPE_ENOENT for a slot that is not loaded.  The base is copied to every device of
 * the context; it is not part of the exported blob (a multi-process deployment sets it on each rank).  Waits for running calls, as
 * a vocabulary load does.  Costs: a call that returns ids for a vocabulary with a base above 0 runs one more small kernel (a read
 * and a write of every id); other calls run nothing more. */
CFBPE_API int cfbpe_vocab_set_id_base(cfbpe_ctx *ctx, uint32_t vocab_id, uint32_t base);
/* the id base of a loaded vocabulary (cfbpe_vocab_set_id_base): CFBPE_EINVAL for a NULL pointer or a bad slot, CFBPE_ENOENT if not loaded */
CFBPE_API int cfbpe_vocab_get_id_base(const cfbpe_ctx *ctx, uint32_t vocab_id, uint32_t *out);

/* Encode as tiktoken's Encoding.encode(text, allowed_special=..., disallowed_special=...) does, per prompt:
 *  1. if a DISALLOWED special occurs anywhere in the prompt's bytes (inside or across an allowed one too), the call fails with
 *     CFBPE_EBADMSG; out_bad[0] = the lowest such prompt, out_bad[1] = the index of the special at its leftmost occurrence
 *     (the longest one there).  This is checked before anything else: it wins over CFBPE_EILSEQ.
 *  2. from the start, the leftmost position where an ALLOWED special occurs, the longest one there: the text before it is
 *     encoded as ordinary text (as a text of its own: its end is the end of the text for the pre-tokenizer), then the special's
 *     id; repeat after it; the rest is ordinary text.  A match never crosses a prompt boundary.
 *  3. an ORDINARY special is plain text.
 * modes[v]: one CFBPE_SPECIAL_* byte per registered special of vocabulary v, or NULL = all DISALLOWED (tiktoken's default);
 * modes == NULL: NULL for every vocabulary.  out_ids == NULL: counts and offsets only.  out_bad (2 entries) may be NULL.
 * Other arguments and errors as cfbpe_encode_batch.  n_prompts + 2 x (allowed matches) must not exceed the context's
 * max_prompts (CFBPE_EINVAL).  A host call runs as one pass on its lane (not pipelined like cfbpe_encode_batch); a call whose
 * prompts hold no allowed and no disallowed special costs one scan over the bytes beside the ordinary path, and a call for which
 * no vocabulary has a special to look for is the ordinary path. */
CFBPE_API int cfbpe_encode_batch_special(cfbpe_ctx *ctx, uint32_t n_prompts, const uint8_t *bytes, const uint64_t *offsets,
                                         const uint8_t *vocab_ids, const uint8_t *const *modes, uint32_t *out_ids, uint64_t out_cap,
                                         uint64_t *out_offsets, uint32_t *out_counts, uint32_t *out_bad);
/* The same on device-resident buffers (as cfbpe_encode_batch_device; modes and out_bad are HOST memory).  When some vocabulary
 * has a special to look for, the call synchronises `stream` once, after the scan, to learn the number of stretches (and whether
 * a disallowed special occurs); the rest is enqueued asynchronously as in cfbpe_encode_batch_device. */
CFBPE_API int cfbpe_encode_batch_special_device(cfbpe_ctx *ctx, uint32_t n_prompts, const uint8_t *d_bytes, uint64_t total_bytes,
                                                const uint64_t *d_offsets, const uint8_t *d_vocab_ids, const uint8_t *const *modes,
                                                uint32_t *d_out_ids, uint64_t out_cap, uint64_t *d_out_offsets, uint32_t *d_out_counts,
                                                uint64_t *n_tokens, uint32_t *out_bad, void *stream);

/* Same path on device-resident buffers, enqueued on `stream` (a cudaStream_t; NULL = the legacy
 * default stream).  d_bytes must be readable for 32 bytes past total_bytes (the kernels read whole 16-byte
 * groups); the contents of that padding do not matter.  d_out_ids may be NULL (count only).  n_tokens (host, may be NULL) is written
 * after an internal stream sync; with n_tokens == NULL the call is fully asynchronous and
 * d_out_offsets[n_prompts] holds the total.  Then malformed UTF-8 and an out_cap that is too small are reported by
 * cfbpe_device_status only: no other call reports them, whatever it synchronises. */
CFBPE_API int cfbpe_encode_batch_device(cfbpe_ctx *ctx, uint32_t n_prompts, const uint8_t *d_bytes, uint64_t total_bytes,
                              const uint64_t *d_offsets, const uint8_t *d_vocab_ids, uint32_t *d_out_ids,
                              uint64_t out_cap, uint64_t *d_out_offsets, uint32_t *d_out_counts,
                              uint64_t *n_tokens, void *stream);
/* cfbpe_encode_batch_starts on device-resident buffers, as cfbpe_encode_batch_device: the starts go straight to d_out_starts
 * (room for out_cap entries).  d_out_ids and d_out_starts are required (NULL: CFBPE_EINVAL). */
CFBPE_API int cfbpe_encode_batch_starts_device(cfbpe_ctx *ctx, uint32_t n_prompts, const uint8_t *d_bytes, uint64_t total_bytes,
                                               const uint64_t *d_offsets, const uint8_t *d_vocab_ids, uint32_t *d_out_ids,
                                               uint32_t *d_out_starts, uint64_t out_cap, uint64_t *d_out_offsets, uint32_t *d_out_counts,
                                               uint64_t *n_tokens, void *stream);
/* cfbpe_encode_batch_char_starts on device-resident buffers, as cfbpe_encode_batch_starts_device: the unit starts go straight to
 * d_out_starts (room for out_cap entries), the lengths to d_out_lens (n_prompts entries, device memory, may be NULL).  d_out_ids
 * and d_out_starts are required and unit must be a CFBPE_UNIT_* value (else CFBPE_EINVAL).  n_tokens (host, may be NULL) is
 * written after an internal stream sync; with n_tokens == NULL the call is fully asynchronous. */
CFBPE_API int cfbpe_encode_batch_char_starts_device(cfbpe_ctx *ctx, uint32_t n_prompts, const uint8_t *d_bytes, uint64_t total_bytes,
                                                    const uint64_t *d_offsets, const uint8_t *d_vocab_ids, uint32_t unit,
                                                    uint32_t *d_out_ids, uint32_t *d_out_starts, uint64_t out_cap, uint64_t *d_out_offsets,
                                                    uint32_t *d_out_counts, uint32_t *d_out_lens, uint64_t *n_tokens, void *stream);
/* cfbpe_truncate_batch on device-resident buffers, enqueued on `stream` as cfbpe_encode_batch_device (d_bytes readable for 32
 * bytes past total_bytes).  d_budgets, d_out_cut, d_out_kept and d_out_counts (may be NULL) are device memory.  Fully
 * asynchronous: nothing has to come back to the host, and the ids, which never exceed max_batch_bytes, stay in the lane's
 * buffers (no CFBPE_ENOSPC).  Malformed UTF-8 and an unloaded vocabulary are reported by cfbpe_device_status only. */
CFBPE_API int cfbpe_truncate_batch_device(cfbpe_ctx *ctx, uint32_t n_prompts, const uint8_t *d_bytes, uint64_t total_bytes,
                                          const uint64_t *d_offsets, const uint8_t *d_vocab_ids, const uint32_t *d_budgets, uint32_t mode,
                                          uint32_t *d_out_cut, uint32_t *d_out_kept, uint32_t *d_out_counts, void *stream);
/* cfbpe_chunk_batch on device-resident buffers, enqueued on `stream` as cfbpe_encode_batch_device (d_bytes readable for 32 bytes
 * past total_bytes).  d_out_spans (room for chunk_cap chunks), d_out_chunk_offsets and d_out_counts (may be NULL) are device
 * memory.  n_chunks (host, may be NULL) is written after an internal stream sync, and then CFBPE_ENOSPC is returned when the
 * chunks exceed chunk_cap; with n_chunks == NULL the call is fully asynchronous, d_out_chunk_offsets[n_prompts] holds the total,
 * and CFBPE_ENOSPC, malformed UTF-8 and an unloaded vocabulary are reported by cfbpe_device_status only.  Chunks at or past
 * chunk_cap are not written. */
CFBPE_API int cfbpe_chunk_batch_device(cfbpe_ctx *ctx, uint32_t n_prompts, const uint8_t *d_bytes, uint64_t total_bytes,
                                       const uint64_t *d_offsets, const uint8_t *d_vocab_ids, uint32_t chunk_tokens,
                                       uint32_t overlap_tokens, uint32_t *d_out_spans, uint64_t chunk_cap,
                                       uint64_t *d_out_chunk_offsets, uint32_t *d_out_counts, uint64_t *n_chunks, void *stream);
/* Encode as if every prompt had first been decoded with Python's bytes.decode("utf-8", errors="replace") and encoded again as
 * UTF-8.  For prompt p with bytes b and R(b) = b.decode("utf-8", "replace").encode("utf-8"):
 *   ids, offsets, counts  those of cfbpe_encode_batch on R(b) for every prompt: tiktoken 0.12.0
 *                         encode_ordinary(b.decode("utf-8", "replace")).  A prompt of valid UTF-8 gets exactly its
 *                         cfbpe_encode_batch ids.
 *   out_replaced[p]       the number of U+FFFD the decode inserted into prompt p (a U+FFFD that was already in the text does not
 *                         count; 0: the prompt is valid UTF-8).  n_prompts entries, may be NULL.  A strict caller can refuse just
 *                         the prompts with out_replaced[p] > 0.
 * The replacement rule is CPython's, the Unicode Standard's "substitution of maximal subparts" (chapter 3), which
 * String::from_utf8_lossy and the WHATWG decoder follow too: each maximal subpart of an ill-formed sequence becomes one U+FFFD
 * (F0 9F 98 -> 1, ED A0 80 -> 3, C0 AF -> 2, F4 90 80 80 -> 4, F0 9F 98 61 -> U+FFFD "a").  A sequence never spans two prompts:
 * a lead byte that ends prompt i is a subpart of its own, and the continuation bytes that open prompt i + 1 are strays.
 * out_ids == NULL: counts and offsets only.  Other arguments and CFBPE_ENOSPC (out_offsets[n_prompts] = ids needed) as
 * cfbpe_encode_batch.  The call never returns CFBPE_EILSEQ.  The repaired batch is up to 3 times the input: when a device's
 * share of it exceeds max_batch_bytes the call returns CFBPE_EINVAL (the message gives the repaired size) and writes no output.
 * A host call runs as one pass on its lane, or as one contiguous shard of whole prompts a device on a multi-device context (not
 * pipelined, and not spread round-robin like cfbpe_encode_batch).  Costs: a scan over the bytes and one synchronisation before the
 * ordinary path; when some byte is not valid UTF-8, the repaired copy is written first (the ordinary path then runs on it).
 * 12 bytes of device memory per prompt of max_prompts on each lane that runs such a call, allocated on its first one
 * (CFBPE_ENOMEM if that fails). */
CFBPE_API int cfbpe_encode_batch_lossy(cfbpe_ctx *ctx, uint32_t n_prompts, const uint8_t *bytes, const uint64_t *offsets,
                                       const uint8_t *vocab_ids, uint32_t *out_ids, uint64_t out_cap, uint64_t *out_offsets,
                                       uint32_t *out_counts, uint32_t *out_replaced);
/* The same on device-resident buffers, as cfbpe_encode_batch_device (d_bytes readable for 32 bytes past total_bytes, whose
 * contents do not matter); d_out_replaced (n_prompts entries, may be NULL) is device memory.  The call synchronises `stream` once,
 * after the scan: the host needs its verdict and the repaired size to choose the launch geometry.  The rest is enqueued
 * asynchronously as in cfbpe_encode_batch_device (n_tokens == NULL: nothing more is waited for).  The repaired batch is written to
 * the library's own buffers; the caller's bytes are only read. */
CFBPE_API int cfbpe_encode_batch_lossy_device(cfbpe_ctx *ctx, uint32_t n_prompts, const uint8_t *d_bytes, uint64_t total_bytes,
                                              const uint64_t *d_offsets, const uint8_t *d_vocab_ids, uint32_t *d_out_ids,
                                              uint64_t out_cap, uint64_t *d_out_offsets, uint32_t *d_out_counts,
                                              uint32_t *d_out_replaced, uint64_t *n_tokens, void *stream);
/* Synchronise `stream`, wait for the CALLING THREAD's last device-path call (cfbpe_*_device) on this context, and return that
 * call's status: 0, CFBPE_EILSEQ, CFBPE_ENOENT (an unloaded vocabulary) or CFBPE_ENOSPC (against its out_cap or chunk_cap); 0
 * when the thread has made none there.  Only a later device-path call of the same thread on the same context replaces it: host
 * calls, decode, other threads' calls and calls on other contexts do not.  A device-path call that fails before its work is
 * queued (a bad argument, a disallowed special token, a repaired batch that does not fit) replaces nothing.  Each device-path
 * call copies its status into a record of the thread when its work ends (one small device-to-host copy on its stream); the
 * context frees the records in cfbpe_destroy. */
CFBPE_API int cfbpe_device_status(cfbpe_ctx *ctx, void *stream);

/* page-locked host memory the DMA engines can read without a staging copy */
CFBPE_API void *cfbpe_host_alloc(cfbpe_ctx *ctx, size_t size);
CFBPE_API void cfbpe_host_free(cfbpe_ctx *ctx, void *ptr);

/* CUDA-event timing of each kernel of the following calls (adds event records, no syncs) */
CFBPE_API int cfbpe_profile_enable(cfbpe_ctx *ctx, int on);
CFBPE_API int cfbpe_profile_read(cfbpe_ctx *ctx, cfbpe_profile *out);

#ifdef __cplusplus
}
#endif
#endif /* CFBPE_H */
