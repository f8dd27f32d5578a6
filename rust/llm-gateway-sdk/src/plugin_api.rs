//! Plugin API trait of tokenizer implementations (shape of `tenant-resolver-sdk/src/plugin_api.rs:28-47`).

use async_trait::async_trait;
use modkit_security::SecurityContext;

use crate::error::TokenizerError;
use crate::models::{chunk_spans, truncate_cut, unit_starts, ChunkBatchResponse, CountTokensRequest, DecodeBatchRequest, DecodeBatchResponse, EncodeBatchRequest, EncodeBatchResponse,
                    InvalidUtf8, OffsetUnit, SpecialTokens, TruncateBatchResponse, TruncateKeep, VocabRef};

/// Each plugin registers this trait with a scoped `ClientHub` entry using its GTS instance id as the scope.  Clients are
/// `Arc<dyn … + Send + Sync>` shared by all tokio tasks (`libs/modkit/src/client_hub.rs:142-165`): calls are concurrent and
/// re-entrant, and an implementation must not block a runtime worker on a device synchronisation (use `spawn_blocking`).
#[async_trait]
pub trait TokenizerPluginClient: Send + Sync {
    /// Token ids of every prompt of the batch.
    ///
    /// # Errors
    /// `InvalidInput` (offsets, malformed UTF-8, batch too large), `VocabNotFound`, `ServiceUnavailable`, `Internal`.
    async fn encode_batch(&self, ctx: &SecurityContext, req: EncodeBatchRequest) -> Result<EncodeBatchResponse, TokenizerError>;

    /// Token count of every prompt of the batch (`usage::count_tokens`); same errors.
    async fn count_tokens(&self, ctx: &SecurityContext, req: CountTokensRequest) -> Result<Vec<u32>, TokenizerError>;

    /// ids -> bytes; `InvalidInput` for an id outside its vocabulary.
    async fn decode_batch(&self, ctx: &SecurityContext, req: DecodeBatchRequest) -> Result<DecodeBatchResponse, TokenizerError>;

    /// Cut every prompt of the batch to its token budget (`budgets`: one per prompt), keeping its first or last tokens, at a
    /// character boundary (`TruncateBatchResponse`).  The default works on any plugin that returns token starts: one
    /// `encode_batch` with `with_starts`, then the cut on the host.  `gpu-bpe-tokenizer-plugin` overrides it with the device
    /// call, which downloads no ids.
    async fn truncate_batch(&self, ctx: &SecurityContext, req: EncodeBatchRequest, budgets: &[u32], keep: TruncateKeep)
        -> Result<TruncateBatchResponse, TokenizerError> {
        let n = req.offsets.len().saturating_sub(1);
        if budgets.len() != n {
            return Err(TokenizerError::InvalidInput("one token budget per prompt".to_owned()));
        }
        let bytes = req.bytes.clone();
        let offsets = req.offsets.clone();
        let enc = self.encode_batch(ctx, EncodeBatchRequest { with_starts: true, starts_unit: OffsetUnit::Byte, ..req }).await?;
        let starts = enc.starts.ok_or_else(|| TokenizerError::ServiceUnavailable("the tokenizer plugin does not return token starts".to_owned()))?;
        let mut out = TruncateBatchResponse { cut: Vec::with_capacity(n), kept: Vec::with_capacity(n), counts: enc.counts };
        for i in 0..n {
            let prompt = &bytes[offsets[i] as usize..offsets[i + 1] as usize];
            let (cut, kept) = truncate_cut(prompt, &starts[enc.offsets[i] as usize..enc.offsets[i + 1] as usize], budgets[i], keep);
            out.cut.push(cut);
            out.kept.push(kept);
        }
        Ok(out)
    }

    /// Cut every prompt of the batch into chunks of at most `chunk_tokens` tokens that overlap by `overlap_tokens`, at character
    /// boundaries of the whole prompt's encoding (`ChunkBatchResponse`).  The default works on any plugin that returns token
    /// starts: one `encode_batch` with `with_starts`, then the cuts on the host.  `gpu-bpe-tokenizer-plugin` overrides it with the
    /// device call, which downloads no ids and no starts.
    async fn chunk_batch(&self, ctx: &SecurityContext, req: EncodeBatchRequest, chunk_tokens: u32, overlap_tokens: u32)
        -> Result<ChunkBatchResponse, TokenizerError> {
        if chunk_tokens == 0 || overlap_tokens >= chunk_tokens {
            return Err(TokenizerError::InvalidInput("the chunk size must be at least 1 and the overlap less than it".to_owned()));
        }
        let n = req.offsets.len().saturating_sub(1);
        let bytes = req.bytes.clone();
        let offsets = req.offsets.clone();
        let enc = self.encode_batch(ctx, EncodeBatchRequest { with_starts: true, starts_unit: OffsetUnit::Byte, ..req }).await?;
        let starts = enc.starts.ok_or_else(|| TokenizerError::ServiceUnavailable("the tokenizer plugin does not return token starts".to_owned()))?;
        let mut out = ChunkBatchResponse { spans: Vec::new(), chunk_offsets: Vec::with_capacity(n + 1), counts: enc.counts };
        out.chunk_offsets.push(0);
        for i in 0..n {
            let prompt = &bytes[offsets[i] as usize..offsets[i + 1] as usize];
            out.spans.extend(chunk_spans(prompt, &starts[enc.offsets[i] as usize..enc.offsets[i + 1] as usize], chunk_tokens, overlap_tokens));
            out.chunk_offsets.push(out.spans.len() as u64);
        }
        Ok(out)
    }

    /// `encode_batch` of a request with `InvalidUtf8::Replace`: every prompt encoded as `String::from_utf8_lossy` would have it,
    /// and `EncodeBatchResponse::replaced` -- `include/cfbpe.h`, `cfbpe_encode_batch_lossy`.  The default works on any plugin: it
    /// repairs every prompt on the host and sends the repaired batch through one strict `encode_batch`.
    /// `gpu-bpe-tokenizer-plugin` overrides it with the device call.
    async fn encode_batch_lossy(&self, ctx: &SecurityContext, req: EncodeBatchRequest) -> Result<EncodeBatchResponse, TokenizerError> {
        if req.with_starts {
            return Err(TokenizerError::InvalidInput("InvalidUtf8::Replace returns no starts: they would index the repaired text".to_owned()));
        }
        let (bytes, offsets, replaced) = repair_utf8(&req.bytes, &req.offsets);
        let mut enc = self.encode_batch(ctx, EncodeBatchRequest { bytes: bytes.into(), offsets, invalid_utf8: InvalidUtf8::Reject, ..req }).await?;
        enc.replaced = Some(replaced);
        Ok(enc)
    }

    /// `count_tokens` of a request with `InvalidUtf8::Replace`; this default repairs on the host, as `encode_batch_lossy`.
    async fn count_tokens_lossy(&self, ctx: &SecurityContext, req: CountTokensRequest) -> Result<Vec<u32>, TokenizerError> {
        let (bytes, offsets, _) = repair_utf8(&req.bytes, &req.offsets);
        self.count_tokens(ctx, CountTokensRequest { bytes: bytes.into(), offsets, invalid_utf8: InvalidUtf8::Reject, ..req }).await
    }

    /// `encode_batch` with every token's start in `req.starts_unit` and, for a character unit, every prompt's length in it
    /// (`EncodeBatchResponse::lens`) -- `include/cfbpe.h`, `cfbpe_encode_batch_char_starts`.  The default works on any plugin that
    /// returns byte starts: one `encode_batch` with byte starts, then `unit_starts` on the host.  `gpu-bpe-tokenizer-plugin`
    /// overrides it with the device call, which walks no text on the host.
    async fn encode_batch_unit_starts(&self, ctx: &SecurityContext, req: EncodeBatchRequest) -> Result<EncodeBatchResponse, TokenizerError> {
        let unit = req.starts_unit;
        let n = req.offsets.len().saturating_sub(1);
        let bytes = req.bytes.clone();
        let offsets = req.offsets.clone();
        let mut enc = self.encode_batch(ctx, EncodeBatchRequest { with_starts: true, starts_unit: OffsetUnit::Byte, ..req }).await?;
        if unit == OffsetUnit::Byte {
            return Ok(enc);
        }
        let byte_starts = enc.starts.take().ok_or_else(|| TokenizerError::ServiceUnavailable("the tokenizer plugin does not return token starts".to_owned()))?;
        let (mut starts, mut lens) = (Vec::with_capacity(byte_starts.len()), Vec::with_capacity(n));
        for i in 0..n {
            let prompt = &bytes[offsets[i] as usize..offsets[i + 1] as usize];
            let (s, len) = unit_starts(prompt, &byte_starts[enc.offsets[i] as usize..enc.offsets[i + 1] as usize], unit);
            starts.extend(s);
            lens.push(len);
        }
        enc.starts = Some(starts);
        enc.lens = Some(lens);
        Ok(enc)
    }

    /// tiktoken's `encode(text, allowed_special = …, disallowed_special = …)` for every prompt of the batch; `InvalidInput` when
    /// a prompt spells a special token that is not allowed.  The default works on any plugin: it cuts every text at the
    /// allowed special tokens on the host (leftmost, then the longest there), sends all stretches of all texts through ONE
    /// `encode_batch`, and puts the special ids back.  `gpu-bpe-tokenizer-plugin` overrides it with the device path.
    async fn encode_batch_special(&self, ctx: &SecurityContext, req: EncodeBatchRequest, special: &SpecialTokens)
        -> Result<EncodeBatchResponse, TokenizerError> {
        let n = req.offsets.len().saturating_sub(1);
        let mut texts = Vec::with_capacity(n);
        for i in 0..n {
            let b = &req.bytes[req.offsets[i] as usize..req.offsets[i + 1] as usize];
            texts.push(std::str::from_utf8(b).map_err(|_| TokenizerError::InvalidInput("a prompt holds malformed UTF-8".to_owned()))?);
        }
        let mut allowed: Vec<&String> = special.allowed.iter().collect();
        allowed.sort_by_key(|t| std::cmp::Reverse(t.len()));
        if special.disallow_all_others {
            for t in &texts {
                if let Some(bad) = special.ids.keys().find(|k| !special.allowed.contains(*k) && t.contains(k.as_str())) {
                    return Err(TokenizerError::InvalidInput(format!("the text holds the special token {bad:?}, which is not allowed here")));
                }
            }
        }
        enum Step { Stretch(usize), Special(u32) }
        let (mut plan, mut stretches): (Vec<Vec<Step>>, Vec<&str>) = (Vec::new(), Vec::new());
        let mut per: Option<Vec<VocabRef>> = req.vocabs_per_prompt.as_ref().map(|_| Vec::new());
        for (p, t) in texts.iter().enumerate() {
            let (mut steps, mut pos) = (Vec::new(), 0usize);
            let vocab_of = |p: usize| req.vocabs_per_prompt.as_ref().map(|v| match &req.vocab_index { Some(ix) => v[ix[p] as usize].clone(), None => v[p].clone() });
            while pos < t.len() {
                let next = allowed.iter().filter_map(|tok| t[pos..].find(tok.as_str()).map(|i| (pos + i, *tok))).min_by_key(|(i, tok)| (*i, std::cmp::Reverse(tok.len())));
                let end = next.map_or(t.len(), |(i, _)| i);
                if end > pos {
                    steps.push(Step::Stretch(stretches.len()));
                    stretches.push(&t[pos..end]);
                    if let (Some(per), Some(v)) = (per.as_mut(), vocab_of(p)) { per.push(v); }
                }
                match next {
                    Some((i, tok)) => { steps.push(Step::Special(special.ids[tok])); pos = i + tok.len(); }
                    None => pos = t.len(),
                }
            }
            plan.push(steps);
        }
        let enc = if stretches.is_empty() {
            EncodeBatchResponse { ids: Vec::new(), offsets: vec![0], counts: Vec::new(), starts: None, lens: None, replaced: None }
        } else {
            let mut bytes = Vec::new();
            let mut offsets = vec![0u64];
            for s in &stretches { bytes.extend_from_slice(s.as_bytes()); offsets.push(bytes.len() as u64); }
            self.encode_batch(ctx, EncodeBatchRequest { vocab: req.vocab.clone(), bytes: bytes.into(), offsets, vocabs_per_prompt: per.take(), vocab_index: None, with_starts: false, starts_unit: OffsetUnit::Byte, invalid_utf8: InvalidUtf8::Reject }).await?
        };
        let mut out = EncodeBatchResponse { ids: Vec::new(), offsets: vec![0u64], counts: Vec::with_capacity(n), starts: None, lens: None, replaced: None };
        for steps in plan {
            let start = out.ids.len();
            for s in steps {
                match s {
                    Step::Stretch(i) => out.ids.extend_from_slice(&enc.ids[enc.offsets[i] as usize..enc.offsets[i + 1] as usize]),
                    Step::Special(id) => out.ids.push(id),
                }
            }
            out.counts.push((out.ids.len() - start) as u32);
            out.offsets.push(out.ids.len() as u64);
        }
        Ok(out)
    }
}

/// Every prompt of a packed batch as `String::from_utf8_lossy` makes it: `(bytes, offsets, replaced)`, `replaced[i]` the U+FFFD the
/// repair inserted into prompt `i` (one per maximal subpart of an ill-formed sequence; a U+FFFD already in the text does not count).
pub fn repair_utf8(bytes: &[u8], offsets: &[u64]) -> (Vec<u8>, Vec<u64>, Vec<u32>) {
    let n = offsets.len().saturating_sub(1);
    let (mut out, mut out_offsets, mut replaced) = (Vec::with_capacity(bytes.len()), Vec::with_capacity(n + 1), Vec::with_capacity(n));
    out_offsets.push(0u64);
    for i in 0..n {
        let prompt = &bytes[offsets[i] as usize..offsets[i + 1] as usize];
        let text = String::from_utf8_lossy(prompt);
        let had = text.matches('\u{FFFD}').count();
        let kept = prompt.windows(3).filter(|w| *w == "\u{FFFD}".as_bytes()).count();
        replaced.push((had - kept) as u32);
        out.extend_from_slice(text.as_bytes());
        out_offsets.push(out.len() as u64);
    }
    (out, out_offsets, replaced)
}
