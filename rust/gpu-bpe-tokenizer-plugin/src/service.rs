//! The plugin's service: owns the device context, resolves vocabularies, maps errors, keeps CUDA syncs off the runtime.

use std::collections::HashMap;
use std::sync::Arc;

use async_trait::async_trait;
use cfbpe_sys::{Ctx, NativeError};
use llm_gateway_sdk::{
    ChunkBatchResponse, CountTokensRequest, DecodeBatchRequest, DecodeBatchResponse, EncodeBatchRequest, EncodeBatchResponse, InvalidUtf8, OffsetUnit, SpecialTokens,
    TokenizerError, TokenizerPluginClient, TruncateBatchResponse, TruncateKeep, VocabRef,
};
use modkit_security::SecurityContext;
use sha2::{Digest, Sha256};

use crate::batcher::CountBatcher;
use crate::config::{GpuBpeTokenizerPluginConfig, Pattern, RankFileFormat};

pub struct Service {
    native: Arc<Ctx>,
    /// vocabulary name or canonical model id -> slot on the device context
    slots: HashMap<String, u8>,
    names: Vec<String>,
    batcher: CountBatcher,
    /// slot -> the special tokens registered on it, in registration order (= the special index of the per-call modes)
    specials: Arc<std::sync::Mutex<HashMap<u8, Vec<(String, u32)>>>>,
}

fn map_native(e: NativeError) -> TokenizerError {
    match e.code {
        // (EBADMSG: the message names the disallowed special token)
        cfbpe_sys::CFBPE_EINVAL | cfbpe_sys::CFBPE_EILSEQ | cfbpe_sys::CFBPE_ENOSPC | cfbpe_sys::CFBPE_EBADMSG => TokenizerError::InvalidInput(e.message),
        cfbpe_sys::CFBPE_ENOENT => TokenizerError::VocabNotFound { vocab: e.message },
        cfbpe_sys::CFBPE_ENODEV | cfbpe_sys::CFBPE_ENOMEM => TokenizerError::ServiceUnavailable(e.message),
        _ => TokenizerError::Internal(e.message),
    }
}

impl Service {
    /// Blocking: called from `spawn_blocking` in `Module::init`.
    pub fn from_config(cfg: &GpuBpeTokenizerPluginConfig) -> anyhow::Result<Self> {
        let native = Ctx::create(&cfg.devices, cfg.max_batch_bytes, cfg.max_prompts, cfg.workspaces)
            .map_err(|e| anyhow::anyhow!("no H100 device context (there is no CPU fallback): {e}"))?;
        let mut slots = HashMap::new();
        let mut names = Vec::new();
        for (slot, v) in cfg.vocabs.iter().enumerate() {
            anyhow::ensure!(slot < cfbpe_sys::CFBPE_MAX_VOCABS as usize, "at most {} vocabularies per context", cfbpe_sys::CFBPE_MAX_VOCABS);
            let file = std::fs::read(&v.path)?;
            let sha = format!("{:x}", Sha256::digest(&file));
            anyhow::ensure!(sha.eq_ignore_ascii_case(&v.sha256), "{}: sha256 {sha} does not match the configured {}", v.path, v.sha256);
            let format = match v.format {
                RankFileFormat::Tiktoken => cfbpe_sys::CFBPE_FORMAT_TIKTOKEN,
                RankFileFormat::TekkenJson => cfbpe_sys::CFBPE_FORMAT_TEKKEN_JSON,
            };
            let pattern = match v.pattern {
                Pattern::Cl100k => 0,
                Pattern::O200k => 1,
                Pattern::Llama3 => 2,
                Pattern::Tekken => 3,
            };
            native.vocab_load(slot as u32, &file, format, pattern, v.max_ranks).map_err(|e| anyhow::anyhow!("{}: {e}", v.name))?;
            if v.id_base > 0 {       // the model's own ids: control tokens first, the ordinary tokens after them
                native.vocab_set_id_base(slot as u32, v.id_base).map_err(|e| anyhow::anyhow!("{}: {e}", v.name))?;
                if let Some(path) = &v.controls_path {
                    let controls: Vec<String> = serde_json::from_slice(&std::fs::read(path)?)?;
                    anyhow::ensure!(controls.len() == v.id_base as usize, "{path}: {} control tokens for id base {}", controls.len(), v.id_base);
                    let specials: Vec<(String, u32)> = controls.into_iter().zip(0u32..).collect();
                    native.vocab_set_specials(slot as u32, &specials).map_err(|e| anyhow::anyhow!("{}: {e}", v.name))?;
                }
            }
            slots.insert(v.name.clone(), slot as u8);
            for m in &v.models {
                slots.insert(m.clone(), slot as u8);
            }
            names.push(v.name.clone());
        }
        let native = Arc::new(native);
        let batcher = CountBatcher::start(native.clone(), cfg.batch_bytes.min(cfg.max_batch_bytes), cfg.max_prompts, cfg.batch_wait_us);
        Ok(Self { native, slots, names, batcher, specials: Arc::default() })
    }

    pub fn vocab_names(&self) -> &[String] {
        &self.names
    }

    fn slot(&self, v: &VocabRef) -> Result<u8, TokenizerError> {
        self.slots.get(&v.0).copied().ok_or_else(|| TokenizerError::VocabNotFound { vocab: v.0.clone() })
    }

    /// one vocabulary id per prompt, or `None` when the whole batch uses slot 0
    fn vocab_ids(&self, vocab: &VocabRef, per_prompt: Option<&[VocabRef]>, index: Option<&[u8]>, n: usize) -> Result<Option<Vec<u8>>, TokenizerError> {
        if let (Some(table), Some(idx)) = (per_prompt, index) {
            // a table of distinct vocabularies + one index per prompt
            if idx.len() != n {
                return Err(TokenizerError::InvalidInput("vocab_index must hold one entry per prompt".to_owned()));
            }
            let lut = table.iter().map(|r| self.slot(r)).collect::<Result<Vec<_>, _>>()?;
            return idx
                .iter()
                .map(|&i| lut.get(i as usize).copied().ok_or_else(|| TokenizerError::InvalidInput(format!("vocab_index names entry {i} of {} vocabularies", lut.len()))))
                .collect::<Result<Vec<_>, _>>()
                .map(Some);
        }
        match per_prompt {
            Some(v) if v.len() != n => Err(TokenizerError::InvalidInput("vocabs_per_prompt must name one vocabulary per prompt".to_owned())),
            Some(v) => v.iter().map(|r| self.slot(r)).collect::<Result<Vec<_>, _>>().map(Some),
            None => {
                let s = self.slot(vocab)?;
                Ok(if s == 0 { None } else { Some(vec![s; n.max(1)]) })
            }
        }
    }
}

#[async_trait]
impl TokenizerPluginClient for Service {
    async fn encode_batch(&self, ctx: &SecurityContext, req: EncodeBatchRequest) -> Result<EncodeBatchResponse, TokenizerError> {
        if req.invalid_utf8 == InvalidUtf8::Replace {
            return self.encode_batch_lossy(ctx, req).await;
        }
        let n = req.offsets.len().saturating_sub(1);
        let vid = self.vocab_ids(&req.vocab, req.vocabs_per_prompt.as_deref(), req.vocab_index.as_deref(), n)?;
        let native = self.native.clone();
        // never block a tokio worker on a CUDA synchronisation (precedent: modules/file-parser/src/infra/parsers/html_parser.rs:47)
        let (out, starts, lens) = tokio::task::spawn_blocking(move || {
            let unit = match req.starts_unit {
                OffsetUnit::Byte => None,
                OffsetUnit::Codepoint => Some(cfbpe_sys::CFBPE_UNIT_CODEPOINT),
                OffsetUnit::Utf16 => Some(cfbpe_sys::CFBPE_UNIT_UTF16),
            };
            match (req.with_starts, unit) {
                (true, Some(u)) => native.encode_batch_char_starts(&req.bytes, &req.offsets, vid.as_deref(), u).map(|(e, s, l)| (e, Some(s), Some(l))),
                (true, None) => native.encode_batch_starts(&req.bytes, &req.offsets, vid.as_deref()).map(|(e, s)| (e, Some(s), None)),
                (false, _) => native.encode_batch(&req.bytes, &req.offsets, vid.as_deref()).map(|e| (e, None, None)),
            }
        })
            .await
            .map_err(|e| TokenizerError::Internal(e.to_string()))?
            .map_err(map_native)?;
        Ok(EncodeBatchResponse { ids: out.ids, offsets: out.offsets, counts: out.counts, starts, lens, replaced: None })
    }

    /// The device path (`cfbpe_encode_batch_lossy`): the bytes are checked, and repaired where they must be, on the device.
    async fn encode_batch_lossy(&self, _ctx: &SecurityContext, req: EncodeBatchRequest) -> Result<EncodeBatchResponse, TokenizerError> {
        if req.with_starts {
            return Err(TokenizerError::InvalidInput("InvalidUtf8::Replace returns no starts: they would index the repaired text".to_owned()));
        }
        let n = req.offsets.len().saturating_sub(1);
        let vid = self.vocab_ids(&req.vocab, req.vocabs_per_prompt.as_deref(), req.vocab_index.as_deref(), n)?;
        let native = self.native.clone();
        let (out, replaced) = tokio::task::spawn_blocking(move || native.encode_batch_lossy(&req.bytes, &req.offsets, vid.as_deref()))
            .await
            .map_err(|e| TokenizerError::Internal(e.to_string()))?
            .map_err(map_native)?;
        Ok(EncodeBatchResponse { ids: out.ids, offsets: out.offsets, counts: out.counts, starts: None, lens: None, replaced: Some(replaced) })
    }

    /// The device path (`cfbpe_encode_batch_lossy` without ids); such requests do not ride in the shared count batches.
    async fn count_tokens_lossy(&self, _ctx: &SecurityContext, req: CountTokensRequest) -> Result<Vec<u32>, TokenizerError> {
        let n = req.offsets.len().saturating_sub(1);
        let vid = self.vocab_ids(&req.vocab, req.vocabs_per_prompt.as_deref(), req.vocab_index.as_deref(), n)?;
        let native = self.native.clone();
        tokio::task::spawn_blocking(move || native.count_batch_lossy(&req.bytes, &req.offsets, vid.as_deref()))
            .await
            .map_err(|e| TokenizerError::Internal(e.to_string()))?
            .map_err(map_native)
    }

    /// The device path (`cfbpe_encode_batch_char_starts`): the unit starts are computed where the ids and byte starts are.
    async fn encode_batch_unit_starts(&self, ctx: &SecurityContext, req: EncodeBatchRequest) -> Result<EncodeBatchResponse, TokenizerError> {
        self.encode_batch(ctx, EncodeBatchRequest { with_starts: true, ..req }).await
    }

    async fn count_tokens(&self, ctx: &SecurityContext, req: CountTokensRequest) -> Result<Vec<u32>, TokenizerError> {
        if req.invalid_utf8 == InvalidUtf8::Replace {
            return self.count_tokens_lossy(ctx, req).await;
        }
        let n = req.offsets.len().saturating_sub(1);
        let vid = self.vocab_ids(&req.vocab, req.vocabs_per_prompt.as_deref(), req.vocab_index.as_deref(), n)?;
        // small requests (a chat message is a few KB) ride in a shared device batch; large ones go straight through
        if (req.bytes.len() as u64) < self.batcher.direct_threshold() {
            return self.batcher.count(req.bytes, req.offsets, vid).await;
        }
        let native = self.native.clone();
        tokio::task::spawn_blocking(move || native.count_batch(&req.bytes, &req.offsets, vid.as_deref()))
            .await
            .map_err(|e| TokenizerError::Internal(e.to_string()))?
            .map_err(map_native)
    }

    async fn decode_batch(&self, _ctx: &SecurityContext, req: DecodeBatchRequest) -> Result<DecodeBatchResponse, TokenizerError> {
        let n = req.offsets.len().saturating_sub(1);
        let vid = self.vocab_ids(&req.vocab, req.vocabs_per_prompt.as_deref(), req.vocab_index.as_deref(), n)?;
        let native = self.native.clone();
        let (bytes, offsets) = tokio::task::spawn_blocking(move || native.decode_batch(&req.ids, &req.offsets, vid.as_deref()))
            .await
            .map_err(|e| TokenizerError::Internal(e.to_string()))?
            .map_err(map_native)?;
        Ok(DecodeBatchResponse { bytes, offsets })
    }

    /// The device path (`cfbpe_truncate_batch`): the cut is a sum of token lengths where the ids are; no id leaves the device.
    async fn truncate_batch(&self, _ctx: &SecurityContext, req: EncodeBatchRequest, budgets: &[u32], keep: TruncateKeep)
        -> Result<TruncateBatchResponse, TokenizerError> {
        let n = req.offsets.len().saturating_sub(1);
        if budgets.len() != n {
            return Err(TokenizerError::InvalidInput("one token budget per prompt".to_owned()));
        }
        let vid = self.vocab_ids(&req.vocab, req.vocabs_per_prompt.as_deref(), req.vocab_index.as_deref(), n)?;
        let mode = match keep { TruncateKeep::Head => cfbpe_sys::CFBPE_TRUNCATE_HEAD, TruncateKeep::Tail => cfbpe_sys::CFBPE_TRUNCATE_TAIL };
        let (native, budgets) = (self.native.clone(), budgets.to_vec());
        let out = tokio::task::spawn_blocking(move || native.truncate_batch(&req.bytes, &req.offsets, vid.as_deref(), &budgets, mode))
            .await
            .map_err(|e| TokenizerError::Internal(e.to_string()))?
            .map_err(map_native)?;
        Ok(TruncateBatchResponse { cut: out.cut, kept: out.kept, counts: out.counts })
    }

    /// The device path (`cfbpe_chunk_batch`): the chunks are cut from the token starts where they are; no id or start leaves the device.
    async fn chunk_batch(&self, _ctx: &SecurityContext, req: EncodeBatchRequest, chunk_tokens: u32, overlap_tokens: u32)
        -> Result<ChunkBatchResponse, TokenizerError> {
        if chunk_tokens == 0 || overlap_tokens >= chunk_tokens {
            return Err(TokenizerError::InvalidInput("the chunk size must be at least 1 and the overlap less than it".to_owned()));
        }
        let n = req.offsets.len().saturating_sub(1);
        let vid = self.vocab_ids(&req.vocab, req.vocabs_per_prompt.as_deref(), req.vocab_index.as_deref(), n)?;
        let native = self.native.clone();
        let out = tokio::task::spawn_blocking(move || native.chunk_batch(&req.bytes, &req.offsets, vid.as_deref(), chunk_tokens, overlap_tokens))
            .await
            .map_err(|e| TokenizerError::Internal(e.to_string()))?
            .map_err(map_native)?;
        Ok(ChunkBatchResponse { spans: out.spans, chunk_offsets: out.chunk_offsets, counts: out.counts })
    }

    /// The device path: scan, cut and splice run as CUDA kernels (`cfbpe_encode_batch_special`).  The caller's special tokens
    /// are registered on every slot the request uses when they differ from what the slot holds.
    async fn encode_batch_special(&self, _ctx: &SecurityContext, req: EncodeBatchRequest, special: &SpecialTokens)
        -> Result<EncodeBatchResponse, TokenizerError> {
        let n = req.offsets.len().saturating_sub(1);
        let vid = self.vocab_ids(&req.vocab, req.vocabs_per_prompt.as_deref(), req.vocab_index.as_deref(), n)?;
        let mut used: Vec<u8> = match &vid { Some(v) => v[..n].to_vec(), None => vec![self.slot(&req.vocab)?] };
        used.sort_unstable();
        used.dedup();
        let want: Vec<(String, u32)> = special.ids.iter().map(|(t, id)| (t.clone(), *id)).collect();
        let modes: Vec<u8> = want.iter().map(|(t, _)| {
            if special.allowed.contains(t) { cfbpe_sys::CFBPE_SPECIAL_ALLOW }
            else if special.disallow_all_others { cfbpe_sys::CFBPE_SPECIAL_DISALLOW }
            else { cfbpe_sys::CFBPE_SPECIAL_ORDINARY }
        }).collect();
        let (native, specials) = (self.native.clone(), self.specials.clone());
        let out = tokio::task::spawn_blocking(move || {
            let mut held = specials.lock().unwrap_or_else(std::sync::PoisonError::into_inner);
            let mut per_vocab: Vec<Option<&[u8]>> = vec![None; cfbpe_sys::CFBPE_MAX_VOCABS as usize];
            for &slot in &used {
                if held.get(&slot) != Some(&want) {
                    native.vocab_set_specials(u32::from(slot), &want)?;
                    held.insert(slot, want.clone());
                }
                per_vocab[slot as usize] = Some(&modes);
            }
            native.encode_batch_special(&req.bytes, &req.offsets, vid.as_deref(), &per_vocab)
        })
        .await
        .map_err(|e| TokenizerError::Internal(e.to_string()))?
        .map_err(map_native)?;
        Ok(EncodeBatchResponse { ids: out.ids, offsets: out.offsets, counts: out.counts, starts: None, lens: None, replaced: None })
    }
}

pub(crate) fn map_native_error(e: NativeError) -> TokenizerError {
    map_native(e)
}
