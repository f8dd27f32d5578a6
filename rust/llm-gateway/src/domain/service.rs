//! `llm-gateway::tokenizer` + `llm-gateway::usage::count_tokens`: the gateway-side domain service.
//! Plugin resolution is lazy and single-flight (`libs/modkit/src/plugins/mod.rs:44-78`): vendor match, lowest priority wins
//! (`:136-191`).  Prompt text is never logged (`docs/DESIGN.md:120-124`): only sizes and counts.

use std::sync::Arc;

use async_trait::async_trait;
use bytes::Bytes;
use llm_gateway_sdk::{
    ChatTemplate, CountTokensRequest, EncodeBatchRequest, InvalidUtf8, OffsetUnit, SpecialTokens, TokenizerClient, TokenizerError, TokenizerPluginClient, TokenizerPluginSpecV1,
    TruncateKeep, Usage, VocabRef,
};
use modkit::client_hub::{ClientHub, ClientScope};
use modkit::plugins::{choose_plugin_instance, GtsPluginSelector};
use modkit_security::SecurityContext;
use serde_json::Value;
use types_registry_sdk::{ListQuery, TypesRegistryClient};

pub struct TokenizerService {
    hub: Arc<ClientHub>,
    vendor: String,
    selector: GtsPluginSelector,
}

/// list[str] -> (packed bytes, n + 1 offsets): the packed multi-tenant prompt buffer the device reads
pub fn pack_texts<S: AsRef<str>>(texts: &[S]) -> (Bytes, Vec<u64>) {
    let mut bytes = Vec::with_capacity(texts.iter().map(|t| t.as_ref().len()).sum());
    let mut offsets = Vec::with_capacity(texts.len() + 1);
    offsets.push(0u64);
    for t in texts {
        bytes.extend_from_slice(t.as_ref().as_bytes());
        offsets.push(bytes.len() as u64);
    }
    (Bytes::from(bytes), offsets)
}

impl TokenizerService {
    pub fn new(hub: Arc<ClientHub>, vendor: String) -> Self {
        Self { hub, vendor, selector: GtsPluginSelector::new() }
    }

    async fn plugin(&self) -> Result<Arc<dyn TokenizerPluginClient>, TokenizerError> {
        let instance_id = self
            .selector
            .get_or_init(|| async {
                let registry = self.hub.get::<dyn TypesRegistryClient>().map_err(|e| TokenizerError::Internal(e.to_string()))?;
                let plugin_type_id = TokenizerPluginSpecV1::gts_schema_id().clone();
                let instances = registry
                    .list(ListQuery::new().with_pattern(format!("{plugin_type_id}*")).with_is_type(false))
                    .await
                    .map_err(|e| TokenizerError::Internal(e.to_string()))?;
                choose_plugin_instance::<TokenizerPluginSpecV1>(&self.vendor, instances.iter().map(|e| (e.gts_id.as_str(), &e.content)))
                    .map_err(|_| TokenizerError::NoPluginAvailable)
            })
            .await?;
        self.hub
            .try_get_scoped::<dyn TokenizerPluginClient>(&ClientScope::gts_id(instance_id.as_ref()))
            .ok_or_else(|| TokenizerError::ServiceUnavailable(format!("tokenizer plugin {instance_id} is not registered yet")))
    }

    /// Per text: its chunks, their `[begin, end)` spans in its UTF-8 and its token count (`POST /llm-gateway/v1/chunk`).  The plugin
    /// does the work: the trait's default cuts on the host from token starts, the GPU plugin cuts on the device.
    pub async fn chunk_with_spans(&self, ctx: &SecurityContext, model: &str, texts: &[String], max_tokens: u32, overlap: u32)
        -> Result<Vec<(Vec<String>, Vec<[u32; 2]>, u32)>, TokenizerError> {
        let (bytes, offsets) = pack_texts(texts);
        let req = EncodeBatchRequest { vocab: VocabRef(model.to_owned()), bytes, offsets, vocabs_per_prompt: None, vocab_index: None, with_starts: false,
                                       starts_unit: OffsetUnit::Byte, invalid_utf8: InvalidUtf8::Reject };
        let r = self.plugin().await?.chunk_batch(ctx, req, max_tokens, overlap).await?;
        texts.iter().enumerate().map(|(i, t)| {
            let spans = r.spans[r.chunk_offsets[i] as usize..r.chunk_offsets[i + 1] as usize].to_vec();
            // a span always ends on character boundaries (include/cfbpe.h); get() refuses anything else instead of panicking
            let chunks = spans.iter().map(|&[b, e]| t.get(b as usize..e as usize).map(str::to_owned)
                .ok_or_else(|| TokenizerError::Internal(format!("the plugin cut text {i} inside a character")))).collect::<Result<Vec<_>, _>>()?;
            Ok((chunks, spans, r.counts[i]))
        }).collect()
    }

    /// the `TextContent.text` parts of a request's messages (`schemas/core/message.v1.schema.json`)
    fn text_parts(messages: &[Value]) -> Vec<String> {
        messages
            .iter()
            .filter_map(|m| m.get("content")?.as_array())
            .flatten()
            .filter(|p| p.get("type").and_then(Value::as_str) == Some("text"))
            .filter_map(|p| p.get("text")?.as_str().map(str::to_owned))
            .collect()
    }
}

#[async_trait]
impl TokenizerClient for TokenizerService {
    async fn encode(&self, ctx: &SecurityContext, model: &str, texts: &[String]) -> Result<Vec<Vec<u32>>, TokenizerError> {
        let (bytes, offsets) = pack_texts(texts);
        let r = self.plugin().await?.encode_batch(ctx, EncodeBatchRequest { vocab: VocabRef(model.to_owned()), bytes, offsets, vocabs_per_prompt: None, vocab_index: None, with_starts: false,
                                       starts_unit: OffsetUnit::Byte, invalid_utf8: InvalidUtf8::Reject }).await?;
        Ok((0..texts.len()).map(|i| r.ids[r.offsets[i] as usize..r.offsets[i + 1] as usize].to_vec()).collect())
    }

    async fn encode_with_offsets(&self, ctx: &SecurityContext, model: &str, texts: &[String], unit: OffsetUnit)
        -> Result<Vec<(Vec<u32>, Vec<[u64; 2]>)>, TokenizerError> {
        let (bytes, offsets) = pack_texts(texts);
        let req = EncodeBatchRequest { vocab: VocabRef(model.to_owned()), bytes, offsets: offsets.clone(), vocabs_per_prompt: None, vocab_index: None,
                                       with_starts: true, starts_unit: unit, invalid_utf8: InvalidUtf8::Reject };
        // a character unit: the plugin does the work (the trait's default converts byte starts on the host, the GPU plugin counts on the device)
        let plugin = self.plugin().await?;
        let r = if unit == OffsetUnit::Byte { plugin.encode_batch(ctx, req).await? } else { plugin.encode_batch_unit_starts(ctx, req).await? };
        let starts = r.starts.ok_or_else(|| TokenizerError::ServiceUnavailable("the tokenizer plugin does not return token starts".to_owned()))?;
        let lens: Vec<u64> = match (unit, &r.lens) {
            (OffsetUnit::Byte, _) => (0..texts.len()).map(|i| offsets[i + 1] - offsets[i]).collect(),
            (_, Some(l)) => l.iter().map(|&x| u64::from(x)).collect(),
            (_, None) => return Err(TokenizerError::ServiceUnavailable("the tokenizer plugin does not return prompt lengths".to_owned())),
        };
        Ok((0..texts.len()).map(|i| {
            let (a, b) = (r.offsets[i] as usize, r.offsets[i + 1] as usize);
            let len = lens[i];
            let spans = (a..b).map(|k| [u64::from(starts[k]), if k + 1 < b { u64::from(starts[k + 1]) } else { len }]).collect();
            (r.ids[a..b].to_vec(), spans)
        }).collect())
    }

    async fn truncate(&self, ctx: &SecurityContext, model: &str, texts: &[String], max_tokens: &[u32], keep: TruncateKeep)
        -> Result<Vec<(String, u32, u32)>, TokenizerError> {
        // the plugin does the work: the trait's default cuts on the host from token starts, the GPU plugin cuts on the device
        if max_tokens.len() != texts.len() {
            return Err(TokenizerError::InvalidInput("one token budget per text".to_owned()));
        }
        let (bytes, offsets) = pack_texts(texts);
        let req = EncodeBatchRequest { vocab: VocabRef(model.to_owned()), bytes, offsets, vocabs_per_prompt: None, vocab_index: None, with_starts: false,
                                       starts_unit: OffsetUnit::Byte, invalid_utf8: InvalidUtf8::Reject };
        let r = self.plugin().await?.truncate_batch(ctx, req, max_tokens, keep).await?;
        texts.iter().enumerate().map(|(i, t)| {
            let cut = r.cut[i] as usize;
            // a cut is always a character boundary (include/cfbpe.h); get() refuses anything else instead of panicking
            let kept = match keep { TruncateKeep::Head => t.get(..cut), TruncateKeep::Tail => t.get(cut..) }
                .ok_or_else(|| TokenizerError::Internal(format!("the plugin cut text {i} inside a character")))?;
            Ok((kept.to_owned(), r.kept[i], r.counts[i]))
        }).collect()
    }

    async fn chunk(&self, ctx: &SecurityContext, model: &str, texts: &[String], max_tokens: u32, overlap: u32)
        -> Result<Vec<Vec<String>>, TokenizerError> {
        Ok(self.chunk_with_spans(ctx, model, texts, max_tokens, overlap).await?.into_iter().map(|(chunks, _, _)| chunks).collect())
    }

    async fn encode_with_special(&self, ctx: &SecurityContext, model: &str, texts: &[String], special: &SpecialTokens)
        -> Result<Vec<Vec<u32>>, TokenizerError> {
        // the plugin does the work: the trait's default cuts on the host, the GPU plugin scans, cuts and splices on the device
        if let Some(unknown) = special.allowed.iter().find(|t| !special.ids.contains_key(*t)) {
            return Err(TokenizerError::InvalidInput(format!("allowed special token without an id: {unknown}")));
        }
        let (bytes, offsets) = pack_texts(texts);
        let req = EncodeBatchRequest { vocab: VocabRef(model.to_owned()), bytes, offsets, vocabs_per_prompt: None, vocab_index: None, with_starts: false,
                                       starts_unit: OffsetUnit::Byte, invalid_utf8: InvalidUtf8::Reject };
        let r = self.plugin().await?.encode_batch_special(ctx, req, special).await?;
        Ok((0..texts.len()).map(|i| r.ids[r.offsets[i] as usize..r.offsets[i + 1] as usize].to_vec()).collect())
    }

    async fn count_tokens(&self, ctx: &SecurityContext, model: &str, messages: &[Value]) -> Result<Usage, TokenizerError> {
        let texts = Self::text_parts(messages);
        if texts.is_empty() {
            return Ok(Usage::default());
        }
        let (bytes, offsets) = pack_texts(&texts);
        let counts = self.plugin().await?.count_tokens(ctx, CountTokensRequest { vocab: VocabRef(model.to_owned()), bytes, offsets, vocabs_per_prompt: None, vocab_index: None, invalid_utf8: InvalidUtf8::Reject }).await?;
        Ok(Usage { input_tokens: counts.iter().map(|c| u64::from(*c)).sum(), output_tokens: 0 })
    }

    async fn count_chat_tokens(&self, ctx: &SecurityContext, model: &str, messages: &[Value], template: &ChatTemplate) -> Result<Usage, TokenizerError> {
        // every stretch of ordinary text of the whole request goes to the device in ONE batch; control tokens count one each
        let content = |m: &Value| -> String {
            m.get("content").and_then(Value::as_array).map(|parts| {
                parts.iter().filter(|p| p.get("type").and_then(Value::as_str) == Some("text")).filter_map(|p| p.get("text").and_then(Value::as_str)).collect::<String>()
            }).unwrap_or_default()
        };
        let role = |m: &Value| m.get("role").and_then(Value::as_str).unwrap_or("").to_owned();
        let (mut fixed, mut texts): (u64, Vec<String>) = (0, Vec::new());
        match template {
            ChatTemplate::Overhead { tokens_per_message, tokens_per_name, reply_priming } => {
                for m in messages {
                    fixed += u64::from(*tokens_per_message);
                    texts.push(role(m));
                    if let Some(name) = m.get("name").and_then(Value::as_str) {
                        fixed += u64::from(*tokens_per_name);
                        texts.push(name.to_owned());
                    }
                    texts.extend(Self::text_parts(std::slice::from_ref(m)));
                }
                fixed += u64::from(*reply_priming);
            }
            ChatTemplate::Rendered { bos, message_prefix, message_suffix, generation_prompt, special_tokens } => {
                // framing text and content between two control tokens form one stretch (the pre-tokenizer may join them)
                let mut run = vec![String::new()];
                let feed = |framing: &str, fixed: &mut u64, run: &mut Vec<String>| {
                    let mut rest = framing;
                    loop {
                        let next = special_tokens.iter().filter_map(|t| rest.find(t.as_str()).map(|i| (i, t.len()))).min_by_key(|(i, l)| (*i, std::cmp::Reverse(*l)));
                        match next {
                            Some((i, l)) => { run.last_mut().expect("never empty").push_str(&rest[..i]); run.push(String::new()); *fixed += 1; rest = &rest[i + l..]; }
                            None => { run.last_mut().expect("never empty").push_str(rest); break; }
                        }
                    }
                };
                feed(bos, &mut fixed, &mut run);
                for m in messages {
                    feed(&message_prefix.replace("{role}", &role(m)), &mut fixed, &mut run);
                    run.last_mut().expect("never empty").push_str(&content(m));
                    feed(message_suffix, &mut fixed, &mut run);
                }
                feed(generation_prompt, &mut fixed, &mut run);
                texts = run;
            }
            ChatTemplate::Mistral => {
                let text = |m: &Value| Self::text_parts(std::slice::from_ref(m)).join("\n\n");
                let bad = |msg: &str| TokenizerError::InvalidInput(msg.to_owned());
                if messages.is_empty() {
                    return Err(bad("a conversation for the mistral template has at least one message"));
                }
                let system = messages.iter().filter(|m| role(m) == "system").map(text).filter(|t| !t.is_empty()).collect::<Vec<_>>().join("\n\n");
                let mut turns: Vec<(String, String)> = Vec::new();
                let mut prev = String::new();
                for m in messages {
                    let r = role(m);
                    match r.as_str() {
                        "system" if prev == "assistant" => return Err(bad("a system message follows an assistant message")),
                        "system" => {}
                        "user" | "assistant" if r == prev => { let last = turns.last_mut().expect("a turn of this role"); last.1.push_str("\n\n"); last.1.push_str(&text(m)); }
                        "user" | "assistant" => turns.push((r.clone(), text(m))),
                        _ => return Err(bad("the mistral template counts system, user and assistant messages")),
                    }
                    prev = r;
                }
                if turns.first().map_or(true, |t| t.0 != "user") {
                    turns.insert(0, ("user".to_owned(), String::new()));
                }
                if turns.last().map_or(true, |t| t.0 != "user") {
                    return Err(bad("a conversation for the mistral template ends with a user message"));
                }
                let last_user = turns.iter().rposition(|t| t.0 == "user").expect("a user turn");
                fixed = 1;                                                  // <s>
                for (i, (r, t)) in turns.into_iter().enumerate() {
                    if r == "user" {
                        texts.push(if i == last_user && !system.is_empty() { format!("{system}\n\n{t}") } else { t });
                        fixed += 2;                                         // [INST] [/INST]
                    } else {
                        if t.is_empty() {
                            return Err(bad("an assistant message without text"));
                        }
                        texts.push(t.trim_end_matches(' ').to_owned());
                        fixed += 1;                                         // </s>
                    }
                }
            }
        }
        texts.retain(|t| !t.is_empty());
        if texts.is_empty() {
            return Ok(Usage { input_tokens: fixed, output_tokens: 0 });
        }
        let (bytes, offsets) = pack_texts(&texts);
        let counts = self.plugin().await?.count_tokens(ctx, CountTokensRequest { vocab: VocabRef(model.to_owned()), bytes, offsets, vocabs_per_prompt: None, vocab_index: None, invalid_utf8: InvalidUtf8::Reject }).await?;
        Ok(Usage { input_tokens: fixed + counts.iter().map(|c| u64::from(*c)).sum::<u64>(), output_tokens: 0 })
    }

    async fn check_budget(&self, ctx: &SecurityContext, model: &str, messages: &[Value], remaining_tokens: u64) -> Result<bool, TokenizerError> {
        Ok(self.count_tokens(ctx, model, messages).await?.input_tokens <= remaining_tokens)
    }
}
