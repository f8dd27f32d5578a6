//! `llm-gateway::tokenizer` + `llm-gateway::usage::count_tokens`: the gateway-side domain service.
//! Plugin resolution is lazy and single-flight (`libs/modkit/src/plugins/mod.rs:44-78`): vendor match, lowest priority wins
//! (`:136-191`).  Prompt text is never logged (`docs/DESIGN.md:120-124`): only sizes and counts.

use std::io;
use std::sync::{Arc, LazyLock};

use async_trait::async_trait;
use bytes::Bytes;
use llm_gateway_sdk::{
    ChatTemplate, CountTokensRequest, EncodeBatchRequest, InvalidUtf8, MistralInstruct, OffsetUnit, SpecialTokens, TokenizerClient, TokenizerError, TokenizerPluginClient, TokenizerPluginSpecV1,
    TruncateKeep, Usage, VocabRef,
};
use modkit::client_hub::{ClientHub, ClientScope};
use modkit::plugins::{choose_plugin_instance, GtsPluginSelector};
use modkit_security::SecurityContext;
use regex::Regex;
use serde::Serialize;
use serde_json::{json, Value};
use types_registry_sdk::{ListQuery, TypesRegistryClient};

/// the roles mistral_common's validator lets follow each role (none: not a role the mistral template counts)
fn mistral_next_roles(role: &str) -> &'static [&'static str] {
    match role {
        "system" => &["user", "assistant", "system"],
        "user" => &["assistant", "system", "user"],
        "assistant" => &["assistant", "user", "tool"],
        "tool" => &["assistant", "tool", "user"],
        _ => &[],
    }
}

// mistral_common's name and call-id rules, Python's re.match(r"^...$"): "$" also matches before a final "\n", so one trailing "\n"
// passes (the regex crate's "$" matches only at the end, hence the explicit "\n?")
static MISTRAL_NAME: LazyLock<Regex> = LazyLock::new(|| Regex::new(r"^[a-zA-Z0-9_-]{1,64}\n?$").expect("a valid pattern"));
static MISTRAL_CALL_ID: LazyLock<Regex> = LazyLock::new(|| Regex::new(r"^[a-zA-Z0-9]{9}\n?$").expect("a valid pattern"));
static NULL: Value = Value::Null;

/// one gateway message as the mistral template reads it: its text parts, its tool calls `{"name", "arguments"[, "id"]}`, its tool
/// result (call id, content) and its `prefix` flag (V7 only)
struct MistralMessage {
    role: String,
    parts: Vec<String>,
    calls: Vec<Value>,
    result: Option<(String, String)>,
    prefix: bool,
}

/// JSON as mistral_common writes it into the prompt, Python's `json.dumps(value, ensure_ascii=False)`: ", " and ": " between
/// items, keys in their order (serde_json's `preserve_order`), non-ASCII as is, floats as Python's `repr`.  Numbers that serde_json
/// reads otherwise than Python's `json` (NaN, Infinity, -0, integers past 64 bits) are the one known difference from the Python
/// mirror.
fn mistral_json(value: &Value) -> String {
    let mut out = Vec::new();
    value.serialize(&mut serde_json::Serializer::with_formatter(&mut out, PythonJson)).expect("a Value always serializes");
    String::from_utf8(out).expect("serde_json writes UTF-8")
}

/// a tool result's content as mistral_common embeds it: the JSON value when the text parses as JSON, else the text; "" is {}
fn mistral_tool_content(content: &str) -> Value {
    if content.is_empty() {
        return json!({});
    }
    serde_json::from_str(content).unwrap_or_else(|_| Value::from(content))
}

/// a tool result's content as mistral_common's V7 request normalizer leaves it: the JSON value it parses to, written again by
/// `mistral_json`, else the text as given; "" is "{}"
fn mistral_normalized_content(content: &str) -> String {
    if content.is_empty() {
        return "{}".to_owned();
    }
    serde_json::from_str::<Value>(content).map_or_else(|_| content.to_owned(), |v| mistral_json(&v))
}

struct PythonJson;

impl serde_json::ser::Formatter for PythonJson {
    fn begin_array_value<W: ?Sized + io::Write>(&mut self, writer: &mut W, first: bool) -> io::Result<()> {
        if first { Ok(()) } else { writer.write_all(b", ") }
    }

    fn begin_object_key<W: ?Sized + io::Write>(&mut self, writer: &mut W, first: bool) -> io::Result<()> {
        if first { Ok(()) } else { writer.write_all(b", ") }
    }

    fn begin_object_value<W: ?Sized + io::Write>(&mut self, writer: &mut W) -> io::Result<()> {
        writer.write_all(b": ")
    }

    fn write_f64<W: ?Sized + io::Write>(&mut self, writer: &mut W, value: f64) -> io::Result<()> {
        writer.write_all(python_float_repr(value).as_bytes())
    }
}

/// Python's `repr` of a finite float: the shortest digits that read back to it, positional when the decimal exponent is in
/// -4 ..= 15 (at least one digit after the point), else `d[.ddd]e±XX`
fn python_float_repr(x: f64) -> String {
    let sci = format!("{x:e}");                                             // shortest digits: "-1.5e-7", "1e16", "0e0"
    let (mantissa, exp) = sci.split_once('e').expect("an exponent");
    let exp: i32 = exp.parse().expect("an integer exponent");
    let (sign, mantissa) = mantissa.strip_prefix('-').map_or(("", mantissa), |m| ("-", m));
    if !(-4..16).contains(&exp) {
        return format!("{sign}{mantissa}e{}{:02}", if exp < 0 { '-' } else { '+' }, exp.abs());
    }
    let digits: String = mantissa.chars().filter(|c| *c != '.').collect();
    let point = exp + 1;                                                    // digits before the decimal point
    if point <= 0 {
        format!("{sign}0.{}{digits}", "0".repeat(point.unsigned_abs() as usize))
    } else if point as usize >= digits.len() {
        format!("{sign}{digits}{}.0", "0".repeat(point as usize - digits.len()))
    } else {
        format!("{sign}{}.{}", &digits[..point as usize], &digits[point as usize..])
    }
}

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

    /// the gateway's tools (`schemas/tools/tool.v1.schema.json`) as mistral_common's `Tool.model_dump()` without `strict`
    /// (Python mirror: `cfbpe/plugin.py:_mistral_tools`)
    fn mistral_tools(tools: &[Value]) -> Result<Vec<Value>, TokenizerError> {
        let bad = |msg: &str| TokenizerError::InvalidInput(msg.to_owned());
        tools.iter().map(|t| {
            let kind = t.get("type").and_then(Value::as_str);
            if kind != Some("unified") {
                return Err(TokenizerError::InvalidInput(format!("the mistral template counts unified tools (name, description, parameters), not {kind:?}")));
            }
            let name = t.get("name").and_then(Value::as_str);
            let description = t.get("description").and_then(Value::as_str);
            let schema = t.get("parameters").and_then(|p| p.get("json_schema")).filter(|s| s.is_object());
            let (Some(name), Some(description), Some(schema)) = (name, description, schema) else {
                return Err(bad("a unified tool has a string name and description and parameters {json_schema: object}"));
            };
            if !MISTRAL_NAME.is_match(name) {
                return Err(bad("a tool name is 1 to 64 of a-z, A-Z, 0-9, '_' and '-'"));
            }
            Ok(json!({"type": "function", "function": {"name": name, "description": description, "parameters": schema}}))
        }).collect()
    }

    /// role, text parts, tool calls, tool result and prefix flag of one gateway message (Python mirror:
    /// `cfbpe/plugin.py:_mistral_message`); other parts (images ...) are not counted here.  A call is {"name", "arguments", "id"}
    /// as mistral_common prints it (no "id" for "null").  `prefix` (Mistral's chat API: the reply continues this assistant
    /// message) is read under V7 and later.
    fn mistral_message(m: &Value, instruct: MistralInstruct) -> Result<MistralMessage, TokenizerError> {
        let bad = |msg: &str| TokenizerError::InvalidInput(msg.to_owned());
        let role = m.get("role").and_then(Value::as_str).unwrap_or("");
        if mistral_next_roles(role).is_empty() {
            return Err(TokenizerError::InvalidInput(format!("the mistral template counts system, user, assistant and tool messages, not {role:?}")));
        }
        let parts: &[Value] = m.get("content").and_then(Value::as_array).map_or(&[], Vec::as_slice);
        let of_type = |p: &&Value, t: &str| p.get("type").and_then(Value::as_str) == Some(t);
        let texts = Self::text_parts(std::slice::from_ref(m));
        let text = texts.join("\n\n");
        let prefix = match (instruct, m.get("prefix")) {
            (MistralInstruct::V7 | MistralInstruct::V11 | MistralInstruct::V13, Some(p)) => p.as_bool().filter(|&p| !p || role == "assistant").ok_or_else(|| bad("prefix is a boolean of an assistant message"))?,
            _ => false,
        };
        let results: Vec<&Value> = parts.iter().filter(|p| of_type(p, "tool_result")).map(|p| p.get("tool_result").unwrap_or(&NULL)).collect();
        let mut calls = Vec::new();
        for p in parts.iter().filter(|p| of_type(p, "tool_call")) {
            let Some(c) = p.get("tool_call").filter(|c| role == "assistant" && c.is_object()) else {
                return Err(bad("a tool_call part belongs to an assistant message"));
            };
            let (id, name, args) = (c.get("id").and_then(Value::as_str), c.get("name").and_then(Value::as_str), c.get("arguments").filter(|a| a.is_object()));
            let (Some(id), Some(name), Some(args)) = (id, name, args) else {
                return Err(bad("a tool call has a string id and name and object arguments"));
            };
            if id != "null" && !MISTRAL_CALL_ID.is_match(id) {
                return Err(bad("a tool call id is 9 of a-z, A-Z and 0-9"));
            }
            if id == "null" && instruct == MistralInstruct::V13 {
                return Err(bad("a tool call has an id under instruct V13"));
            }
            if !MISTRAL_NAME.is_match(name) {
                return Err(bad("a tool call's name is 1 to 64 of a-z, A-Z, 0-9, '_' and '-'"));
            }
            let mut call = json!({"name": name, "arguments": args});
            if id != "null" {
                call["id"] = Value::from(id);
            }
            calls.push(call);
        }
        if instruct == MistralInstruct::V3 && role == "assistant" && text.is_empty() == calls.is_empty() {       // (V7: text, calls or both, once merged)
            return Err(bad(if text.is_empty() { "an assistant message without text or tool calls" } else { "an assistant message holds text or tool calls, one of the two" }));
        }
        if (role == "tool") == results.is_empty() {
            return Err(bad(if results.is_empty() { "a tool message holds a tool_result part" } else { "a tool_result part belongs to a tool message" }));
        }
        let mut result = None;
        if role == "tool" {
            let r = results[0];
            let (content, id) = (r.get("content").and_then(Value::as_str), r.get("tool_call_id").and_then(Value::as_str));
            let (Some(content), Some(id), 1, true) = (content, id, results.len(), text.is_empty()) else {
                return Err(bad("a tool message holds one tool_result {tool_call_id: string, content: string} and no text"));
            };
            if !MISTRAL_CALL_ID.is_match(id) {
                return Err(bad("a tool result's tool_call_id is 9 of a-z, A-Z and 0-9"));
            }
            result = Some((id.to_owned(), content.to_owned()));
        }
        Ok(MistralMessage { role: role.to_owned(), parts: texts, calls, result, prefix })
    }

    /// MistralRequestValidatorV13's check of tool results against the calls they answer (V11 and V13), on messages
    /// `mistral_message` read: the first message is not checked (Python mirror: `cfbpe/plugin.py:_check_mistral_call_ids`)
    fn check_mistral_call_ids(msgs: &[MistralMessage]) -> Result<(), TokenizerError> {
        let bad = |msg: String| TokenizerError::InvalidInput(msg);
        let (mut expected, mut answered) = (std::collections::HashSet::new(), std::collections::HashSet::new());
        for m in &msgs[1..] {
            match m.role.as_str() {
                "tool" => {
                    let id = m.result.as_ref().expect("a tool message has its result").0.as_str();
                    if answered.contains(id) {
                        return Err(bad(format!("two tool results answer the call {id:?}")));
                    }
                    if !expected.contains(id) {
                        return Err(bad(format!("a tool result answers {id:?}, not a call of the assistant message before it")));
                    }
                    answered.insert(id);
                }
                "assistant" => {
                    if answered.len() != expected.len() {
                        return Err(bad("an assistant message follows tool calls without a tool result each".to_owned()));
                    }
                    (expected, answered) = (std::collections::HashSet::new(), std::collections::HashSet::new());
                    for c in &m.calls {
                        let id = c.get("id").and_then(Value::as_str).unwrap_or("null");
                        if !expected.insert(id) {
                            return Err(bad(format!("two tool calls of one assistant message have the id {id:?}")));
                        }
                    }
                }
                _ => {}
            }
        }
        Ok(())
    }

    /// the texts and control tokens of a conversation under V7, V11 or V13, on messages `mistral_message` read and the caller
    /// checked (Python mirror: `cfbpe/plugin.py:_mistral_v7_texts`)
    fn mistral_v7_texts(msgs: Vec<MistralMessage>, tool_defs: Vec<Value>, instruct: MistralInstruct) -> Result<(Vec<String>, u64), TokenizerError> {
        let prefix = msgs.last().is_some_and(|m| m.prefix);
        let mut turns: Vec<MistralMessage> = Vec::new();                    // after merging
        let mut prev = String::new();
        for m in msgs {
            let role = m.role.clone();
            if (role == "user" || role == "assistant") && role == prev {
                let last = turns.last_mut().expect("a turn of this role");
                last.parts.extend(m.parts);
                last.calls.extend(m.calls);
            } else {
                turns.push(m);
            }
            prev = role;
        }
        let tools_at = if instruct == MistralInstruct::V13 {
            turns.iter().position(|t| t.role == "user")
        } else {
            turns.iter().rposition(|t| t.role == "user")
        };
        let n_turns = turns.len();
        let (mut texts, mut fixed) = (Vec::new(), 1u64);                    // <s>
        let mut tool_defs = Some(tool_defs);
        for (i, t) in turns.into_iter().enumerate() {
            let text = t.parts.join("\n\n");
            match t.role.as_str() {
                "system" => {
                    texts.push(text);
                    fixed += 2;                                             // [SYSTEM_PROMPT] [/SYSTEM_PROMPT]
                }
                "user" => {
                    if Some(i) == tools_at {
                        if let Some(defs) = tool_defs.take().filter(|d| !d.is_empty()) {
                            texts.push(mistral_json(&Value::Array(defs)));
                            fixed += 2;                                     // [AVAILABLE_TOOLS] [/AVAILABLE_TOOLS]
                        }
                    }
                    texts.push(text);
                    fixed += 2;                                             // [INST] [/INST]
                }
                "assistant" => {
                    if text.is_empty() && t.calls.is_empty() {
                        return Err(TokenizerError::InvalidInput("an assistant message without text or tool calls (also once merged)".to_owned()));
                    }
                    texts.push(text.trim_end_matches(' ').to_owned());
                    if instruct == MistralInstruct::V7 && !t.calls.is_empty() {
                        texts.push(mistral_json(&Value::Array(t.calls)));
                        fixed += 1;                                         // [TOOL_CALLS]
                    } else {
                        for c in t.calls {
                            texts.push(c["name"].as_str().expect("a call has a name").to_owned());
                            if let (MistralInstruct::V11, Some(id)) = (instruct, c.get("id").and_then(Value::as_str)) {
                                texts.push(id.to_owned());
                                fixed += 1;                                 // [CALL_ID]
                            }
                            texts.push(mistral_json(&c["arguments"]));
                            fixed += 2;                                     // [TOOL_CALLS] [ARGS]
                        }
                    }
                    if !(prefix && i == n_turns - 1) {
                        fixed += 1;                                         // </s>
                    }
                }
                _ => {
                    let (id, content) = t.result.expect("a tool message has its result");
                    if instruct == MistralInstruct::V13 {
                        texts.push(mistral_normalized_content(&content));
                        fixed += 2;                                         // [TOOL_RESULTS] [/TOOL_RESULTS]
                    } else {
                        texts.push(id);
                        texts.push(mistral_normalized_content(&content));
                        fixed += 3;                                         // [TOOL_RESULTS] [TOOL_CONTENT] [/TOOL_RESULTS]
                    }
                }
            }
        }
        Ok((texts, fixed))
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
        self.count_chat_tokens_with_tools(ctx, model, messages, &[], template).await
    }

    async fn count_chat_tokens_with_tools(&self, ctx: &SecurityContext, model: &str, messages: &[Value], tools: &[Value], template: &ChatTemplate)
        -> Result<Usage, TokenizerError> {
        // every stretch of ordinary text of the whole request, tool JSON included, goes to the device in ONE batch; control tokens
        // count one each
        if !tools.is_empty() && !matches!(template, ChatTemplate::Mistral { .. }) {
            return Err(TokenizerError::InvalidInput("only the mistral chat template counts tools".to_owned()));
        }
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
            ChatTemplate::Mistral { instruct } => {
                let bad = |msg: &str| TokenizerError::InvalidInput(msg.to_owned());
                let mut tool_defs = Self::mistral_tools(tools)?;
                if messages.is_empty() {
                    return Err(bad("a conversation for the mistral template has at least one message"));
                }
                let msgs = messages.iter().map(|m| Self::mistral_message(m, *instruct)).collect::<Result<Vec<_>, _>>()?;
                let roles: Vec<String> = msgs.iter().map(|m| m.role.clone()).collect();
                if msgs[..msgs.len() - 1].iter().any(|m| m.prefix) {
                    return Err(bad("an assistant message with prefix is the last message"));
                }
                if roles.len() == 1 && !matches!(roles[0].as_str(), "user" | "system") {
                    return Err(bad("a conversation of one message for the mistral template is a user or system message"));
                }
                if roles.len() > 1 && roles[roles.len() - 1] == "assistant" && !msgs[msgs.len() - 1].prefix {
                    return Err(bad(if *instruct != MistralInstruct::V3 {
                        "a conversation for the mistral template ends with a user or tool message or an assistant message with prefix"
                    } else {
                        "a conversation for the mistral template ends with a user or tool message"
                    }));
                }
                for w in roles.windows(2) {
                    if !mistral_next_roles(&w[0]).contains(&w[1].as_str()) {
                        return Err(TokenizerError::InvalidInput(format!("a message of role {:?} follows one of role {:?}", w[1], w[0])));
                    }
                }
                if matches!(instruct, MistralInstruct::V11 | MistralInstruct::V13) {
                    Self::check_mistral_call_ids(&msgs)?;
                } else {
                    let mut pending = 0i64;                                 // tool messages the last tool-calling assistant message still waits for
                    for m in &msgs[1..] {
                        match m.role.as_str() {
                            "tool" => pending -= 1,
                            "assistant" if pending != 0 => return Err(bad("an assistant message follows tool calls without exactly one tool message each")),
                            "assistant" => pending = m.calls.len() as i64,
                            _ => {}
                        }
                    }
                }
                if *instruct != MistralInstruct::V3 {
                    (texts, fixed) = Self::mistral_v7_texts(msgs, tool_defs, *instruct)?;
                } else {
                    // V3: the texts are each message's text parts joined with "\n\n"
                    let system = msgs.iter().filter(|m| m.role == "system").map(|m| m.parts.join("\n\n")).filter(|t| !t.is_empty()).collect::<Vec<_>>().join("\n\n");
                    let mut turns: Vec<(String, String, Vec<Value>, Option<(String, String)>)> = Vec::new();   // (role, text, calls, result) after merging
                    let mut prev = String::new();
                    for m in msgs {
                        let role = m.role.clone();
                        let text = m.parts.join("\n\n");
                        if (role == "user" || role == "assistant") && role == prev {
                            let last = turns.last_mut().expect("a turn of this role");
                            if m.calls.is_empty() {                         // (a message with tool calls has no text to merge)
                                last.1.push_str("\n\n");
                                last.1.push_str(&text);
                            }
                            last.2.extend(m.calls);
                            if !last.1.is_empty() && !last.2.is_empty() {
                                return Err(bad("merged assistant messages hold both text and tool calls"));
                            }
                        } else if role != "system" {
                            turns.push((role.clone(), text, m.calls, m.result));
                        }
                        prev = role;
                    }
                    if turns.first().map_or(true, |t| t.0 != "user") {
                        turns.insert(0, ("user".to_owned(), String::new(), Vec::new(), None));
                    }
                    let last_user = turns.iter().rposition(|t| t.0 == "user").expect("a user turn");
                    fixed = 1;                                              // <s>
                    for (i, (role, text, calls, result)) in turns.into_iter().enumerate() {
                        match role.as_str() {
                            "user" => {
                                if i == last_user && !tool_defs.is_empty() {
                                    texts.push(mistral_json(&Value::Array(std::mem::take(&mut tool_defs))));
                                    fixed += 2;                             // [AVAILABLE_TOOLS] [/AVAILABLE_TOOLS]
                                }
                                texts.push(if i == last_user && !system.is_empty() { format!("{system}\n\n{text}") } else { text });
                                fixed += 2;                                 // [INST] [/INST]
                            }
                            "assistant" if !calls.is_empty() => {
                                texts.push(mistral_json(&Value::Array(calls)));
                                fixed += 2;                                 // [TOOL_CALLS] </s>
                            }
                            "assistant" => {
                                texts.push(text.trim_end_matches(' ').to_owned());
                                fixed += 1;                                 // </s>
                            }
                            _ => {
                                let (id, content) = result.expect("a tool message has its result");
                                texts.push(mistral_json(&json!({"content": mistral_tool_content(&content), "call_id": id})));
                                fixed += 2;                                 // [TOOL_RESULTS] [/TOOL_RESULTS]
                            }
                        }
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
