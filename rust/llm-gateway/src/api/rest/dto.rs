//! REST DTOs of `POST /llm-gateway/v1/tokenize`, `POST /llm-gateway/v1/count-tokens`, `POST /llm-gateway/v1/truncate` and
//! `POST /llm-gateway/v1/chunk`.

use schemars::JsonSchema;
use serde::{Deserialize, Serialize};

#[derive(Debug, Deserialize, JsonSchema)]
#[serde(deny_unknown_fields)]
pub struct TokenizeRequest {
    /// canonical model id (`{provider_slug}::{provider_model_id}`) or vocabulary name
    pub model: String,
    /// texts to tokenize (one entry per prompt)
    pub texts: Vec<String>,
    /// return the ids as well as the counts
    #[serde(default)]
    pub return_ids: bool,
    /// return each token's `[start, end)` span in its text as well
    #[serde(default)]
    pub return_offsets: bool,
    /// the unit of `offsets`: `byte` (UTF-8, the default), `codepoint` (Python string indices) or `utf16` (JavaScript, Java and C#
    /// string indices).  In a character unit, byte tokens of one character share its start, so some spans are empty.
    #[serde(default)]
    pub offset_unit: llm_gateway_sdk::OffsetUnit,
}

#[derive(Debug, Serialize, JsonSchema)]
pub struct TokenizeResponse {
    /// token count of every text (`Usage.input_tokens` is their sum)
    pub counts: Vec<u32>,
    pub input_tokens: u64,
    /// token ids of every text, when asked for
    #[serde(skip_serializing_if = "Option::is_none")]
    pub ids: Option<Vec<Vec<u32>>>,
    /// span of every token of every text in `offset_unit`, when asked for
    #[serde(skip_serializing_if = "Option::is_none")]
    pub offsets: Option<Vec<Vec<[u64; 2]>>>,
}

/// A token budget: one for every text, or one per text.
#[derive(Debug, Deserialize, JsonSchema)]
#[serde(untagged)]
pub enum MaxTokens {
    All(u32),
    PerText(Vec<u32>),
}

#[derive(Debug, Deserialize, JsonSchema)]
#[serde(deny_unknown_fields)]
pub struct TruncateRequest {
    /// canonical model id or vocabulary name
    pub model: String,
    /// texts to fit into the budget (one entry per prompt)
    pub texts: Vec<String>,
    /// the token budget
    pub max_tokens: MaxTokens,
    /// `head` keeps the first tokens (a document, retrieved context), `tail` the last ones (a chat history); default `head`
    #[serde(default)]
    pub keep: llm_gateway_sdk::TruncateKeep,
}

#[derive(Debug, Serialize, JsonSchema)]
pub struct TruncateResponse {
    /// every text cut at a token boundary of its whole encoding, moved to a character boundary (valid UTF-8)
    pub texts: Vec<String>,
    /// tokens of every text's encoding wholly inside the kept text: the budget, or one to three fewer when the cut moved
    pub kept_tokens: Vec<u32>,
    /// token count of every whole text, as `counts` of `/tokenize`
    pub counts: Vec<u32>,
}

#[derive(Debug, Deserialize, JsonSchema)]
#[serde(deny_unknown_fields)]
pub struct ChunkRequest {
    /// canonical model id or vocabulary name
    pub model: String,
    /// texts to split (one entry per document)
    pub texts: Vec<String>,
    /// the most tokens a chunk holds (>= 1)
    pub max_tokens: u32,
    /// tokens consecutive chunks share (< max_tokens); default 0
    #[serde(default)]
    pub overlap: u32,
}

#[derive(Debug, Serialize, JsonSchema)]
pub struct ChunkResponse {
    /// every text's chunks, cut at token boundaries of its whole encoding moved to character boundaries (valid UTF-8)
    pub chunks: Vec<Vec<String>>,
    /// every chunk's `[begin, end)` byte span in its text's UTF-8, in the order of `chunks`
    pub spans: Vec<Vec<[u32; 2]>>,
    /// token count of every whole text, as `counts` of `/tokenize`
    pub counts: Vec<u32>,
}

/// How the provider frames the messages (`llm_gateway_sdk::ChatTemplate`): a template's name (`ChatTemplate::named`:
/// "openai-chatml", "mistral-v3", "mistral-v7", "mistral-v11", "mistral-v13", "llama3-instruct") or the template spelled out;
/// absent: content only.
#[derive(Debug, Deserialize, JsonSchema)]
#[serde(untagged)]
pub enum TemplateDto {
    Named(String),
    Spec(ChatTemplateDto),
}

#[derive(Debug, Deserialize, JsonSchema)]
#[serde(tag = "kind", rename_all = "snake_case", deny_unknown_fields)]
pub enum ChatTemplateDto {
    Overhead { tokens_per_message: u32, tokens_per_name: u32, reply_priming: u32 },
    Rendered { bos: String, message_prefix: String, message_suffix: String, generation_prompt: String, special_tokens: Vec<String> },
    Mistral {
        /// mistral_common's instruct tokenizer version, 3, 7, 11 or 13; absent: 3
        #[serde(default = "mistral_instruct_default")]
        instruct_version: u8,
    },
}

fn mistral_instruct_default() -> u8 {
    3
}

#[derive(Debug, Deserialize, JsonSchema)]
#[serde(deny_unknown_fields)]
pub struct CountTokensRequest {
    /// canonical model id or vocabulary name
    pub model: String,
    /// chat messages (`llm-gateway-sdk/schemas/core/message.v1.schema.json`): only their `text` content parts are counted
    pub messages: Vec<serde_json::Value>,
    /// the provider's framing; absent: the sum over the text parts
    pub template: Option<TemplateDto>,
    /// the request's tools (`llm-gateway-sdk/schemas/tools/tool.v1.schema.json`): counted by the `mistral` template (unified tools
    /// only); any other template, or none, refuses them
    #[serde(default)]
    pub tools: Vec<serde_json::Value>,
}

/// `gts.x.llmgw.core.usage.v1~` restricted to what a pre-call estimate knows
#[derive(Debug, Serialize, JsonSchema)]
pub struct CountTokensResponse {
    pub input_tokens: u64,
}
