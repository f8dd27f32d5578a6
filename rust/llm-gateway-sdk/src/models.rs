//! Request / response models of the tokenizer API.
//!
//! A batch is ONE packed buffer: the UTF-8 bytes of all prompts back to back plus `n + 1` byte offsets — the layout the device
//! path reads with coalesced 16-byte loads; requests of many tenants share a batch, each prompt naming its vocabulary.

use std::collections::BTreeMap;

use bytes::Bytes;
use serde::{Deserialize, Serialize};

/// Names a vocabulary: a registry name (`cl100k_base`) or a model-registry canonical id (`openai::gpt-4`,
/// `{provider_slug}::{provider_model_id}`, `modules/model-registry/docs/PRD.md:197`).
#[derive(Debug, Clone, PartialEq, Eq, Hash, Serialize, Deserialize)]
pub struct VocabRef(pub String);

#[derive(Debug, Clone)]
pub struct EncodeBatchRequest {
    pub vocab: VocabRef,
    /// packed UTF-8 of all prompts
    pub bytes: Bytes,
    /// `n + 1` offsets into `bytes`, `offsets[0] == 0`, non-decreasing
    pub offsets: Vec<u64>,
    /// multi-tenant batches: one vocabulary per prompt (overrides `vocab`)
    pub vocabs_per_prompt: Option<Vec<VocabRef>>,
    /// with it, `vocabs_per_prompt` lists the DISTINCT vocabularies and `vocab_index[i]` picks prompt i's
    /// (a 65 536-prompt batch carries three names and 64 KiB of indices, not 65 536 strings)
    pub vocab_index: Option<Vec<u8>>,
    /// also return every token's byte offset within its prompt (`EncodeBatchResponse::starts`); `false` for a plain encode
    pub with_starts: bool,
}

#[derive(Debug, Clone, Default, Serialize, Deserialize)]
pub struct EncodeBatchResponse {
    /// dense id stream of all prompts (tiktoken `encode_ordinary` semantics, bit-exact)
    pub ids: Vec<u32>,
    /// `n + 1` offsets into `ids`
    pub offsets: Vec<u64>,
    pub counts: Vec<u32>,
    /// with `with_starts`: one entry per id, the byte offset of the token within its prompt (token k of prompt i covers
    /// `bytes[offsets_in[i] + starts[k] .. offsets_in[i] + end)`, `end` the next start or the prompt's length)
    #[serde(default, skip_serializing_if = "Option::is_none")]
    pub starts: Option<Vec<u32>>,
}

#[derive(Debug, Clone)]
pub struct CountTokensRequest {
    pub vocab: VocabRef,
    pub bytes: Bytes,
    pub offsets: Vec<u64>,
    pub vocabs_per_prompt: Option<Vec<VocabRef>>,
    pub vocab_index: Option<Vec<u8>>,
}

#[derive(Debug, Clone)]
pub struct DecodeBatchRequest {
    pub vocab: VocabRef,
    pub ids: Vec<u32>,
    pub offsets: Vec<u64>,
    pub vocabs_per_prompt: Option<Vec<VocabRef>>,
    pub vocab_index: Option<Vec<u8>>,
}

#[derive(Debug, Clone, Default)]
pub struct DecodeBatchResponse {
    /// the sequences' bytes back to back (tiktoken `decode_bytes`: not necessarily valid UTF-8)
    pub bytes: Vec<u8>,
    pub offsets: Vec<u64>,
}

/// Special tokens of a vocabulary and which of them a request may spell out (tiktoken `Encoding.encode`: by default none is
/// allowed and every one is disallowed, so user text that spells a control token is refused, not turned into one).
#[derive(Debug, Clone, Default)]
pub struct SpecialTokens {
    pub ids: BTreeMap<String, u32>,
    pub allowed: Vec<String>,
    pub disallow_all_others: bool,
}

/// How a provider frames a list of chat messages into the token stream it bills as `Usage.input_tokens`
/// (Python mirror: `cfbpe/plugin.py:ChatTemplate`).  Message content is always ordinary text: a message that spells a control
/// token costs the pieces of that spelling and never becomes the control token.
#[derive(Debug, Clone, PartialEq, Eq)]
pub enum ChatTemplate {
    /// a fixed number of framing tokens a message (OpenAI ChatML accounting: 3 a message, 1 a name, 3 to prime the reply)
    Overhead { tokens_per_message: u32, tokens_per_name: u32, reply_priming: u32 },
    /// the conversation rendered to text around control tokens (Llama 3, Mistral): `bos`, then per message
    /// `message_prefix` (with `{role}`) + content + `message_suffix`, then `generation_prompt`; every string of
    /// `special_tokens` counts one token, the text between two of them is tokenised as ONE stretch of ordinary text
    Rendered { bos: String, message_prefix: String, message_suffix: String, generation_prompt: String, special_tokens: Vec<String> },
}

/// `gts.x.llmgw.core.usage.v1~` (`llm-gateway-sdk/schemas/core/usage.v1.schema.json:8-12`)
#[derive(Debug, Clone, Copy, Default, PartialEq, Eq, Serialize, Deserialize)]
pub struct Usage {
    pub input_tokens: u64,
    pub output_tokens: u64,
}
