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
    /// with `with_starts`: the unit of the starts (`OffsetUnit::Byte` for byte offsets; a character unit also fills
    /// `EncodeBatchResponse::lens`)
    pub starts_unit: OffsetUnit,
    /// bytes that are not valid UTF-8: `Reject` fails the request, `Replace` encodes every prompt as `String::from_utf8_lossy`
    /// would have it and fills `EncodeBatchResponse::replaced` (not with `with_starts`)
    pub invalid_utf8: InvalidUtf8,
}

/// What a request does with bytes that are not valid UTF-8 (`include/cfbpe.h`, `cfbpe_encode_batch_lossy`).
#[derive(Debug, Clone, Copy, PartialEq, Eq, Default, Serialize, Deserialize, schemars::JsonSchema)]
#[serde(rename_all = "lowercase")]
pub enum InvalidUtf8 {
    /// fail the request (tiktoken only accepts valid text)
    #[default]
    Reject,
    /// replace each maximal subpart of an ill-formed sequence with U+FFFD (`String::from_utf8_lossy`, Python's
    /// `decode("utf-8", "replace")`, the WHATWG decoder)
    Replace,
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
    /// with a character `starts_unit`: every prompt's length in that unit (closes the last token's span)
    #[serde(default, skip_serializing_if = "Option::is_none")]
    pub lens: Option<Vec<u32>>,
    /// with `InvalidUtf8::Replace`: every prompt's U+FFFD inserted by the repair (0: valid UTF-8)
    #[serde(default, skip_serializing_if = "Option::is_none")]
    pub replaced: Option<Vec<u32>>,
}

/// What a token start counts (`include/cfbpe.h`, `cfbpe_encode_batch_char_starts`).
#[derive(Debug, Clone, Copy, PartialEq, Eq, Default, Serialize, Deserialize, schemars::JsonSchema)]
#[serde(rename_all = "lowercase")]
pub enum OffsetUnit {
    /// bytes of the UTF-8 text
    #[default]
    Byte,
    /// Unicode code points: Python `str` indices, tiktoken's `decode_with_offsets`
    Codepoint,
    /// UTF-16 code units (a code point >= U+10000 counts 2): JavaScript, Java and C# string indices
    Utf16,
}

/// The unit-start contract on the host, from every token's byte start (`EncodeBatchResponse::starts`): `(starts, len)` of prompt
/// `prompt` (its UTF-8 bytes, valid), whose tokens start at byte `byte_starts`, in `unit`.  A token's start is the number of units
/// before the character that holds its first byte; `len` is the prompt's length in units.
pub fn unit_starts(prompt: &[u8], byte_starts: &[u32], unit: OffsetUnit) -> (Vec<u32>, u32) {
    if unit == OffsetUnit::Byte {
        return (byte_starts.to_vec(), prompt.len() as u32);
    }
    let weight = |b: u8| -> u32 {
        if b & 0xC0 == 0x80 { 0 } else if unit == OffsetUnit::Utf16 && b >= 0xF0 { 2 } else { 1 }
    };
    // units[x] = units of the characters that start before byte x
    let mut units = Vec::with_capacity(prompt.len() + 1);
    units.push(0u32);
    for &b in prompt {
        units.push(units.last().copied().unwrap_or(0) + weight(b));
    }
    let starts = byte_starts.iter().map(|&x| {
        let mut x = x as usize;
        while x > 0 && x < prompt.len() && prompt[x] & 0xC0 == 0x80 { x -= 1; }
        units[x]
    }).collect();
    (starts, units[prompt.len()])
}

/// Which tokens a truncation keeps.
#[derive(Debug, Clone, Copy, PartialEq, Eq, Default, Serialize, Deserialize, schemars::JsonSchema)]
#[serde(rename_all = "lowercase")]
pub enum TruncateKeep {
    /// the first ones: a long document or retrieved context
    #[default]
    Head,
    /// the last ones: a chat history
    Tail,
}

/// Where every prompt of a batch is cut to its token budget, one entry per prompt (`include/cfbpe.h`, `cfbpe_truncate_batch`).
/// For prompt i with tokens t_0 .. t_{c-1} and k = min(budget, c): `Head` keeps `bytes[0 .. cut)`, cut = the character start at or
/// before the end of t_{k-1}; `Tail` keeps `bytes[cut .. len)`, cut = the character start at or after the start of t_{c-k}.  The
/// boundaries are those of the WHOLE prompt's encoding; encoding the kept text again may give other ids (BPE is not prefix-stable).
#[derive(Debug, Clone, Default, Serialize, Deserialize)]
pub struct TruncateBatchResponse {
    /// byte position of the cut within the prompt (always a character boundary: the kept text is valid UTF-8)
    pub cut: Vec<u32>,
    /// tokens of the prompt's encoding wholly inside the kept text: k, or fewer when the cut moved off a token boundary
    pub kept: Vec<u32>,
    /// tokens of the whole prompt
    pub counts: Vec<u32>,
}

/// The truncation contract on the host, from every token's start (`EncodeBatchResponse::starts`): `(cut, kept)` of prompt
/// `prompt` (its UTF-8 bytes), whose tokens start at `starts`.
pub fn truncate_cut(prompt: &[u8], starts: &[u32], budget: u32, keep: TruncateKeep) -> (u32, u32) {
    let (c, len) = (starts.len(), prompt.len());
    let k = (budget as usize).min(c);
    let j = if keep == TruncateKeep::Tail { c - k } else { k };
    let mut x = if j < c { starts[j] as usize } else { len };
    let cont = |b: u8| b & 0xC0 == 0x80;
    match keep {
        TruncateKeep::Tail => {
            while x < len && cont(prompt[x]) { x += 1; }
            (x as u32, (c - starts.partition_point(|&s| (s as usize) < x)) as u32)
        }
        TruncateKeep::Head => {
            while x > 0 && x < len && cont(prompt[x]) { x -= 1; }
            let ends = |i: usize| if i + 1 < c { starts[i + 1] as usize } else { len };
            ((x as u32), (0..c).take_while(|&i| ends(i) <= x).count() as u32)
        }
    }
}

/// Every prompt of a batch cut into chunks of at most N tokens (`include/cfbpe.h`, `cfbpe_chunk_batch`).  Windows of N tokens start
/// every N - overlap tokens until one reaches the last token; chunk k covers tokens [a, e) and its bytes are [F(a), F(e)), F(j) =
/// the character start at or before token j's start, F(c) = the prompt's length.  With no overlap the chunks tile the prompt.
#[derive(Debug, Clone, Default, Serialize, Deserialize)]
pub struct ChunkBatchResponse {
    /// `[begin, end)` of every chunk within its prompt (always character boundaries: every chunk is valid UTF-8)
    pub spans: Vec<[u32; 2]>,
    /// prompt i's chunks are `spans[chunk_offsets[i] .. chunk_offsets[i + 1]]` (n + 1 entries)
    pub chunk_offsets: Vec<u64>,
    /// tokens of every whole prompt
    pub counts: Vec<u32>,
}

/// The chunking contract on the host, from every token's start (`EncodeBatchResponse::starts`): the `[begin, end)` spans of prompt
/// `prompt` (its UTF-8 bytes), whose tokens start at `starts`.  `chunk_tokens` >= 1, `overlap_tokens` < `chunk_tokens`.
pub fn chunk_spans(prompt: &[u8], starts: &[u32], chunk_tokens: u32, overlap_tokens: u32) -> Vec<[u32; 2]> {
    let (c, len) = (starts.len(), prompt.len());
    let (n, step) = (chunk_tokens as usize, (chunk_tokens - overlap_tokens) as usize);
    let floor = |j: usize| -> u32 {
        if j >= c {
            return len as u32;
        }
        let mut x = starts[j] as usize;
        while x > 0 && x < len && prompt[x] & 0xC0 == 0x80 { x -= 1; }
        x as u32
    };
    let k = if c == 0 { 0 } else if c <= n { 1 } else { 1 + (c - n).div_ceil(step) };
    (0..k).map(|q| [floor(q * step), floor((q * step + n).min(c))]).collect()
}

#[derive(Debug, Clone)]
pub struct CountTokensRequest {
    pub vocab: VocabRef,
    pub bytes: Bytes,
    pub offsets: Vec<u64>,
    pub vocabs_per_prompt: Option<Vec<VocabRef>>,
    pub vocab_index: Option<Vec<u8>>,
    /// as `EncodeBatchRequest::invalid_utf8`
    pub invalid_utf8: InvalidUtf8,
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
