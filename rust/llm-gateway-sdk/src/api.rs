//! Public API trait for consumers of the gateway's tokenizer (unscoped in `ClientHub`).

use async_trait::async_trait;
use modkit_security::SecurityContext;
use serde_json::Value;

use crate::error::TokenizerError;
use crate::models::{ChatTemplate, OffsetUnit, SpecialTokens, TruncateKeep, Usage};

#[async_trait]
pub trait TokenizerClient: Send + Sync {
    /// `encode_ordinary` of every text under the vocabulary of `model` (canonical id or vocabulary name).
    async fn encode(&self, ctx: &SecurityContext, model: &str, texts: &[String]) -> Result<Vec<Vec<u32>>, TokenizerError>;

    /// Per text: the ids and each token's `[start, end)` span in `unit`: bytes of the text's UTF-8, code points, or UTF-16 code
    /// units (cut to a context window or into chunks at a span boundary).  In a character unit, byte tokens of one character share
    /// its start, so some spans are empty; the spans still tile the text.
    async fn encode_with_offsets(&self, ctx: &SecurityContext, model: &str, texts: &[String], unit: OffsetUnit)
        -> Result<Vec<(Vec<u32>, Vec<[u64; 2]>)>, TokenizerError>;

    /// Fit texts into a context window: per text, (the kept text, its tokens, the tokens of the whole text).  `max_tokens`: one
    /// budget per text; `keep`: the first or the last tokens.  The cut is at a character boundary, so the kept text is valid UTF-8.
    async fn truncate(&self, ctx: &SecurityContext, model: &str, texts: &[String], max_tokens: &[u32], keep: TruncateKeep)
        -> Result<Vec<(String, u32, u32)>, TokenizerError>;

    /// Split texts into chunks of at most `max_tokens` tokens that overlap by `overlap` tokens (a RAG splitter's chunk_size /
    /// chunk_overlap, an embedding endpoint's long inputs): per text, its chunks.  The cuts are at character boundaries, so every
    /// chunk is valid UTF-8; with no overlap the chunks join back into the text.
    async fn chunk(&self, ctx: &SecurityContext, model: &str, texts: &[String], max_tokens: u32, overlap: u32)
        -> Result<Vec<Vec<String>>, TokenizerError>;

    /// tiktoken's `encode(text, allowed_special = …, disallowed_special = …)`.
    async fn encode_with_special(&self, ctx: &SecurityContext, model: &str, texts: &[String], special: &SpecialTokens)
        -> Result<Vec<Vec<u32>>, TokenizerError>;

    /// `Usage.input_tokens` of one chat request: the sum over its `TextContent.text` parts
    /// (`schemas/core/message.v1.schema.json`, `schemas/content/text_content.v1.schema.json`); `messages` are the request's
    /// message objects as JSON.
    async fn count_tokens(&self, ctx: &SecurityContext, model: &str, messages: &[Value]) -> Result<Usage, TokenizerError>;

    /// Pre-call estimate against a remaining budget (`docs/DESIGN.md:833-855`).
    /// `Usage.input_tokens` as the provider counts it: content AND the framing of `template`
    async fn count_chat_tokens(&self, ctx: &SecurityContext, model: &str, messages: &[Value], template: &ChatTemplate) -> Result<Usage, TokenizerError>;

    /// `count_chat_tokens` of a request that also carries `tools` (`schemas/core/request.v1.schema.json`, `tools`): the
    /// `ChatTemplate::Mistral` kind counts the tool definitions as mistral_common does; the other kinds refuse a non-empty `tools`
    /// with `InvalidInput`.  This default counts requests without tools only.
    async fn count_chat_tokens_with_tools(&self, ctx: &SecurityContext, model: &str, messages: &[Value], tools: &[Value], template: &ChatTemplate)
        -> Result<Usage, TokenizerError> {
        if !tools.is_empty() {
            return Err(TokenizerError::InvalidInput("this tokenizer client does not count tools".to_owned()));
        }
        self.count_chat_tokens(ctx, model, messages, template).await
    }

    async fn check_budget(&self, ctx: &SecurityContext, model: &str, messages: &[Value], remaining_tokens: u64) -> Result<bool, TokenizerError>;
}
