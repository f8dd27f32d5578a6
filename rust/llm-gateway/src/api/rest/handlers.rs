//! Handlers: translate DTOs, map `TokenizerError` to RFC 9457 `Problem` (`libs/modkit-errors/src/problem.rs:41-53`).

use std::sync::Arc;

use axum::{Extension, Json};
use llm_gateway_sdk::{ChatTemplate, TokenizerClient, TokenizerError};
use modkit_errors::Problem;
use modkit_security::SecurityContext;

use crate::api::rest::dto::{
    ChatTemplateDto, ChunkRequest, ChunkResponse, CountTokensRequest, CountTokensResponse, MaxTokens, TokenizeRequest, TokenizeResponse, TruncateRequest, TruncateResponse,
};
use crate::domain::service::TokenizerService;

fn problem(e: TokenizerError) -> Problem {
    let (status, title) = match &e {
        TokenizerError::InvalidInput(_) => (http::StatusCode::BAD_REQUEST, "Invalid input"),
        TokenizerError::VocabNotFound { .. } => (http::StatusCode::NOT_FOUND, "Vocabulary not found"),
        TokenizerError::NoPluginAvailable | TokenizerError::ServiceUnavailable(_) => (http::StatusCode::SERVICE_UNAVAILABLE, "Tokenizer unavailable"),
        TokenizerError::Internal(_) => (http::StatusCode::INTERNAL_SERVER_ERROR, "Internal error"),
    };
    Problem::new(status, title, e.to_string())
}

pub async fn tokenize(
    Extension(ctx): Extension<SecurityContext>,
    Extension(service): Extension<Arc<TokenizerService>>,
    Json(req): Json<TokenizeRequest>,
) -> Result<Json<TokenizeResponse>, Problem> {
    // only sizes are logged, never the text (docs/DESIGN.md:120-124)
    tracing::debug!(model = %req.model, texts = req.texts.len(), bytes = req.texts.iter().map(String::len).sum::<usize>(), "tokenize");
    let (ids, offsets) = if req.return_offsets {
        let r = service.encode_with_offsets(&ctx, &req.model, &req.texts, req.offset_unit).await.map_err(problem)?;
        let (ids, spans): (Vec<_>, Vec<_>) = r.into_iter().unzip();
        (ids, Some(spans))
    } else {
        (service.encode(&ctx, &req.model, &req.texts).await.map_err(problem)?, None)
    };
    let counts: Vec<u32> = ids.iter().map(|v| v.len() as u32).collect();
    let input_tokens = counts.iter().map(|c| u64::from(*c)).sum();
    Ok(Json(TokenizeResponse { counts, input_tokens, ids: req.return_ids.then_some(ids), offsets }))
}

pub async fn truncate(
    Extension(ctx): Extension<SecurityContext>,
    Extension(service): Extension<Arc<TokenizerService>>,
    Json(req): Json<TruncateRequest>,
) -> Result<Json<TruncateResponse>, Problem> {
    tracing::debug!(model = %req.model, texts = req.texts.len(), bytes = req.texts.iter().map(String::len).sum::<usize>(), "truncate");
    let budgets = match req.max_tokens {
        MaxTokens::All(b) => vec![b; req.texts.len()],
        MaxTokens::PerText(v) if v.len() == req.texts.len() => v,
        MaxTokens::PerText(_) => return Err(problem(TokenizerError::InvalidInput("max_tokens needs one budget per text".to_owned()))),
    };
    let r = service.truncate(&ctx, &req.model, &req.texts, &budgets, req.keep).await.map_err(problem)?;
    let mut out = TruncateResponse { texts: Vec::with_capacity(r.len()), kept_tokens: Vec::with_capacity(r.len()), counts: Vec::with_capacity(r.len()) };
    for (text, kept, count) in r {
        out.texts.push(text);
        out.kept_tokens.push(kept);
        out.counts.push(count);
    }
    Ok(Json(out))
}

pub async fn chunk(
    Extension(ctx): Extension<SecurityContext>,
    Extension(service): Extension<Arc<TokenizerService>>,
    Json(req): Json<ChunkRequest>,
) -> Result<Json<ChunkResponse>, Problem> {
    tracing::debug!(model = %req.model, texts = req.texts.len(), bytes = req.texts.iter().map(String::len).sum::<usize>(), "chunk");
    let r = service.chunk_with_spans(&ctx, &req.model, &req.texts, req.max_tokens, req.overlap).await.map_err(problem)?;
    let mut out = ChunkResponse { chunks: Vec::with_capacity(r.len()), spans: Vec::with_capacity(r.len()), counts: Vec::with_capacity(r.len()) };
    for (chunks, spans, count) in r {
        out.chunks.push(chunks);
        out.spans.push(spans);
        out.counts.push(count);
    }
    Ok(Json(out))
}

pub async fn count_tokens(
    Extension(ctx): Extension<SecurityContext>,
    Extension(service): Extension<Arc<TokenizerService>>,
    Json(req): Json<CountTokensRequest>,
) -> Result<Json<CountTokensResponse>, Problem> {
    tracing::debug!(model = %req.model, messages = req.messages.len(), "count_tokens");
    let usage = match req.template {
        None => service.count_tokens(&ctx, &req.model, &req.messages).await,
        Some(t) => {
            let template = match t {
                ChatTemplateDto::Overhead { tokens_per_message, tokens_per_name, reply_priming } => ChatTemplate::Overhead { tokens_per_message, tokens_per_name, reply_priming },
                ChatTemplateDto::Rendered { bos, message_prefix, message_suffix, generation_prompt, special_tokens } => {
                    ChatTemplate::Rendered { bos, message_prefix, message_suffix, generation_prompt, special_tokens }
                }
            };
            service.count_chat_tokens(&ctx, &req.model, &req.messages, &template).await
        }
    }
    .map_err(problem)?;
    Ok(Json(CountTokensResponse { input_tokens: usage.input_tokens }))
}
