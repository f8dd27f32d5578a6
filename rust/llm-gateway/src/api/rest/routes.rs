//! Route registration (OperationBuilder pattern of `modules/file-parser/src/api/rest/routes.rs:49-71`; versioned path: DE0801).

use std::sync::Arc;

use axum::{Extension, Router};
use modkit::api::{operation_builder::LicenseFeature, OpenApiRegistry, OperationBuilder};

use crate::api::rest::{dto, handlers};
use crate::domain::service::TokenizerService;

struct License;

impl AsRef<str> for License {
    fn as_ref(&self) -> &'static str {
        "gts.x.core.lic.feat.v1~x.core.global.base.v1"
    }
}

impl LicenseFeature for License {}

#[allow(clippy::needless_pass_by_value)] // Arc is intentionally passed by value for the Extension layer
pub fn register_routes(mut router: Router, openapi: &dyn OpenApiRegistry, service: Arc<TokenizerService>) -> Router {
    // POST /llm-gateway/v1/tokenize - token ids / counts of a list of texts under a model's vocabulary
    router = OperationBuilder::post("/llm-gateway/v1/tokenize")
        .operation_id("llm_gateway.tokenize")
        .summary("Tokenize texts with the vocabulary of a model")
        .tag("LLM Gateway")
        .authenticated()
        .require_license_features::<License>([])
        .json_request::<dto::TokenizeRequest>(openapi, "Texts and the model whose vocabulary applies")
        .allow_content_types(&["application/json"])
        .handler(handlers::tokenize)
        .json_response_with_schema::<dto::TokenizeResponse>(openapi, http::StatusCode::OK, "Token counts (and ids)")
        .standard_errors(openapi)
        .error_415(openapi)
        .register(router, openapi);
    // POST /llm-gateway/v1/count-tokens - Usage.input_tokens of a chat request before it is sent (budget / context-window checks)
    router = OperationBuilder::post("/llm-gateway/v1/count-tokens")
        .operation_id("llm_gateway.count_tokens")
        .summary("Count the input tokens of a chat request, with the provider's framing if a template is given")
        .tag("LLM Gateway")
        .authenticated()
        .require_license_features::<License>([])
        .json_request::<dto::CountTokensRequest>(openapi, "Messages, the model whose vocabulary applies, and optionally its chat template")
        .allow_content_types(&["application/json"])
        .handler(handlers::count_tokens)
        .json_response_with_schema::<dto::CountTokensResponse>(openapi, http::StatusCode::OK, "Usage.input_tokens")
        .standard_errors(openapi)
        .error_415(openapi)
        .register(router, openapi);
    // POST /llm-gateway/v1/truncate - cut texts to a token budget (keep the head or the tail) at a character boundary
    router = OperationBuilder::post("/llm-gateway/v1/truncate")
        .operation_id("llm_gateway.truncate")
        .summary("Cut texts to a token budget of a model's vocabulary, keeping their first or last tokens")
        .tag("LLM Gateway")
        .authenticated()
        .require_license_features::<License>([])
        .json_request::<dto::TruncateRequest>(openapi, "Texts, the model whose vocabulary applies, the budget and which end to keep")
        .allow_content_types(&["application/json"])
        .handler(handlers::truncate)
        .json_response_with_schema::<dto::TruncateResponse>(openapi, http::StatusCode::OK, "The kept texts, their tokens and the full counts")
        .standard_errors(openapi)
        .error_415(openapi)
        .register(router, openapi);
    // POST /llm-gateway/v1/chunk - split texts into chunks of at most N tokens, optionally overlapping, at character boundaries
    router = OperationBuilder::post("/llm-gateway/v1/chunk")
        .operation_id("llm_gateway.chunk")
        .summary("Split texts into chunks of at most N tokens of a model's vocabulary, with an optional overlap")
        .tag("LLM Gateway")
        .authenticated()
        .require_license_features::<License>([])
        .json_request::<dto::ChunkRequest>(openapi, "Texts, the model whose vocabulary applies, the chunk size and the overlap")
        .allow_content_types(&["application/json"])
        .handler(handlers::chunk)
        .json_response_with_schema::<dto::ChunkResponse>(openapi, http::StatusCode::OK, "The chunks, their byte spans and the full counts")
        .standard_errors(openapi)
        .error_415(openapi)
        .register(router, openapi);
    router.layer(Extension(service))
}
