//! Plugin configuration (`ctx.config::<T>()`; convention `#[serde(default, deny_unknown_fields)]`,
//! `docs/MODKIT_PLUGINS.md:644-659`; `vendor` + `priority` as in `static-tr-plugin/src/config.rs`).

use serde::Deserialize;

#[derive(Debug, Clone, Deserialize)]
#[serde(default, deny_unknown_fields)]
pub struct GpuBpeTokenizerPluginConfig {
    /// Vendor name for GTS instance registration.
    pub vendor: String,
    /// Plugin priority (lower = higher priority).
    pub priority: i16,
    /// CUDA device ordinals.
    pub devices: Vec<i32>,
    /// Largest packed batch one call may carry (bytes; below 4 GiB) and its prompt count.
    pub max_batch_bytes: u64,
    pub max_prompts: u32,
    /// Independent workspaces per device = host calls that run concurrently on the context.
    pub workspaces: u32,
    /// Micro-batcher for `count_tokens`: how long the first queued request waits for company, and the batch size that ends the wait.
    pub batch_wait_us: u64,
    pub batch_bytes: u64,
    pub vocabs: Vec<VocabConfig>,
}

impl Default for GpuBpeTokenizerPluginConfig {
    fn default() -> Self {
        Self {
            vendor: "cyberfabric".to_owned(),
            priority: 10,
            devices: vec![0],
            max_batch_bytes: 16 << 20,
            max_prompts: 1 << 16,
            workspaces: 4,
            batch_wait_us: 500,
            batch_bytes: 8 << 20,
            vocabs: Vec::new(),
        }
    }
}

#[derive(Debug, Clone, Copy, Deserialize, PartialEq, Eq)]
#[serde(rename_all = "snake_case")]
pub enum RankFileFormat {
    Tiktoken,
    TekkenJson,
}

#[derive(Debug, Clone, Copy, Deserialize, PartialEq, Eq)]
#[serde(rename_all = "snake_case")]
pub enum Pattern {
    Cl100k,
    O200k,
    Llama3,
    Tekken,
}

/// One vocabulary: where its rank file is, what it must hash to, which models use it
/// (the model-registry side: `tokenizer{vocab_id, pattern_id, sha256}`, `docs/model-registry-tokenizer-proposal.md`).
#[derive(Debug, Clone, Deserialize)]
#[serde(deny_unknown_fields)]
pub struct VocabConfig {
    pub name: String,
    pub path: String,
    /// hex sha256 of the rank file; a mismatch fails `init` (a stand-in vocabulary must never be served silently)
    pub sha256: String,
    pub format: RankFileFormat,
    pub pattern: Pattern,
    /// use only the first `max_ranks` ranks (0 = all)
    #[serde(default)]
    pub max_ranks: u32,
    /// canonical model ids `{provider_slug}::{provider_model_id}` served by this vocabulary
    #[serde(default)]
    pub models: Vec<String>,
    /// id of the ordinary token of rank 0 (0 = ids are ranks; Mistral's Tekken: 1000, after its control tokens)
    #[serde(default)]
    pub id_base: u32,
    /// JSON list of the control tokens in id order, ids 0 .. id_base - 1 (`vocabs/tekken_controls.json`), registered as the
    /// vocabulary's special tokens
    #[serde(default)]
    pub controls_path: Option<String>,
}
