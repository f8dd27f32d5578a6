//! GPU BPE tokenizer plugin (NVIDIA H100, `libcfbpe.so`).
//!
//! ```yaml
//! modules:
//!   gpu-bpe-tokenizer-plugin:
//!     vendor: "cyberfabric"
//!     priority: 10
//!     devices: [0]                 # CUDA ordinals; several = one context that shards every batch by bytes
//!     max_batch_bytes: 16777216
//!     max_prompts: 65536
//!     workspaces: 4                # concurrent host calls per device
//!     vocabs:
//!       - name: "cl100k_base"
//!         path: "/var/lib/cyberfabric/vocabs/cl100k_base.tiktoken"
//!         sha256: "223921b76ee99bde995b7ff738513eef100fb51d18c93597a113bcffe865b2a7"
//!         format: tiktoken
//!         pattern: cl100k
//!         models: ["openai::gpt-4", "openai::gpt-3.5-turbo"]
//! ```
//! NOT COMPILED where this file lives (no Rust toolchain); Python mirror: `cyberfabric-core_b200/cfbpe/plugin.py`.

pub mod batcher;
pub mod config;
pub mod module;
pub mod service;

pub use module::GpuBpeTokenizerPlugin;
