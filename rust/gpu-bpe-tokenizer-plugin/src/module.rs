//! Module declaration and `init` (pattern: `static-tr-plugin/src/module.rs:25-89`).

use std::sync::{Arc, OnceLock};

use async_trait::async_trait;
use llm_gateway_sdk::{TokenizerPluginClient, TokenizerPluginSpecV1};
use modkit::client_hub::ClientScope;
use modkit::context::ModuleCtx;
use modkit::gts::BaseModkitPluginV1;
use modkit::Module;
use tracing::info;
use types_registry_sdk::{RegisterResult, TypesRegistryClient};

use crate::config::GpuBpeTokenizerPluginConfig;
use crate::service::Service;

/// **Plugin registration pattern:** the gateway registers the plugin schema; this plugin registers its instance and its scoped client.
#[modkit::module(
    name = "gpu-bpe-tokenizer-plugin",
    deps = ["types-registry"]
)]
pub struct GpuBpeTokenizerPlugin {
    service: OnceLock<Arc<Service>>,
}

impl Default for GpuBpeTokenizerPlugin {
    fn default() -> Self {
        Self { service: OnceLock::new() }
    }
}

#[async_trait]
impl Module for GpuBpeTokenizerPlugin {
    async fn init(&self, ctx: &ModuleCtx) -> anyhow::Result<()> {
        info!("Initializing {} module", Self::MODULE_NAME);
        let cfg: GpuBpeTokenizerPluginConfig = ctx.config()?;

        // Device context + vocabulary tables.  Blocking (file reads, CUDA allocation, table build: ~1 s per vocabulary): off the runtime.
        // Fails when no sm_90 device is visible -- there is no CPU fallback, the module must not come up half-working.
        let cfg_for_service = cfg.clone();
        let service = tokio::task::spawn_blocking(move || Service::from_config(&cfg_for_service)).await??;
        let service = Arc::new(service);
        info!(devices = ?cfg.devices, vocabs = service.vocab_names().len(), "device context ready");

        let instance_id = TokenizerPluginSpecV1::gts_make_instance_id("cyberfabric.gpu_bpe.b200.v1");
        let registry = ctx.client_hub().get::<dyn TypesRegistryClient>()?;
        let instance = BaseModkitPluginV1::<TokenizerPluginSpecV1> {
            id: instance_id.clone(),
            vendor: cfg.vendor.clone(),
            priority: cfg.priority,
            properties: TokenizerPluginSpecV1,
        };
        let results = registry.register(vec![serde_json::to_value(&instance)?]).await?;
        RegisterResult::ensure_all_ok(&results)?;

        self.service
            .set(service.clone())
            .map_err(|_| anyhow::anyhow!("{} module already initialized", Self::MODULE_NAME))?;
        let api: Arc<dyn TokenizerPluginClient> = service;
        ctx.client_hub()
            .register_scoped::<dyn TokenizerPluginClient>(ClientScope::gts_id(&instance_id), api);
        info!(instance_id = %instance_id, "{} module initialized successfully", Self::MODULE_NAME);
        Ok(())
    }
}
