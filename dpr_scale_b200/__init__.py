"""dpr_scale_b200 — H100-native (sm_90a) bi-encoder training path behind dpr-scale's plugin surface.

Only what the hot path needs lives here: ``csrc/`` (CUDA kernels + the C ABI of ``include/dprb.h``),
``_lib`` (ctypes binding), ``ops`` (tensor-level wrappers), ``models`` / ``task`` (mirrors of
``dpr_scale.models.hf_model.HFEncoder`` and ``dpr_scale.task.dpr_task.DenseRetrieverTask``),
``conf`` (Hydra-style YAML groups) and ``utils`` (config composer, mini trainer, samplers).
"""
__version__ = "0.1.0"
