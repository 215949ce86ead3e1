"""flashmoe_b200 -- Hopper (sm_90a) native fused distributed-MoE forward, drop-in for the hot path of
osayamenja/FlashMoE (`flashmoe.run_moe`, `flashmoe.ops`, `flashmoe._C`).

    import flashmoe_b200 as flashmoe      # or `import flashmoe` (shim package re-exporting this one)
    flashmoe.run_moe()                    # single GPU, synthetic tensors sized by csrc/flashmoe_config.json
    flashmoe.run_moe(n_processes=8)       # one process per GPU, expert-parallel over NVLink

Compile-time configuration (same 15 keys as the reference): edit csrc/flashmoe_config.json, then
`python -m flashmoe_b200._build`.  There is no CPU fallback: without the native library every call raises.
"""
from .ops import get_compiled_config, run_moe  # noqa: F401

try:  # soft import like the reference (flashmoe/__init__.py:20-30): the package stays importable for tooling
    from . import _C  # noqa: F401
except Exception as _e:  # pragma: no cover - only when the native library is missing
    import warnings

    warnings.warn(f"flashmoe_b200 native library not available ({_e}); build it with `python -m flashmoe_b200._build`")

__version__ = "0.1.0"
__all__ = ["run_moe", "get_compiled_config"]
