"""Compile-time configuration surface: csrc/flashmoe_config.json -> derived constants.

Mirrors the reference's JSON -> `-D` macros -> `flashmoe::ACC` chain
(reference csrc/CMakeLists.txt:114-237, setup.py:227-292, csrc/include/flashmoe/types.cuh:441-512).
One module is shared by the build (`_build.py` bakes the JSON into the shared library), the
oracle, the tests and bench.py, so every consumer derives S / EC / pEC / PX the same way.
"""
from __future__ import annotations

import dataclasses
import json
import os
from pathlib import Path
from typing import Any, Dict, Optional

REPO_ROOT = Path(__file__).resolve().parent.parent
DEFAULT_CONFIG_PATH = REPO_ROOT / "csrc" / "flashmoe_config.json"
SCHEMA_PATH = REPO_ROOT / "csrc" / "flashmoe_config.schema.json"

BLOCK_M = 128  # token rows per tile (reference BLOCK_M, types.cuh:499 pads EC to it)
REF_BLOCK_N = 64  # the reference pads the gate's expert axis to its BLOCK_N (types.cuh:480)

# keys the reference's build reads (CMakeLists.txt:217-237); all 15 are accepted.
ALL_KEYS = (
    "capacity_factor", "drop_tokens", "expert_top_k", "global_batch", "is_training", "hidden_act",
    "hidden_size", "intermediate_size", "mini_batch", "moe_frequency", "num_experts", "num_layers",
    "sequence_len", "torch_dtype", "vocab_size",
)
REQUIRED_KEYS = tuple(k for k in ALL_KEYS if k != "global_batch")

DTYPE_BF16 = 2  # schema: 0 fp32, 1 tf32, 2 bf16, 3 fp16 (flashmoe_config.schema.json:64-68)
ACT_RELU, ACT_GELU, ACT_SWIGLU = 0, 1, 2


class ConfigError(ValueError):
    """Raised for a config that violates the schema or a hot-path constraint."""


def _ceil_div(a: int, b: int) -> int:
    return -(-a // b)


def validate_raw(raw: Dict[str, Any]) -> None:
    """Validate `raw` against csrc/flashmoe_config.schema.json (hand-rolled: jsonschema is not installed)."""
    with open(SCHEMA_PATH) as f:
        schema = json.load(f)
    for key in schema["required"]:
        if key not in raw:
            raise ConfigError(f"missing required config key '{key}'")
    for key, val in raw.items():
        spec = schema["properties"].get(key)
        if spec is None:
            raise ConfigError(f"unknown config key '{key}'")
        if isinstance(val, bool) or not isinstance(val, int):
            raise ConfigError(f"config key '{key}' must be an integer, got {val!r}")
        if "enum" in spec and val not in spec["enum"]:
            raise ConfigError(f"config key '{key}'={val} not in {spec['enum']}")
        if "minimum" in spec and val < spec["minimum"]:
            raise ConfigError(f"config key '{key}'={val} < minimum {spec['minimum']}")
        if "multipleOf" in spec and (val <= 0 or val % spec["multipleOf"]):
            raise ConfigError(f"config key '{key}'={val} must be a positive multiple of {spec['multipleOf']}")


@dataclasses.dataclass(frozen=True)
class MoEConfig:
    """The `ACC` equivalent: raw keys + everything derived from them (types.cuh:441-512)."""

    capacity_factor: int = 1
    drop_tokens: int = 1
    expert_top_k: int = 2
    global_batch: int = 256
    is_training: int = 0
    hidden_act: int = 0
    hidden_size: int = 1024
    intermediate_size: int = 4096
    mini_batch: int = 1
    moe_frequency: int = 1
    num_experts: int = 8
    num_layers: int = 1
    sequence_len: int = 4096
    torch_dtype: int = DTYPE_BF16
    vocab_size: int = 32000

    # ---- derived (names follow the reference) ----
    @property
    def S(self) -> int:  # tokens per rank (types.cuh:470)
        return self.sequence_len * self.mini_batch

    @property
    def H(self) -> int:
        return self.hidden_size

    @property
    def P(self) -> int:
        return self.intermediate_size

    @property
    def E(self) -> int:
        return self.num_experts

    @property
    def k(self) -> int:
        return self.expert_top_k

    @property
    def expert_mats(self) -> int:
        """Matrices per expert in the expert weights: [W_up, W_down], or SwiGLU's [W_gate, W_up, W_down]."""
        return 3 if self.hidden_act == ACT_SWIGLU else 2

    @property
    def PX(self) -> int:  # padded expert axis of gateOut (types.cuh:480)
        return _ceil_div(self.E, REF_BLOCK_N) * REF_BLOCK_N

    @property
    def EC(self) -> int:  # expert capacity in token-expert pairs per source rank (types.cuh:497)
        return self.EC_of(self.S)

    def EC_of(self, n_tokens: int) -> int:
        """Expert capacity of a forward over `n_tokens` tokens (MoEContext.forward_tokens): what a config with
        S = n_tokens has as EC."""
        base = _ceil_div(n_tokens, self.E) if self.drop_tokens else n_tokens
        return base * self.capacity_factor * self.k

    @property
    def pEC(self) -> int:  # EC padded to the row tile (types.cuh:499)
        return _ceil_div(self.EC, BLOCK_M) * BLOCK_M

    @property
    def TCM(self) -> int:  # row tiles per (source rank, expert) packet (types.cuh:504)
        return _ceil_div(self.EC, BLOCK_M)

    def num_local_experts(self, world: int) -> int:
        """Static contiguous placement, expert e -> rank e // (E/W) (reference bootstrap.cuh:35-52)."""
        if world < 1 or self.E % world:
            raise ConfigError(f"num_experts={self.E} must be divisible by world size {world}")
        return self.E // world

    def check_hot_path(self) -> None:
        """Constraints the kernels rely on (reference asserts: bootstrap.cuh:542-544, types.cuh:496)."""
        if self.torch_dtype != DTYPE_BF16:
            raise ConfigError("this build computes in bf16 only (torch_dtype must be 2)")
        if self.is_training not in (0, 1):
            raise ConfigError("is_training must be 0 or 1")
        if self.S % BLOCK_M:
            raise ConfigError(f"S={self.S} must be a multiple of {BLOCK_M}")
        if self.H % 64 or self.P % 64:
            raise ConfigError("hidden_size and intermediate_size must be multiples of 64")
        if not (1 <= self.k <= self.E):
            raise ConfigError(f"expert_top_k={self.k} must be in [1, num_experts={self.E}]")
        if self.k > 8:
            raise ConfigError("expert_top_k > 8 is not supported by the router kernel")
        if self.E > 1024:
            raise ConfigError("num_experts > 1024 is not supported by the router kernel")

    def raw(self) -> Dict[str, int]:
        return {k: getattr(self, k) for k in ALL_KEYS}

    def compiled_dict(self) -> Dict[str, int]:
        """Same keys as the reference's `_C.get_compiled_config()` (python_bindings.cu:170-179)."""
        return {"S": self.S, "H": self.H, "E": self.E, "P": self.P, "PX": self.PX, "Element_size": 2}

    def replace(self, **kw: int) -> "MoEConfig":
        return dataclasses.replace(self, **kw)


def from_dict(raw: Dict[str, Any], *, validate: bool = True) -> MoEConfig:
    if validate:
        validate_raw(raw)
    return MoEConfig(**{k: int(v) for k, v in raw.items()})


def load_config(path: Optional[os.PathLike] = None) -> MoEConfig:
    """Load and validate a config JSON; default is csrc/flashmoe_config.json (the reference's dangling
    default `csrc/kleos_config.json`, ops.py:22 / launcher.py:12, is not reproduced)."""
    p = Path(path) if path is not None else DEFAULT_CONFIG_PATH
    if not p.exists():
        raise FileNotFoundError(f"Config file not found: {p}")
    with open(p) as f:
        raw = json.load(f)
    return from_dict(raw)


# The BASELINE.json configurations (SURVEY.md section 8 header / Appendix B).  A: CPU plumbing case; B: the single-GPU
# headline; C: Mixtral-8x7B layer shape on 8 GPUs; D*: token sweep (32 experts, d_model 2048, ffn 2048 = the
# reference's default intermediate_size, csrc/flashmoe_config.json:9); E*: expert sweep at 8192 tokens per rank.
def _sweep(E: int, S: int) -> "MoEConfig":
    return MoEConfig(num_experts=E, expert_top_k=2, sequence_len=S, hidden_size=2048, intermediate_size=2048)


BASELINE_CONFIGS: Dict[str, MoEConfig] = {
    "A": MoEConfig(num_experts=2, expert_top_k=1, sequence_len=128, hidden_size=512, intermediate_size=2048),
    "B": MoEConfig(num_experts=8, expert_top_k=2, sequence_len=4096, hidden_size=1024, intermediate_size=4096),
    "C": MoEConfig(num_experts=8, expert_top_k=2, sequence_len=4096, hidden_size=4096, intermediate_size=14336),
    "D1k": _sweep(32, 1024), "D4k": _sweep(32, 4096), "D16k": _sweep(32, 16384), "D64k": _sweep(32, 65536),
    "E8": _sweep(8, 8192), "E16": _sweep(16, 8192), "E32": _sweep(32, 8192), "E64": _sweep(64, 8192),
    "E128": _sweep(128, 8192),
}

CONFIG_DESCRIPTIONS: Dict[str, str] = {
    "A": "configs[0]: 2 experts top-1 seq=128 d_model=512 ffn=2048 (CPU plumbing case)",
    "B": "configs[1]: 8 experts top-2 seq=4096 d_model=1024 ffn=4096 bf16 (per rank); experts sharded E/N",
    "C": "configs[2]: 8 experts top-2 seq=4096 d_model=4096 ffn=14336 bf16 (Mixtral-8x7B layer shape, per rank); experts sharded E/N",
    **{f"D{n}": f"configs[3] token sweep: 32 experts top-2 seq={s} d_model=2048 ffn=2048 bf16 (per rank); experts sharded E/N"
       for n, s in (("1k", 1024), ("4k", 4096), ("16k", 16384), ("64k", 65536))},
    **{f"E{e}": f"configs[4] expert sweep: {e} experts top-2 seq=8192 d_model=2048 ffn=2048 bf16 (per rank); experts sharded E/N"
       for e in (8, 16, 32, 64, 128)},
}
