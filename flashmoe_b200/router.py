"""Router rules of the gated forward (`MoEContext.forward_gated` -> fm_moe_forward_gated): which scores, bias, group
limit and weight scaling the kernel applies to the router's logits.  The checks mirror the C entry point's, so a bad
rule fails here with the field's name before any launch."""
from __future__ import annotations

import dataclasses
import math

from . import _lib

MAX_GROUPS = 32   # the kernel keeps a token's groups in one 32-bit mask


@dataclasses.dataclass(frozen=True)
class RouterSpec:
    """scoring: "softmax" (the built-in router's probabilities) or "sigmoid"; n_group: experts split into n_group
    contiguous groups of E / n_group (1 = no group limit); topk_group: groups kept per token; group_top: a group's score
    is its largest (1) or the sum of its two largest (2) biased scores; renormalize: divide the picked scores by their
    sum; scale: multiplies every weight.

    Examples: DeepSeek-V3 `RouterSpec("sigmoid", 8, 4, 2, True, 2.5)`; DeepSeek-V2 `RouterSpec("softmax", 8, 3, 1,
    False, 16.0)`; Qwen-MoE / OLMoE `RouterSpec("softmax", renormalize=False)`; Llama 4 (k = 1)
    `RouterSpec("sigmoid", renormalize=False)`."""
    scoring: str = "softmax"
    n_group: int = 1
    topk_group: int = 1
    group_top: int = 1
    renormalize: bool = True
    scale: float = 1.0

    def __post_init__(self):
        if self.scoring not in ("softmax", "sigmoid"):
            raise ValueError(f"scoring must be 'softmax' or 'sigmoid', got {self.scoring!r}")
        for name in ("n_group", "topk_group", "group_top"):
            v = getattr(self, name)
            if isinstance(v, bool) or not isinstance(v, int):
                raise ValueError(f"{name} must be an int, got {v!r}")
        if not 1 <= self.n_group <= MAX_GROUPS:
            raise ValueError(f"n_group must be in [1, {MAX_GROUPS}], got {self.n_group}")
        if not 1 <= self.topk_group <= self.n_group:
            raise ValueError(f"topk_group must be in [1, n_group={self.n_group}], got {self.topk_group}")
        if self.n_group > 1 and self.group_top not in (1, 2):
            raise ValueError(f"group_top must be 1 or 2, got {self.group_top}")
        if self.renormalize not in (True, False):   # (0 / 1 too)
            raise ValueError(f"renormalize must be a bool, got {self.renormalize!r}")
        if isinstance(self.scale, bool) or not isinstance(self.scale, (int, float)) or not math.isfinite(self.scale) \
                or not self.scale > 0:
            raise ValueError(f"scale must be finite and > 0, got {self.scale!r}")

    def check(self, E: int, k: int) -> None:
        """The conditions that involve the context: n_group divides E, group_top fits a group, k fits the kept
        groups."""
        if E % self.n_group:
            raise ValueError(f"n_group={self.n_group} does not divide E={E}")
        gs = E // self.n_group
        if self.n_group > 1 and self.group_top > gs:
            raise ValueError(f"group_top={self.group_top} exceeds the group size E / n_group = {gs}")
        if k > self.topk_group * gs:
            raise ValueError(f"k={k} exceeds the {self.topk_group * gs} experts of the topk_group={self.topk_group} "
                             f"kept groups")

    def to_c(self) -> _lib.FmRouter:
        return _lib.FmRouter(1 if self.scoring == "sigmoid" else 0, self.n_group, self.topk_group, self.group_top,
                             int(bool(self.renormalize)), float(self.scale))
