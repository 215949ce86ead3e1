"""Plain torch CPU statement of the gated forward's routing (fm_moe_forward_gated, steps 2-6 of its contract), written
from the contract alone; the rest of the forward is tests/torch_routed.moe_forward_routed_cpu on that routing.

TEST INFRASTRUCTURE ONLY.  Per token, on fp32 logits l [E]:
  * scores s: softmax or sigmoid of l (torch's fp32 functions, not the kernel's approximations);
  * choice values c = fl(s + b) (c = s without a bias); NaN never compares greater (here: NaN -> -inf);
  * n_group > 1: G_g = the largest c of the group, or fl(largest + second largest); topk_group rounds keep the group
    with the largest G not yet kept, the lower index on equal values, index 0 when nothing is greater than -inf;
  * k rounds pick the allowed, not yet picked expert with the largest c, same tie and fallback rules;
  * w_j = s[e_j]; renormalize: W = fp32 sum in pick order from +0, w_j = W > 0 ? w_j / W : 0; then w_j = fl(w_j scale).
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from flashmoe_b200.router import RouterSpec
from tests.torch_routed import moe_forward_routed_cpu


def _first_argmax(v: torch.Tensor) -> torch.Tensor:
    """Index of the first largest value per row (torch.argmax's documented tie rule, made explicit)."""
    m = v.max(dim=1, keepdim=True).values
    hit = v == m
    return torch.where(hit, torch.arange(v.shape[1]).expand_as(v), v.shape[1]).min(dim=1).values


def gated_routing_cpu(logits: torch.Tensor, router: RouterSpec, k: int,
                      score_bias: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
    """logits fp32 [n, E] -> scores (fp32 [n, E], the unbiased s), topk_idx (int32 [n, k]) and topk_w (fp32 [n, k],
    before the bf16 rounding the kernel stores)."""
    l = logits.float()
    n, E = l.shape
    router.check(E, k)
    s = torch.softmax(l, dim=1) if router.scoring == "softmax" else torch.sigmoid(l)
    c = s + score_bias.float()[None, :] if score_bias is not None else s.clone()
    c = torch.where(torch.isnan(c), torch.full_like(c, -float("inf")), c)
    rows = torch.arange(n)
    allowed = torch.ones(n, E, dtype=torch.bool)
    if router.n_group > 1:
        G, GS = router.n_group, E // router.n_group
        top = c.view(n, G, GS).sort(dim=2, descending=True).values
        gscore = top[:, :, 0] if router.group_top == 1 else top[:, :, 0] + top[:, :, 1]
        kept = torch.zeros(n, G, dtype=torch.bool)
        for _ in range(router.topk_group):
            cand = torch.where(kept, torch.full_like(gscore, -float("inf")), gscore)
            kept[rows, _first_argmax(cand)] = True
        allowed = kept.repeat_interleave(GS, dim=1)
    taken = torch.zeros(n, E, dtype=torch.bool)
    idx = torch.zeros(n, k, dtype=torch.int64)
    for j in range(k):
        cand = torch.where(allowed & ~taken, c, torch.full_like(c, -float("inf")))
        e = _first_argmax(cand)   # (a row of -inf only: index 0)
        idx[:, j] = e
        taken[rows, e] = True
    w = s.gather(1, idx)
    if router.renormalize:
        W = torch.zeros(n)
        for j in range(k):   # fp32, in pick order
            W = W + w[:, j]
        w = torch.where((W > 0)[:, None], w / W[:, None], torch.zeros_like(w))
    w = w * torch.tensor(router.scale, dtype=torch.float32)
    return {"scores": s, "topk_idx": idx.to(torch.int32), "topk_w": w}


def moe_forward_gated_cpu(x: torch.Tensor, gate_weights: torch.Tensor, expert_weights: torch.Tensor,
                          router: RouterSpec, k: int, *, EC: int, act: int = 0,
                          score_bias: Optional[torch.Tensor] = None, bias_up: Optional[torch.Tensor] = None,
                          bias_down: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
    """Single rank, all experts local.  x [n, H] bf16, gate_weights [H, E] bf16 read flat as Wg_eff [E, H] (as the
    kernel reads it), expert_weights [E, 2, P, H] bf16.  Returns moe_forward_routed_cpu's tables plus gate_out
    (bf16 [n, E] of the unbiased scores) and the fp32 weights `w`."""
    H = x.shape[1]
    E = expert_weights.shape[0]
    wg_eff = gate_weights.reshape(-1).reshape(E, H).float()
    r = gated_routing_cpu(x.float() @ wg_eff.t(), router, k, score_bias)
    res = moe_forward_routed_cpu(x, r["topk_idx"], r["topk_w"], expert_weights, EC=EC, act=act, bias_up=bias_up,
                                 bias_down=bias_down)
    res["gate_out"] = r["scores"].to(torch.bfloat16)
    res["w"] = r["topk_w"]
    return res
