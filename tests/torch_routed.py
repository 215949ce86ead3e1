"""Plain torch CPU statement of the caller-routing forward (fm_moe_forward_routed): the expert FFN and combine of
oracle/torch_moe.py on routing the caller supplies, written from the contract alone.

TEST INFRASTRUCTURE ONLY.  Contract:
  * an index outside [0, E) is no pick (-1 and, after the kernel's report, any other out-of-range value);
  * slots in ascending (token, pick) order among the picks of one expert, a skipped pick takes none; kept = slot < EC;
  * a token may name one expert twice: each pick is its own row;
  * out[t] = bf16 accumulation, in ascending pick order from +0, of rne(rne_bf16(w_j) * y_j) over the kept picks --
    k = 1 is scaled too; y_j = rne(act(x W_up^T + b_up) W_down^T + b_down) as on the router path.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

INT32_MAX = 2 ** 31 - 1


def _rne(t: torch.Tensor) -> torch.Tensor:
    return t.to(torch.bfloat16).to(torch.float32)


def _act(t: torch.Tensor, act: int) -> torch.Tensor:
    return torch.relu(t) if act == 0 else torch.nn.functional.gelu(t)


def moe_forward_routed_cpu(x: torch.Tensor, topk_idx: torch.Tensor, topk_w: torch.Tensor,
                           expert_weights: torch.Tensor, *, EC: int, act: int = 0,
                           bias_up: Optional[torch.Tensor] = None,
                           bias_down: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
    """Single rank, all experts local.  x [n, H] bf16, topk_idx [n, k] integer, topk_w [n, k] float, expert_weights
    [E, 2, P, H] bf16 (the down block read flat as W_down [H, P]), CPU tensors.  Returns out (bf16 [n, H]), topk_idx
    (int32, invalid picks -1), topk_w (bf16), slot (int32, INT32_MAX for a skipped pick), counts and kept."""
    n, H = x.shape
    E, _, P, _ = expert_weights.shape
    k = topk_idx.shape[1]
    idx = topk_idx.long()
    valid = (idx >= 0) & (idx < E)
    idx = torch.where(valid, idx, torch.full_like(idx, -1))
    w = _rne(topk_w.float())
    # slot of each (token, pick): the number of earlier valid picks of the same expert in (token, pick) order
    flat = idx.reshape(-1)
    onehot = torch.nn.functional.one_hot(flat.clamp(min=0), E) * valid.reshape(-1, 1)
    before = torch.cumsum(onehot, dim=0) - onehot
    slot = before.gather(1, flat.clamp(min=0)[:, None])[:, 0].view(n, k)
    slot = torch.where(valid, slot, torch.full_like(slot, INT32_MAX))
    kept = valid & (slot < EC)
    xf = x.float()
    terms = torch.zeros(k, n, H)
    for e in range(E):
        tok, j = ((idx == e) & kept).nonzero(as_tuple=True)
        if tok.numel() == 0:
            continue
        w_up = expert_weights[e, 0].float()
        w_down = expert_weights[e, 1].contiguous().view(-1).view(H, P).float()
        h = xf[tok] @ w_up.t()
        if bias_up is not None:
            h = h + bias_up[e].float()
        h = _rne(_act(h, act))
        y = h @ w_down.t()
        if bias_down is not None:
            y = y + bias_down[e].float()
        terms[j, tok] = _rne(w[tok, j][:, None] * _rne(y))
    out = torch.zeros(n, H)
    for j in range(k):   # bf16 accumulation in ascending pick order
        out = torch.where(kept[:, j][:, None], _rne(out + terms[j]), out)
    counts = torch.bincount(idx[valid], minlength=E)
    return {"out": out.to(torch.bfloat16), "topk_idx": idx.to(torch.int32), "topk_w": w.to(torch.bfloat16),
            "slot": slot.to(torch.int32), "counts": counts.to(torch.int32), "kept": kept}
