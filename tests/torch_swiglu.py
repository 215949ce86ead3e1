"""Plain torch CPU statement of the SwiGLU forward (hidden_act = 2), written from the contract alone, on the built-in
router's routing (oracle/torch_moe.route) or on the caller's (the conventions of tests/torch_routed.py).

TEST INFRASTRUCTURE ONLY.  Contract:
  * expert_weights [E, 3, P, H] bf16: [e,0] = W_gate, [e,1] = W_up, [e,2] read flat as W_down [H, P];
    bias_up [E, 2, P] (gate, then up) and bias_down [E, H], optional;
  * g = x W_gate^T + b_g and u = x W_up^T + b_u in fp32; h = rne_bf16(silu(g) * u) (torch's fp32 silu, not the kernel's
    ex2 / reciprocal); y = rne_bf16(h W_down^T + b_down);
  * router route: out = y for k = 1; otherwise the bf16 accumulation, in ascending pick order from +0, of
    rne(p~_j rne(y_j / mcw)), p~ = rne_bf16(p) (oracle/torch_moe.py's combine, unchanged);
  * caller route: an index outside [0, E) is no pick; out = the bf16 accumulation of rne(rne_bf16(w_j) y_j) for every k.
Slots: ascending (token, pick) order among the valid picks of one expert; kept = slot < EC.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch
import torch.nn.functional as F

from oracle.torch_moe import route

INT32_MAX = 2 ** 31 - 1


def _rne(t: torch.Tensor) -> torch.Tensor:
    return t.to(torch.bfloat16).to(torch.float32)


def _slots(idx: torch.Tensor, E: int, EC: int):
    n, k = idx.shape
    valid = idx >= 0
    flat = idx.reshape(-1).clamp(min=0)
    onehot = F.one_hot(flat, E) * valid.reshape(-1, 1)
    before = torch.cumsum(onehot, dim=0) - onehot
    slot = before.gather(1, flat[:, None])[:, 0].view(n, k)
    slot = torch.where(valid, slot, torch.full_like(slot, INT32_MAX))
    return slot, valid & (slot < EC)


def _experts(xf, idx, slot, kept, expert_weights, EC, bias_up, bias_down):
    """Per-pick y [k, n, H] (fp32 of bf16) and the packets h [E, EC, P] / y [E, EC, H] (bf16, rows by slot)."""
    n, k = idx.shape
    E, _, P, H = expert_weights.shape
    y_pick = torch.zeros(k, n, H)
    h_pkt = torch.zeros(E, EC, P, dtype=torch.bfloat16)
    y_pkt = torch.zeros(E, EC, H, dtype=torch.bfloat16)
    for e in range(E):
        tok, j = ((idx == e) & kept).nonzero(as_tuple=True)
        if tok.numel() == 0:
            continue
        w = expert_weights[e].float()
        g = xf[tok] @ w[0].t()
        u = xf[tok] @ w[1].t()
        if bias_up is not None:
            g = g + bias_up[e, 0].float()
            u = u + bias_up[e, 1].float()
        h = _rne(F.silu(g) * u)
        y = h @ expert_weights[e, 2].contiguous().view(-1).view(H, P).float().t()
        if bias_down is not None:
            y = y + bias_down[e].float()
        y = _rne(y)
        y_pick[j, tok] = y
        h_pkt[e, slot[tok, j]] = h.bfloat16()
        y_pkt[e, slot[tok, j]] = y.bfloat16()
    return y_pick, h_pkt, y_pkt


def _accumulate(terms, kept):
    out = torch.zeros(terms.shape[1:])
    for j in range(terms.shape[0]):   # bf16 accumulation in ascending pick order
        out = torch.where(kept[:, j][:, None], _rne(out + terms[j]), out)
    return out


def moe_forward_swiglu_cpu(x: torch.Tensor, gate_weights: torch.Tensor, expert_weights: torch.Tensor, *, k: int,
                           EC: int, bias_up: Optional[torch.Tensor] = None,
                           bias_down: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
    """Router route, one rank.  x [n, H], gate_weights [H, E], expert_weights [E, 3, P, H], bf16 CPU tensors."""
    E = expert_weights.shape[0]
    probs, topk, mcw = route(x, gate_weights, k)
    slot, kept = _slots(topk, E, EC)
    y_pick, h_pkt, y_pkt = _experts(x.float(), topk, slot, kept, expert_weights, EC, bias_up, bias_down)
    p_tilde = _rne(probs)
    if k == 1:
        out = torch.where(kept[:, 0][:, None], y_pick[0], torch.zeros(()))
    else:
        q = _rne(y_pick / mcw[None, :, None])
        terms = _rne(p_tilde.gather(1, topk).t()[:, :, None] * q)
        out = _accumulate(terms, kept)
    return {"out": out.to(torch.bfloat16), "topk_idx": topk.to(torch.int32), "topk_w": p_tilde.gather(1, topk),
            "mcw": mcw, "slot": slot.to(torch.int32), "kept": kept, "hidden": h_pkt, "ret_y": y_pkt}


def moe_forward_swiglu_routed_cpu(x: torch.Tensor, topk_idx: torch.Tensor, topk_w: torch.Tensor,
                                  expert_weights: torch.Tensor, *, EC: int, bias_up: Optional[torch.Tensor] = None,
                                  bias_down: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
    """Caller route, one rank: topk_idx [n, k] integer, topk_w [n, k] float."""
    E = expert_weights.shape[0]
    idx = topk_idx.long()
    idx = torch.where((idx >= 0) & (idx < E), idx, torch.full_like(idx, -1))
    slot, kept = _slots(idx, E, EC)
    y_pick, h_pkt, y_pkt = _experts(x.float(), idx, slot, kept, expert_weights, EC, bias_up, bias_down)
    w = _rne(topk_w.float())
    out = _accumulate(_rne(w.t()[:, :, None] * y_pick), kept)
    return {"out": out.to(torch.bfloat16), "topk_idx": idx.to(torch.int32), "topk_w": w, "mcw": torch.ones(len(x)),
            "slot": slot.to(torch.int32), "kept": kept, "hidden": h_pkt, "ret_y": y_pkt}
