"""Plain torch statement of Hugging Face's `Llama4TextMoe.forward` in bf16, written from its semantics (transformers is
not imported: a test machine need not have it), and the conversion of its tensors to this project's layouts.

TEST INFRASTRUCTURE ONLY.  Hugging Face layouts (E experts, H hidden, P intermediate, Ps the shared MLP's):
  router_w [E, H] (nn.Linear), gate_up [E, H, 2P] (gate columns, then up), down [E, P, H], shared gate / up [Ps, H] and
  shared down [H, Ps] (nn.Linear weights).
Semantics, on CPU or CUDA tensors alike:
  logits = x router_w^T (bf16); one pick per token, the largest logit (or the given `picks`);
  scores = sigmoid(fp32 of the picked logit) rounded to bf16, 0 for every other expert;
  routed_in[e] = x * scores[:, e] (bf16 * bf16 -> bf16: the weight scales the input);
  routed_out[e] = (up * silu(gate)) down with gate, up = routed_in[e] gate_up[e] split in half (bf16 bmm, no bias);
  out = shared(x) + sum_e routed_out[e], the shared MLP on the unscaled x, the add in bf16.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F


def router_scores(x: torch.Tensor, router_w: torch.Tensor, picks: Optional[torch.Tensor] = None,
                  weights: Optional[torch.Tensor] = None):
    """(scores [n, E] bf16, picks [n, 1] int64): Llama4Router on x [n, H] bf16, or on the given picks (and with the
    given bf16 weights [n, 1] of those picks instead of their sigmoid scores)."""
    logits = x @ router_w.t()
    if picks is None:
        picks = logits.topk(1, dim=1).indices
    picks = picks.long()
    scores = torch.sigmoid(torch.full_like(logits, float("-inf")).scatter_(1, picks, logits.gather(1, picks)).float())
    scores = scores.to(x.dtype)
    if weights is not None:
        scores = torch.zeros_like(scores).scatter_(1, picks, weights.to(x.dtype))
    return scores, picks


def shared_mlp(x: torch.Tensor, gate: torch.Tensor, up: torch.Tensor, down: torch.Tensor,
               inside: Optional[torch.dtype] = None) -> torch.Tensor:
    """Llama4TextMLP: down(silu(gate x) * up x), every product in bf16; `inside` (float32 or float64): in that type with
    h and the output rounded to bf16 (this project's rounding points)."""
    if inside is not None:
        xf = x.to(inside)
        h = (F.silu(F.linear(xf, gate.to(inside))) * F.linear(xf, up.to(inside))).bfloat16().to(inside)
        return F.linear(h, down.to(inside)).bfloat16()
    return F.linear(F.silu(F.linear(x, gate)) * F.linear(x, up), down)


def llama4_moe(x: torch.Tensor, router_w: torch.Tensor, gate_up: torch.Tensor, down: torch.Tensor,
               sh_gate: torch.Tensor, sh_up: torch.Tensor, sh_down: torch.Tensor,
               picks: Optional[torch.Tensor] = None, weights: Optional[torch.Tensor] = None,
               inside: Optional[torch.dtype] = None):
    """(out [n, H] bf16, picks [n, 1]) of Llama4TextMoe on x [n, H] bf16.  `inside` (float32 or float64): the expert
    and shared FFNs in that type with h and y rounded to bf16 once each, as this project computes them (Hugging Face
    also rounds W_gate x, W_up x and silu); the routing, the bf16 x * score and the final add are unchanged."""
    E, H = router_w.shape
    scores, picks = router_scores(x, router_w, picks, weights)
    routed_in = (x.repeat(E, 1) * scores.t().reshape(-1, 1)).view(E, -1, H)
    if inside is not None:
        g, u = torch.bmm(routed_in.to(inside), gate_up.to(inside)).chunk(2, dim=-1)
        routed_out = torch.bmm((u * F.silu(g)).bfloat16().to(inside), down.to(inside)).bfloat16()
    else:
        g, u = torch.bmm(routed_in, gate_up).chunk(2, dim=-1)
        routed_out = torch.bmm(u * F.silu(g), down)
    out = shared_mlp(x, sh_gate, sh_up, sh_down, inside)
    out.add_(routed_out.sum(0))
    return out, picks


def convert_experts(gate_up: torch.Tensor, down: torch.Tensor) -> torch.Tensor:
    """Hugging Face's gate_up_proj [E, H, 2P] and down_proj [E, P, H] as this project's SwiGLU expert_weight
    [E, 3, P, H] (W_gate, W_up, W_down flat-viewed), one copy."""
    E, H, P2 = gate_up.shape
    P = P2 // 2
    return torch.stack([gate_up[:, :, :P].transpose(1, 2), gate_up[:, :, P:].transpose(1, 2),
                        down.transpose(1, 2).reshape(E, P, H)], 1)


def convert_shared(gate: torch.Tensor, up: torch.Tensor, down: torch.Tensor) -> torch.Tensor:
    """The shared MLP's gate / up [Ps, H] and down [H, Ps] weights as a SwiGLU shared_weight [3, Ps, H]."""
    Ps, H = gate.shape
    return torch.stack([gate, up, down.reshape(Ps, H)])


def convert_router(router_w: torch.Tensor) -> torch.Tensor:
    """The router's [E, H] weight as gate_weight [H, E]: the flat reinterpretation the header documents, no transpose."""
    E, H = router_w.shape
    return router_w.view(H, E)
