"""Operator-style API on top of the drop-in surface (SURVEY.md section 8f rank 1): a forward-only `torch.nn.Module` that owns
the layer's parameters, uses them in place (no per-call re-upload like the reference's wrapper, python_bindings.cu:76-120),
supports the bias vectors and GELU the reference kernel has but cannot reach from Python, and can return the routing
decisions next to the output.  Inference only: no autograd (the reference is forward-only as well)."""
from __future__ import annotations

from typing import NamedTuple, Optional

import torch

from .config import MoEConfig
from .router import RouterSpec
from .runtime import MoEContext, SharedExpert


class MoEOutput(NamedTuple):
    out: torch.Tensor                 # [B, T, H] bf16
    topk_idx: torch.Tensor            # [B*T, k] int32   expert picked per token, in pick order
    topk_weight: torch.Tensor         # [B*T, k] bf16    gateOut[t, e_j] (bf16-rounded softmax probability); after a
                                      #                  routed call the caller's weights rounded to bf16; with a
                                      #                  `router` rule the rule's weights w rounded to bf16
    slot: torch.Tensor                # [B*T, k] int32   slot in the (rank, expert) packet; >= capacity means dropped
                                      #                  (INT32_MAX for a -1 pick of a routed call)
    aux_loss: Optional[torch.Tensor] = None   # is_training = 1: f32 [2E+1] = gML[E] | gMeC[E] | load-balancing loss


class FlashMoELayer(torch.nn.Module):
    """One expert-parallel MoE layer: y[t] = sum_{e in topk(t), kept} (p~_e / sum_topk p) * FFN_e(x[t]).

    Parameters are held in the reference's layouts: `gate_weight` [H, E] (consumed flat as [E, H]),
    `expert_weight` [nLx, 2, P, H] (this rank's experts), optional `bias_up` [nLx, P] / `bias_down` [nLx, H].

    With `cfg.hidden_act = 2` (SwiGLU, y = W_down (silu(W_gate x) * (W_up x)), Mixtral / Qwen3-MoE / DeepSeek-V3 experts)
    `expert_weight` is [nLx, 3, P, H]: [i,0] = W_gate, [i,1] = W_up, [i,2] flat-viewed as W_down [H, P]; from Hugging
    Face tensors, once at load time, `torch.stack([w_gate, w_up, w_down.reshape(nLx, P, H)], 1)`.  `bias_up` is then
    [nLx, 2, P] (gate, then up), `shared_weight` [3, Ps, H] and `shared_bias_up` [2, Ps].  h = silu(g) * u is computed
    in fp32 and rounded to bf16 once (Hugging Face rounds W_gate x, silu and the product separately).

    `router`: a `RouterSpec` (sigmoid scores, group-limited top-k, no renormalisation, a route scale, ...) the kernel
    applies to the gate's logits instead of the built-in softmax / top-k / renormalise (`MoEContext.forward_gated`).
    `score_bias` (with a `router` only): hold an fp32 [E] selection bias, `score_bias` (Hugging Face's
    `e_score_correction_bias`), zero-initialised; the caller updates it in place, e.g. from the `counts` buffer.
    `shared_inter`: hold a shared expert of that intermediate size Ps, `shared_weight` [2, Ps, H] (one routed expert's
    layout; plus `shared_bias_up` [Ps] / `shared_bias_down` [H] with `bias`), which every token passes through on every
    route: out[t] = rne_bf16(routed[t] + s[t]) (`MoEContext.forward_tokens`'s `shared_expert`).

    `weight_on_input` (k = 1, E > 1): the router weight scales each routed token's input row, rne_bf16(x[t] * w~), and
    the combine takes weight 1 -- Hugging Face's `Llama4TextMoe` (`MoEContext`'s `weight_on_input`).  On the gated
    and the caller route only.  Llama 4 Scout / Maverick are `hidden_act = 2`, k = 1, `drop_tokens = 0`,
    `router=RouterSpec("sigmoid", renormalize=False)`, `shared_inter = P` and `weight_on_input=True`; their Hugging
    Face tensors convert once at load time (E experts, P = intermediate_size, Ps = the shared MLP's):

        gu, dp = experts.gate_up_proj, experts.down_proj           # [E, H, 2P], [E, P, H]
        expert_weight = torch.stack([gu[:, :, :P].transpose(1, 2), gu[:, :, P:].transpose(1, 2),
                                     dp.transpose(1, 2).reshape(E, P, H)], 1)
        shared_weight = torch.stack([shared_expert.gate_proj.weight, shared_expert.up_proj.weight,
                                     shared_expert.down_proj.weight.reshape(Ps, H)])
        gate_weight = router.weight.view(H, E)                     # [E, H] read flat, not transposed
    """

    def __init__(self, cfg: MoEConfig, rank: int = 0, world: int = 1, device: Optional[int] = None, group=None,
                 bias: bool = False, router: Optional[RouterSpec] = None, score_bias: bool = False,
                 shared_inter: Optional[int] = None, weight_on_input: bool = False):
        super().__init__()
        cfg.check_hot_path()
        if router is not None:
            if not isinstance(router, RouterSpec):
                raise TypeError(f"router must be a RouterSpec, got {type(router).__name__}")
            router.check(cfg.E, cfg.k)
        elif score_bias:
            raise ValueError("score_bias needs a router rule (router=RouterSpec(...))")
        self.cfg = cfg
        self.router = router
        self.ctx = MoEContext(cfg, rank=rank, world=world, device=device, group=group, shared_inter=shared_inter,
                              weight_on_input=weight_on_input)
        dev = self.ctx.device
        nlx = self.ctx.num_local_experts
        scale = cfg.H ** -0.5
        self.gate_weight = torch.nn.Parameter(torch.randn(cfg.H, cfg.E, device=dev).mul_(scale).bfloat16(),
                                              requires_grad=False)
        m = cfg.expert_mats
        up = (2,) if m == 3 else ()   # SwiGLU: a gate and an up bias
        self.expert_weight = torch.nn.Parameter(torch.randn(nlx, m, cfg.P, cfg.H, device=dev).mul_(scale).bfloat16(),
                                                requires_grad=False)
        if bias:
            self.bias_up = torch.nn.Parameter(torch.zeros(nlx, *up, cfg.P, device=dev, dtype=torch.bfloat16),
                                              requires_grad=False)
            self.bias_down = torch.nn.Parameter(torch.zeros(nlx, cfg.H, device=dev, dtype=torch.bfloat16), requires_grad=False)
        else:
            self.bias_up = None
            self.bias_down = None
        self.score_bias = (torch.nn.Parameter(torch.zeros(cfg.E, device=dev, dtype=torch.float32), requires_grad=False)
                           if score_bias else None)
        self.shared_inter = shared_inter
        self.shared_weight = self.shared_bias_up = self.shared_bias_down = None
        if shared_inter is not None:
            self.shared_weight = torch.nn.Parameter(torch.randn(m, shared_inter, cfg.H, device=dev).mul_(scale).bfloat16(),
                                                    requires_grad=False)
            if bias:
                self.shared_bias_up = torch.nn.Parameter(torch.zeros(*up, shared_inter, device=dev, dtype=torch.bfloat16),
                                                         requires_grad=False)
                self.shared_bias_down = torch.nn.Parameter(torch.zeros(cfg.H, device=dev, dtype=torch.bfloat16),
                                                           requires_grad=False)

    @torch.no_grad()
    def forward(self, x: torch.Tensor, return_routing: bool = False, n_tokens: Optional[torch.Tensor] = None,
                topk_idx: Optional[torch.Tensor] = None, topk_weight: Optional[torch.Tensor] = None):
        """x [B, T, H] bf16 on this layer's device with B*T <= S (the capacity is that of B*T tokens,
        `cfg.EC_of(B*T)`).  Asynchronous on torch's current stream unless `return_routing` (reading the routing tables
        synchronises).  `n_tokens`: a one-element int32 tensor on the device with the token count n; x then holds
        B*T = S rows of which the first n are the tokens (see `MoEContext.forward_tokens`), and the call can be captured
        once in a CUDA graph and replayed for any n.  The routing tables then hold the n rows of the last launch.

        `topk_idx` / `topk_weight` [B*T, k] (both or neither): the caller's routing instead of this layer's gate
        (`MoEContext.forward_routed`; -1 = no expert, k = 1 is scaled by its weight too).  The indices may be any
        integer type (int64 from `torch.topk` is converted to int32), the weights any floating type (converted to
        float32); `gate_weight` is not used.  Otherwise, with a `router` rule, the gated forward runs."""
        if x.dim() != 3:
            raise RuntimeError("Input must be 3D [batch, seq, H]")
        if (topk_idx is None) != (topk_weight is None):
            raise RuntimeError("pass both topk_idx and topk_weight, or neither")
        shared = (SharedExpert(self.shared_weight, self.shared_bias_up, self.shared_bias_down)
                  if self.shared_weight is not None else None)
        if topk_idx is not None:
            if topk_idx.is_floating_point() or not topk_weight.is_floating_point():
                raise RuntimeError("topk_idx must be an integer tensor and topk_weight a floating-point one")
            out = self.ctx.forward_routed(x, topk_idx.to(torch.int32).contiguous(),
                                          topk_weight.to(torch.float32).contiguous(), self.expert_weight,
                                          bias_up=self.bias_up, bias_down=self.bias_down, n_tokens=n_tokens,
                                          shared_expert=shared)
        elif self.router is not None:
            out = self.ctx.forward_gated(x, self.gate_weight, self.expert_weight, self.router,
                                         score_bias=self.score_bias, bias_up=self.bias_up, bias_down=self.bias_down,
                                         n_tokens=n_tokens, shared_expert=shared)
        else:
            out = self.ctx.forward_tokens(x, self.gate_weight, self.expert_weight, bias_up=self.bias_up,
                                          bias_down=self.bias_down, n_tokens=n_tokens, shared_expert=shared)
        if not return_routing:
            return out
        return self.routing(out)

    def routing(self, out: torch.Tensor) -> MoEOutput:
        """The routing decisions of this layer's last launch -- an eager call or a replay of a captured graph -- next to
        its output `out`.  Synchronises."""
        self.ctx.synchronize()
        n = self.ctx.launch_record()[1]   # (the device's record: right after a replay as after an eager call)
        idx = torch.from_numpy(self.ctx.read("topk_idx")[:n].copy())
        w = torch.from_numpy(self.ctx.read("topk_w")[:n].view("int16").copy()).view(torch.bfloat16)
        slot = torch.from_numpy(self.ctx.read("slot")[:n].copy())
        aux = torch.from_numpy(self.ctx.read("aux_loss")) if self.cfg.is_training else None
        return MoEOutput(out, idx, w, slot, aux)

    def extra_repr(self) -> str:
        c = self.cfg
        return (f"S={c.S}, H={c.H}, P={c.P}, E={c.E}, k={c.k}, act={('relu', 'gelu', 'swiglu')[c.hidden_act]}, "
                f"rank={self.ctx.rank}/{self.ctx.world}"
                + (f", shared_inter={self.shared_inter}" if self.shared_inter is not None else "")
                + (", weight_on_input=True" if getattr(self.ctx, "weight_on_input", False) else ""))
