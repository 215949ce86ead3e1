#!/usr/bin/env python
"""Llama 4 MoE layers (the router weight on the input, fm_set_weight_on_input) against the same forward with the weight
on the output and against Hugging Face's formulation in torch: device time per token count.

    python scripts/bench_llama4.py [--configs SCOUT,MAVERICK] [--tokens 1,128,4096] [--steps K] [--warmup W] [--rounds R]

Shapes: Scout (E 16) and Maverick (E 128), k 1, H 5120, P = Ps = 8192, SwiGLU, drop_tokens 0, the gated route with
Llama 4's rule (sigmoid, no renormalisation) and a shared expert; Maverick's 32 GB of expert weights are generated on
the device.  For every config and n three arms run alternating, `rounds` times `steps` forwards each (medians reported):
  ms_input   the fused forward with the weight on the input (Llama 4's layer);
  ms_output  the same context with the setting off (the weight on the output): the gap is the cost of scaling the rows;
  ms_torch   Llama4TextMoe's arithmetic in torch eager over the device's routing: x * score in bf16, each expert's SwiGLU
             on its tokens, the shared MLP on x, the bf16 add.
TFLOP/s are algorithmic: 6 * P * H per kept pick plus 6 * Ps * H per token, over the median.  One GPU; prints one JSON
line with the card's name and power limit next to the figures; writes no files.
"""
from __future__ import annotations

import argparse
import functools
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from flashmoe_b200.config import MoEConfig  # noqa: E402
from flashmoe_b200.router import RouterSpec  # noqa: E402
from scripts import bench_common as common  # noqa: E402

RULE = RouterSpec("sigmoid", renormalize=False)   # Llama 4's router: the top-1 logit's sigmoid, no renormalisation
SHAPES = {name: MoEConfig(num_experts=E, expert_top_k=1, sequence_len=4096, hidden_size=5120, intermediate_size=8192,
                          hidden_act=2, drop_tokens=0)
          for name, E in (("SCOUT", 16), ("MAVERICK", 128))}


def weights(cfg, dev):
    """Seeded x [S, H], gate weights [H, E], experts [E, 3, P, H] and the shared expert [3, Ps, H], on the device."""
    g = torch.Generator(device=dev).manual_seed(0x11A4)
    s = cfg.H ** -0.5
    x = torch.randn(cfg.S, cfg.H, generator=g, device=dev).bfloat16()
    wg = (torch.randn(cfg.H, cfg.E, generator=g, device=dev) * s).bfloat16()
    we = torch.empty(cfg.E, 3, cfg.P, cfg.H, dtype=torch.bfloat16, device=dev)
    for e in range(cfg.E):   # (one expert at a time: no fp32 copy of the weights)
        we[e] = (torch.randn(3, cfg.P, cfg.H, generator=g, device=dev) * s).bfloat16()
    ws = (torch.randn(3, cfg.P, cfg.H, generator=g, device=dev) * s).bfloat16()
    return x, wg, we, ws


def torch_llama4(x, idx, w, we, ws):
    """Llama4TextMoe's arithmetic on the routing (idx, w) [n, 1]: the weight scales the input in bf16."""
    E, _, P, H = we.shape
    out = F.linear(F.silu(F.linear(x, ws[0])) * F.linear(x, ws[1]), ws[2].reshape(-1).view(H, P))
    routed = torch.zeros_like(x)
    xs = x * w.to(x.dtype)
    for e in range(E):
        t = (idx[:, 0] == e).nonzero()[:, 0]
        if t.numel():
            xe = xs[t]
            h = F.linear(xe, we[e, 1]) * F.silu(F.linear(xe, we[e, 0]))
            routed.index_copy_(0, t, F.linear(h, we[e, 2].reshape(-1).view(H, P)))
    return out.add_(routed)


def run_config(name, tokens, steps, warmup, rounds, dev):
    from flashmoe_b200.runtime import MoEContext, SharedExpert

    cfg = SHAPES[name]
    ctx = MoEContext(cfg, device=dev.index, timeout_ms=60000, shared_inter=cfg.P)
    x, wg, we, ws = weights(cfg, dev)
    se = SharedExpert(ws)
    sync = functools.partial(torch.cuda.synchronize, dev)
    entries = []
    for n in tokens:
        xn = x[:n]
        out = torch.empty_like(xn)

        def fused(on):
            if ctx.weight_on_input != on:
                ctx.set_weight_on_input(on)
            return ctx.forward_gated(xn, wg, we, RULE, out=out, shared_expert=se)

        fused(True)
        ctx.synchronize()
        idx = torch.from_numpy(ctx.read("topk_idx")[:n].copy()).to(dev)
        w = torch.from_numpy(ctx.read("topk_w")[:n].view("int16").copy()).view(torch.bfloat16).to(dev)
        kept = int((ctx.read("slot")[:n] < cfg.EC_of(n)).sum())
        arms = {"ms_input": lambda: fused(True), "ms_output": lambda: fused(False),
                "ms_torch": lambda: torch_llama4(xn, idx, w, we, ws)}
        times = common.alternate(arms, warmup, rounds, sync, lambda fn: common.device_ms(fn, steps, sync))
        ctx.check()
        flop = 6.0 * cfg.H * (cfg.P * kept + cfg.P * n)
        e = {"tokens": n, "kept_picks": kept}
        e.update(common.medians(times))
        for k in ("ms_input", "ms_output", "ms_torch"):
            e["tflops_" + k[3:]] = flop / (e[k] * 1e-3) / 1e12
        e["input_minus_output_us"] = (e["ms_input"] - e["ms_output"]) * 1e3
        entries.append(e)
    ctx.close()
    del x, wg, we, ws, se
    torch.cuda.empty_cache()
    conf = {"name": name, "experts": cfg.E, "top_k": 1, "d_model": cfg.H, "ffn": cfg.P, "shared_inter": cfg.P,
            "route": "gated (Llama 4 rule) + shared expert", "drop_tokens": 0}
    return {"config": conf, "entries": entries}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--configs", default="SCOUT,MAVERICK")
    common.add_run_args(ap, tokens="1,128,4096", steps=20, warmup=3, rounds=3)
    args = ap.parse_args()
    names = common.parse_names(ap, "--configs", args.configs, SHAPES)
    tokens = {c: common.parse_tokens(ap, args.tokens, SHAPES[c].S) for c in names}
    common.check_counts(ap, args, warmup=True)
    if not torch.cuda.is_available():
        return common.no_cuda("bench_llama4.py")
    dev = torch.device("cuda", torch.cuda.current_device())
    runs = [run_config(c, tokens[c], args.steps, args.warmup, args.rounds, dev) for c in names]
    print(json.dumps({"metric": "moe_layer_fwd_llama4_ms", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup,
                      "rounds": args.rounds, "card": common.card(dev), "runs": runs}), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
