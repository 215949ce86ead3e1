#!/usr/bin/env python
"""SwiGLU experts (hidden_act = 2) in the fused forward against the same context shape with GELU and against a torch
eager SwiGLU over the device's routing: device time per forward and algorithmic TFLOP/s.

    python scripts/bench_swiglu.py [--shapes mixtral,dsv3] [--tokens 1,128,4096] [--steps K] [--warmup W] [--rounds R]

For every shape and n three arms run alternating, `rounds` times `steps` forwards each (medians reported):
  ms_swiglu   the fused forward of a hidden_act = 2 context, expert weights [E, 3, P, H];
  ms_gelu     the same shape with hidden_act = 1, weights [E, 2, P, H];
  ms_torch    the SwiGLU layer in torch eager over the fused arm's routing (read once, outside the timing): per expert
              index_select of its rows, three F.linear, silu, and a weighted index_add_ into the output.
Shapes: Mixtral-8x7B (E 8, k 2, H 4096, P 14336, S 4096, built-in router) and DeepSeek-V3 (E 256, k 8, H 7168, P 2048,
the V3 rule, shared Ps 2048; the torch arm adds the shared expert).  TFLOP/s are algorithmic, from the picks the
kernel kept: 6 P H per kept pick for SwiGLU, 4 P H for GELU (plus the shared expert's on every token).  One GPU; prints
one JSON line with the card's name and power limit next to the figures; writes no files.
"""
from __future__ import annotations

import argparse
import functools
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from flashmoe_b200.config import MoEConfig  # noqa: E402
from scripts import bench_common as common  # noqa: E402
from scripts.bench_common import DSV3, RULE  # noqa: E402

SHAPES = {
    "mixtral": (MoEConfig(num_experts=8, expert_top_k=2, sequence_len=4096, hidden_size=4096, intermediate_size=14336),
                None),
    "dsv3": (DSV3, 2048),
}


def run_shape(name, tokens, steps, warmup, rounds, dev):
    from flashmoe_b200.runtime import MoEContext, SharedExpert

    base, ps = SHAPES[name]
    E, k, H, P, S = base.E, base.k, base.H, base.P, base.S
    g = torch.Generator(device=dev).manual_seed(0x5EED)
    x = torch.randn(S, H, generator=g, device=dev, dtype=torch.bfloat16)
    wg = (torch.randn(H, E, generator=g, device=dev) * H ** -0.5).bfloat16()
    s = H ** -0.5
    we3 = torch.randn(E, 3, P, H, generator=g, device=dev, dtype=torch.bfloat16).mul_(s)
    ws3 = None if ps is None else torch.randn(3, ps, H, generator=g, device=dev, dtype=torch.bfloat16).mul_(s)
    gated = ps is not None
    arms = {}
    for act in (2, 1):
        cfg = base.replace(hidden_act=act)
        ctx = MoEContext(cfg, device=dev.index, timeout_ms=30000, shared_inter=ps)
        we = we3 if act == 2 else we3[:, 1:].contiguous()   # GELU: [W_up, W_down]
        se = None if ps is None else SharedExpert(ws3 if act == 2 else ws3[1:].contiguous())
        arms[act] = (ctx, we, se)

    def fused(act, n):
        ctx, we, se = arms[act]
        if gated:
            return ctx.forward_gated(x[:n], wg, we, RULE, shared_expert=se)
        return ctx.forward_tokens(x[:n], wg, we, shared_expert=se)

    sync = functools.partial(torch.cuda.synchronize, dev)

    entries = []
    for n in tokens:
        ctx = arms[2][0]
        fused(2, n)
        ctx.synchronize()
        idx = torch.from_numpy(ctx.read("topk_idx")[:n].copy()).to(dev).long()
        slot = torch.from_numpy(ctx.read("slot")[:n].copy()).to(dev)
        tw = torch.from_numpy(ctx.read("topk_w")[:n].view("int16").copy()).view(torch.bfloat16).to(dev).float()
        mcw = torch.from_numpy(ctx.read("mcw")[:n].copy()).to(dev)
        kept = slot < base.EC_of(n)
        w = torch.where(kept, tw / mcw[:, None], torch.zeros((), device=dev))
        picks = int(kept.sum())
        groups = []
        for e in range(E):
            tok, j = ((idx == e) & kept).nonzero(as_tuple=True)
            if tok.numel():
                groups.append((e, tok, w[tok, j].to(torch.bfloat16)[:, None]))

        def torch_arm():
            out = torch.zeros(n, H, device=dev, dtype=torch.bfloat16)
            for e, tok, we_ in groups:
                xe = x.index_select(0, tok)
                h = F.silu(F.linear(xe, we3[e, 0])) * F.linear(xe, we3[e, 1])
                out.index_add_(0, tok, F.linear(h, we3[e, 2].view(H, P)) * we_)
            if ws3 is not None:
                xs = x[:n]
                out += F.linear(F.silu(F.linear(xs, ws3[0])) * F.linear(xs, ws3[1]), ws3[2].view(H, ps))
            return out

        fns = {"swiglu": lambda: fused(2, n), "gelu": lambda: fused(1, n), "torch": torch_arm}
        ms = common.alternate(fns, warmup, rounds, sync, lambda fn: common.device_ms(fn, steps, sync))
        med = {a: statistics.median(v) for a, v in ms.items()}
        shared_flops = 0 if ps is None else 2 * n * ps * H
        f_glu = 6.0 * P * H * picks + 3 * shared_flops
        f_gelu = 4.0 * P * H * picks + 2 * shared_flops
        entries.append({"shape": name, "n": n, "kept_picks": picks,
                        "ms_swiglu": round(med["swiglu"], 4), "ms_gelu": round(med["gelu"], 4),
                        "ms_torch": round(med["torch"], 4),
                        "tflops_swiglu": round(f_glu / med["swiglu"] * 1e-9, 1),
                        "tflops_gelu": round(f_gelu / med["gelu"] * 1e-9, 1),
                        "tflops_torch": round(f_glu / med["torch"] * 1e-9, 1),
                        "spread_ms": {a: [round(min(v), 4), round(max(v), 4)] for a, v in ms.items()}})
        print(json.dumps(entries[-1]), file=sys.stderr)
    for ctx, _, _ in arms.values():
        ctx.close()
    return entries


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--shapes", default="mixtral,dsv3")
    common.add_run_args(ap, tokens="1,128,4096", steps=20, warmup=3, rounds=3)
    a = ap.parse_args(argv)
    shapes = common.parse_names(ap, "--shapes", a.shapes, SHAPES)
    tokens = common.parse_tokens(ap, a.tokens, 4096)
    common.check_counts(ap, a)
    if not torch.cuda.is_available():
        return common.no_cuda("bench_swiglu.py")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    res = {"card": common.card(dev), "results": []}
    for s in shapes:
        res["results"] += run_shape(s, tokens, a.steps, a.warmup, a.rounds, dev)
    print(json.dumps(res))
    return 0


if __name__ == "__main__":
    sys.exit(main())
