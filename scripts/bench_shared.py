#!/usr/bin/env python
"""Shared experts fused into the forward kernel against the same forward plus a torch shared FFN: device time per token
count.

    python scripts/bench_shared.py [--configs B,DSV3] [--tokens 1,128,4096] [--steps K] [--warmup W] [--rounds R]

For every config and n three arms run alternating, `rounds` times `steps` forwards each (medians reported):
  ms_fused       forward_*(n, shared_expert=...): the shared expert's tiles in the same persistent kernel;
  ms_torch       the same forward without one, then F.linear -> act -> F.linear (bf16 out) and out + s in bf16, in torch
                 on the same stream;
  ms_plain       the forward without a shared expert (the floor).
Configs: B (bench.py's, built-in router, Ps = P) and DSV3 (bench_common.py's DeepSeek-V3 layer shape, gated with the V3
rule, Ps = 2048).  The torch arm is also a reference: the fraction of output elements bit-identical to the fused arm's,
and the fraction within one bf16 ulp of s, are reported.  One GPU; prints one JSON line with the card's name and power
limit next to the figures; writes no files.
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

import bench  # noqa: E402   (seeded inputs; bench.py itself is not changed by this script)
from scripts import bench_common as common  # noqa: E402
from scripts.bench_common import DSV3, RULE  # noqa: E402


def run_config(name, tokens, steps, warmup, rounds, dev):
    from flashmoe_b200.runtime import MoEContext, SharedExpert

    cfg = bench.BASELINE_CONFIGS[name] if name in bench.BASELINE_CONFIGS else DSV3
    ps = cfg.P if name in bench.BASELINE_CONFIGS else 2048
    ctx = MoEContext(cfg, device=dev.index, timeout_ms=30000, shared_inter=ps)
    xd, wgd, wed = common.inputs(name, cfg, dev)
    g = torch.Generator(device=dev).manual_seed(0x5AED)
    se = SharedExpert((torch.randn(2, ps, cfg.H, generator=g, device=dev) * cfg.H ** -0.5).bfloat16())
    w_up, w_down = se.w[0], se.w[1].reshape(-1).view(cfg.H, ps)   # [1] flat-viewed as W_down [H, Ps]
    act = F.gelu if cfg.hidden_act else F.relu
    bias = (torch.randn(cfg.E, generator=torch.Generator(device=dev).manual_seed(7), device=dev) * 0.05).float()
    gated = name not in bench.BASELINE_CONFIGS

    sync = functools.partial(torch.cuda.synchronize, dev)

    entries = []
    for n in tokens:
        xn = xd[:n]
        out_n, out_f = torch.empty_like(xn), torch.empty_like(xn)

        def forward(out, shared=None):
            kw = dict(out=out, shared_expert=shared)
            if gated:
                return ctx.forward_gated(xn, wgd, wed, RULE, score_bias=bias, **kw)
            return ctx.forward_tokens(xn, wgd, wed, **kw)

        def torch_arm():
            r = forward(out_n)
            s = F.linear(act(F.linear(xn, w_up)), w_down)
            return r + s

        fused = forward(out_f, se).clone()
        ref = torch_arm()
        ctx.synchronize()
        s = torch.from_numpy(ctx.read("shared_y")[:n].copy()).view(torch.bfloat16).to(dev).float()
        ulp = torch.where(s == 0, torch.full_like(s, 2.0 ** -133),
                          torch.ldexp(torch.ones_like(s), torch.frexp(s).exponent - 8))
        same = (fused.view(torch.int16) == ref.view(torch.int16)).float().mean().item() if n else 1.0
        within = ((fused.float() - ref.float()).abs() <= ulp).float().mean().item() if n else 1.0

        arms = {"ms_fused": lambda: forward(out_f, se), "ms_torch": torch_arm, "ms_plain": lambda: forward(out_n)}
        times = common.alternate(arms, warmup, rounds, sync, lambda fn: common.device_ms(fn, steps, sync))
        ctx.check()
        e = {"tokens": n, "bitwise_equal_to_torch": same, "within_one_ulp_of_s": within}
        e.update(common.medians(times))
        e["torch_minus_fused_us"] = (e["ms_torch"] - e["ms_fused"]) * 1e3
        e["fused_minus_plain_us"] = (e["ms_fused"] - e["ms_plain"]) * 1e3
        entries.append(e)
    ctx.close()
    del xd, wgd, wed
    torch.cuda.empty_cache()
    conf = {"name": name, "experts": cfg.E, "top_k": cfg.k, "tokens": cfg.S, "d_model": cfg.H, "ffn": cfg.P,
            "shared_inter": ps, "route": "gated (DeepSeek-V3 rule)" if gated else "router"}
    return {"config": conf, "entries": entries}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--configs", default="B,DSV3")
    common.add_run_args(ap, tokens="1,128,4096", steps=200, warmup=32, rounds=3)
    args = ap.parse_args()
    known = {**bench.BASELINE_CONFIGS, "DSV3": DSV3}
    names = common.parse_names(ap, "--configs", args.configs, known)
    tokens = {c: common.parse_tokens(ap, args.tokens, known[c].S) for c in names}
    common.check_counts(ap, args)
    if not torch.cuda.is_available():
        return common.no_cuda("bench_shared.py")
    dev = torch.device("cuda", torch.cuda.current_device())
    runs = [run_config(c, tokens[c], args.steps, args.warmup, args.rounds, dev) for c in names]
    print(json.dumps({"metric": "moe_layer_fwd_shared_ms", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup,
                      "rounds": args.rounds, "card": common.card(dev), "runs": runs}), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
