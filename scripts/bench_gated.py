#!/usr/bin/env python
"""Gated forwards (MoEContext.forward_gated) against the built-in router and a torch router: device time per token count.

    python scripts/bench_gated.py [--configs E128,DSV3] [--tokens 1,128,4096] [--steps K] [--warmup W] [--rounds R]

For every config and n three arms run alternating, `rounds` times `steps` forwards each (medians reported):
  ms_router          forward_tokens(n): the in-kernel softmax router;
  ms_gated           forward_gated(n) with DeepSeek-V3's rule (sigmoid, score bias, n_group 8, topk_group 4, top-2
                     group scores, renormalise, scale 2.5);
  ms_torch_router    DeepSeek's router formula (its Gate.forward) in torch on the device, then forward_routed(n).
Configs: bench.py's (E128: 128 experts, top-2, d_model 2048, ffn 2048) and DSV3 (bench_common.py): DeepSeek-V3's layer
shape on one GPU (E = 256, k = 8, H = 7168, P = 2048, S = 4096; 15 GB of expert weights, generated on the device from a
seeded generator).  The gated arm's picks are compared with the torch arm's (fraction of tokens with the same top-k
set).  One GPU; prints one JSON line with the card's name and power limit next to the figures; writes no files.
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

import bench  # noqa: E402   (seeded inputs; bench.py itself is not changed by this script)
from scripts import bench_common as common  # noqa: E402
from scripts.bench_common import DSV3, RULE  # noqa: E402


def deepseek_router(x, wg_eff, bias, rule, k):
    """DeepSeek-V3's Gate.forward: sigmoid scores, biased group scores (sum of the top 2), topk_group groups, top-k of
    the biased scores inside them, weights = the unbiased scores renormalised and scaled."""
    scores = (x.float() @ wg_eff.float().t()).sigmoid()
    original = scores
    s = scores + bias
    n = s.shape[0]
    gs = s.view(n, rule.n_group, -1).topk(2, dim=-1)[0].sum(dim=-1)
    gidx = gs.topk(rule.topk_group, dim=-1)[1]
    mask = s.new_ones(n, rule.n_group, dtype=torch.bool).scatter_(1, gidx, False)
    s = s.view(n, rule.n_group, -1).masked_fill(mask.unsqueeze(-1), float("-inf")).flatten(1)
    idx = s.topk(k, dim=-1)[1]
    w = original.gather(1, idx)
    w = w / w.sum(dim=-1, keepdim=True) * rule.scale
    return idx.to(torch.int32), w.float()


def run_config(name, tokens, steps, warmup, rounds, dev):
    from flashmoe_b200.runtime import MoEContext

    cfg = bench.BASELINE_CONFIGS[name] if name in bench.BASELINE_CONFIGS else DSV3
    ctx = MoEContext(cfg, device=dev.index, timeout_ms=30000)
    xd, wgd, wed = common.inputs(name, cfg, dev)
    wg_eff = wgd.view(-1).view(cfg.E, cfg.H)
    bias = (torch.randn(cfg.E, generator=torch.Generator(device=dev).manual_seed(7), device=dev) * 0.05).float()

    sync = functools.partial(torch.cuda.synchronize, dev)

    entries = []
    for n in tokens:
        xn = xd[:n]
        out_n = torch.empty_like(xn)
        ctx.forward_gated(xn, wgd, wed, RULE, score_bias=bias, out=out_n)
        ctx.synchronize()
        got = torch.from_numpy(ctx.read("topk_idx")[:n].copy()).long()
        i_t, _ = deepseek_router(xn, wg_eff, bias, RULE, cfg.k)
        same = (got.sort(dim=1).values == i_t.cpu().long().sort(dim=1).values).all(dim=1).float().mean().item() \
            if n else 1.0

        def torch_arm():
            i, w = deepseek_router(xn, wg_eff, bias, RULE, cfg.k)
            ctx.forward_routed(xn, i, w, wed, out=out_n)

        arms = {"ms_router": lambda: ctx.forward_tokens(xn, wgd, wed, out=out_n),
                "ms_gated": lambda: ctx.forward_gated(xn, wgd, wed, RULE, score_bias=bias, out=out_n),
                "ms_torch_router": torch_arm}
        times = common.alternate(arms, warmup, rounds, sync, lambda fn: common.device_ms(fn, steps, sync))
        ctx.check()
        e = {"tokens": n, "ec": cfg.EC_of(n), "same_picks_as_torch": same}
        e.update(common.medians(times))
        e["gated_minus_router_us"] = (e["ms_gated"] - e["ms_router"]) * 1e3
        e["torch_minus_gated_us"] = (e["ms_torch_router"] - e["ms_gated"]) * 1e3
        entries.append(e)
    ctx.close()
    del xd, wgd, wed
    torch.cuda.empty_cache()
    conf = {"name": name, "experts": cfg.E, "top_k": cfg.k, "tokens": cfg.S, "d_model": cfg.H, "ffn": cfg.P}
    return {"config": conf, "rule": RULE.__dict__, "entries": entries}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--configs", default="E128,DSV3")
    common.add_run_args(ap, tokens="1,128,4096", steps=200, warmup=32, rounds=3)
    args = ap.parse_args()
    known = {**bench.BASELINE_CONFIGS, "DSV3": DSV3}
    names = common.parse_names(ap, "--configs", args.configs, known)
    tokens = {c: common.parse_tokens(ap, args.tokens, known[c].S) for c in names}
    common.check_counts(ap, args)
    if not torch.cuda.is_available():
        return common.no_cuda("bench_gated.py")
    dev = torch.device("cuda", torch.cuda.current_device())
    runs = [run_config(c, tokens[c], args.steps, args.warmup, args.rounds, dev) for c in names]
    print(json.dumps({"metric": "moe_layer_fwd_gated_ms", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup,
                      "rounds": args.rounds, "card": common.card(dev), "runs": runs}), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
