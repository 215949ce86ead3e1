#!/usr/bin/env python
"""Forwards on the caller's routing (MoEContext.forward_routed) against the built-in router: device time per token count.

    python scripts/bench_routed.py [--configs B,E128] [--tokens 1,128,4096] [--steps K] [--warmup W] [--rounds R]

For every config and n three arms run alternating, `rounds` times `steps` forwards each (medians reported):
  ms_router          forward_tokens(n): the in-kernel router;
  ms_routed          forward_routed(n) fed with the kernel's own routing from the router arm (its topk_idx, and its
                     topk_w as float32);
  ms_torch_router    a torch router on the device (x @ Wg, softmax, topk, renormalise) followed by forward_routed(n).
Parity line per (config, n): the routed arm's slot / counts / recv_cnt must be bit-identical to the router arm's.  One
GPU; inputs are bench.py's seeded synthetic tensors.  Prints one JSON line with the card's name and power limit next to
the figures; writes no files.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402   (seeded inputs; bench.py itself is not changed by this script)
from scripts.bench_varlen import card, parse_tokens  # noqa: E402


def torch_router(x, wg, k):
    p = torch.softmax(x.float() @ wg.float(), dim=-1)
    w, i = torch.topk(p, k, dim=-1)
    return i.to(torch.int32), (w / w.sum(-1, keepdim=True)).float()


def run_config(name, tokens, steps, warmup, rounds, dev):
    from flashmoe_b200.runtime import MoEContext

    cfg = bench.BASELINE_CONFIGS[name]
    S, H = cfg.S, cfg.H
    ctx = MoEContext(cfg, device=dev.index, timeout_ms=30000)
    x, wg, we = bench.make_inputs(cfg, cfg.E, 0)
    xd, wgd, wed = x.to(dev).view(S, H), wg.to(dev), we.to(dev)
    del we

    def device_ms(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize(dev)
        return e0.elapsed_time(e1) / steps

    entries = []
    for n in tokens:
        xn = xd[:n]
        out_n = torch.empty_like(xn)
        ctx.forward_tokens(xn, wgd, wed, out=out_n)
        ctx.synchronize()
        want = {k: ctx.read(k)[:n].copy() for k in ("slot",)}
        want.update(counts=ctx.read("counts").copy(), recv_cnt=ctx.read("recv_cnt").copy())
        idx = torch.from_numpy(ctx.read("topk_idx")[:n].copy()).to(dev)
        w = torch.from_numpy(ctx.read("topk_w")[:n].view(np.int16).copy()).view(torch.bfloat16).float().to(dev)
        ctx.forward_routed(xn, idx, w, wed, out=out_n)
        ctx.synchronize()
        parity = {k: bool(np.array_equal(ctx.read(k)[: (n if k == "slot" else None)], v)) for k, v in want.items()}

        def torch_arm():
            i, ww = torch_router(xn, wgd, cfg.k)
            ctx.forward_routed(xn, i, ww, wed, out=out_n)

        arms = {"ms_router": lambda: ctx.forward_tokens(xn, wgd, wed, out=out_n),
                "ms_routed": lambda: ctx.forward_routed(xn, idx, w, wed, out=out_n),
                "ms_torch_router": torch_arm}
        for fn in arms.values():
            for _ in range(warmup):
                fn()
        torch.cuda.synchronize(dev)
        times = {k: [] for k in arms}
        for _ in range(rounds):
            for k, fn in arms.items():
                times[k].append(device_ms(fn))
        ctx.check()
        e = {"tokens": n, "ec": cfg.EC_of(n), "parity_slot_counts_recv_cnt": parity}
        for k, v in times.items():
            e[k] = statistics.median(v)
            e[k + "_runs"] = v
        e["routed_minus_router_us"] = (e["ms_routed"] - e["ms_router"]) * 1e3
        entries.append(e)
    ctx.close()
    torch.cuda.empty_cache()
    return {"config": bench.config_dict(name, cfg, 1), "entries": entries}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--configs", default="B,E128")
    ap.add_argument("--tokens", default="1,128,4096", metavar="N1,N2,..")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    names = [c for c in args.configs.split(",") if c]
    bad = [c for c in names if c not in bench.BASELINE_CONFIGS]
    if not names or bad:
        ap.error(f"--configs: unknown {bad}; choose from {sorted(bench.BASELINE_CONFIGS)}")
    tokens = {c: parse_tokens(ap, args.tokens, bench.BASELINE_CONFIGS[c].S) for c in names}
    if args.steps < 1 or args.rounds < 1:
        ap.error("--steps and --rounds must be >= 1")
    if not torch.cuda.is_available():
        print("bench_routed.py: no CUDA device; the MoE forward path has no CPU fallback", file=sys.stderr)
        return 3
    dev = torch.device("cuda", torch.cuda.current_device())
    runs = [run_config(c, tokens[c], args.steps, args.warmup, args.rounds, dev) for c in names]
    print(json.dumps({"metric": "moe_layer_fwd_routed_ms", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup,
                      "rounds": args.rounds, "card": card(dev), "runs": runs}), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
