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
import functools
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402   (seeded inputs; bench.py itself is not changed by this script)
from scripts import bench_common as common  # noqa: E402


def torch_router(x, wg, k):
    p = torch.softmax(x.float() @ wg.float(), dim=-1)
    w, i = torch.topk(p, k, dim=-1)
    return i.to(torch.int32), (w / w.sum(-1, keepdim=True)).float()


def run_config(name, tokens, steps, warmup, rounds, dev):
    from flashmoe_b200.runtime import MoEContext

    cfg = bench.BASELINE_CONFIGS[name]
    ctx = MoEContext(cfg, device=dev.index, timeout_ms=30000)
    xd, wgd, wed = common.inputs(name, cfg, dev)

    sync = functools.partial(torch.cuda.synchronize, dev)

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
        times = common.alternate(arms, warmup, rounds, sync, lambda fn: common.device_ms(fn, steps, sync))
        ctx.check()
        e = {"tokens": n, "ec": cfg.EC_of(n), "parity_slot_counts_recv_cnt": parity}
        e.update(common.medians(times))
        e["routed_minus_router_us"] = (e["ms_routed"] - e["ms_router"]) * 1e3
        entries.append(e)
    ctx.close()
    torch.cuda.empty_cache()
    return {"config": bench.config_dict(name, cfg, 1), "entries": entries}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--configs", default="B,E128")
    common.add_run_args(ap, tokens="1,128,4096", steps=200, warmup=32, rounds=3)
    args = ap.parse_args()
    names = common.parse_names(ap, "--configs", args.configs, bench.BASELINE_CONFIGS)
    tokens = {c: common.parse_tokens(ap, args.tokens, bench.BASELINE_CONFIGS[c].S) for c in names}
    common.check_counts(ap, args)
    if not torch.cuda.is_available():
        return common.no_cuda("bench_routed.py")
    dev = torch.device("cuda", torch.cuda.current_device())
    runs = [run_config(c, tokens[c], args.steps, args.warmup, args.rounds, dev) for c in names]
    print(json.dumps({"metric": "moe_layer_fwd_routed_ms", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup,
                      "rounds": args.rounds, "card": common.card(dev), "runs": runs}), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
