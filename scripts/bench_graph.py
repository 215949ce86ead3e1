#!/usr/bin/env python
"""Forwards replayed from CUDA graphs against eager calls, at decode and prefill token counts.

    python scripts/bench_graph.py [--config B] [--layers 8] [--tokens 1,8,128,4096] [--steps K] [--warmup W] [--rounds R]

One context of --config runs an L-layer stack: one weight set per layer, every layer through the same context on one
stream.  Every layer reads the same seeded activations, so each does the expert work of one forward of n tokens.  A
step is one pass through the L layers.  For every n three arms
run alternating, `rounds` windows of `steps` steps each:
  eager        forward_tokens(n) per layer, issued from Python;
  graph_per_n  one CUDA graph of the L-layer stack captured for this n (host-side count), replayed;
  graph_dev_n  one CUDA graph of the stack captured once with the count in device memory (forward_tokens(...,
               n_tokens=<int32 tensor>), x and out of S rows), replayed after setting n on the device.
Reported per arm: the median and the range over the windows of the wall time per step (host clock around a
synchronised window) and of the device time per step (CUDA events), and the same per layer.  Inputs are seeded
synthetic tensors.  Prints one JSON line with the card's name and power limit next to the figures; writes no files.
Single GPU.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402   (configs and their description; bench.py itself is not changed by this script)
from scripts import bench_common as common  # noqa: E402


def run_graph(name, layers, tokens, steps, warmup, rounds, dev):
    from flashmoe_b200.runtime import MoEContext

    cfg = bench.BASELINE_CONFIGS[name]
    S, H, P, E = cfg.S, cfg.H, cfg.P, cfg.E
    ctx = MoEContext(cfg, device=dev.index, timeout_ms=30000)
    g = torch.Generator(device=dev).manual_seed(20)
    wgs = [(torch.randn(H, E, device=dev, generator=g) * H ** -0.5).bfloat16() for _ in range(layers)]
    wes = [(torch.randn(E, 2, P, H, device=dev, generator=g) * H ** -0.5).bfloat16() for _ in range(layers)]
    # Every layer reads the same seeded activations (S rows) and writes its own output buffer.  Chaining the layers'
    # outputs instead skews the routing of random weights layer by layer until most tokens are dropped, and the stack
    # would then time less expert work than one forward of real activations.
    x = torch.randn(S, H, device=dev, generator=g).bfloat16()
    outs = [torch.empty(S, H, dtype=torch.bfloat16, device=dev) for _ in range(layers)]
    n_dev = torch.zeros(1, dtype=torch.int32, device=dev)

    def stack(n, device_count):
        for l in range(layers):
            src, dst = x, outs[l]
            if device_count:
                ctx.forward_tokens(src, wgs[l], wes[l], out=dst, n_tokens=n_dev)
            else:
                ctx.forward_tokens(src[:n], wgs[l], wes[l], out=dst[:n])

    def capture(n, device_count):
        stack(n, device_count)   # warm-up outside capture (tensor maps encoded, library loaded)
        torch.cuda.synchronize(dev)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            stack(n, device_count)
        return graph

    graph_dev = capture(S, True)

    def window(fn):
        """(wall, device) ms per step; the wall clock runs from a synchronised start to the synchronise that ends the
        event window."""
        torch.cuda.synchronize(dev)
        t = [time.perf_counter()]

        def settle():
            torch.cuda.synchronize(dev)
            t.append(time.perf_counter())

        device = common.device_ms(fn, steps, settle)
        return (t[1] - t[0]) * 1e3 / steps, device

    entries = []
    for n in tokens:
        graph_n = capture(n, False)
        arms = {"eager": lambda: stack(n, False), "graph_per_n": graph_n.replay, "graph_dev_n": graph_dev.replay}
        n_dev.fill_(n)
        runs = common.alternate(arms, warmup, rounds, ctx.synchronize, window)
        ctx.synchronize()   # raises if a launch reported a problem
        e = {"tokens": n}
        for k, r in runs.items():
            for i, what in enumerate(("wall", "device")):
                v = [w[i] for w in r]
                e[f"{k}_{what}_ms_per_step"] = statistics.median(v)
                e[f"{k}_{what}_ms_per_step_range"] = [min(v), max(v)]
                e[f"{k}_{what}_ms_per_layer"] = statistics.median(v) / layers
        entries.append(e)
        del graph_n
    ctx.close()
    return entries


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--config", default="B", choices=sorted(bench.BASELINE_CONFIGS))
    ap.add_argument("--layers", type=int, default=8)
    common.add_run_args(ap, tokens="1,8,128,4096", steps=50, warmup=5, rounds=5)
    args = ap.parse_args()
    tokens = common.parse_tokens(ap, args.tokens, bench.BASELINE_CONFIGS[args.config].S)
    if args.layers < 1:
        ap.error("--layers must be >= 1")
    common.check_counts(ap, args, warmup=True)
    if not torch.cuda.is_available():
        return common.no_cuda("bench_graph.py")
    dev = torch.device("cuda", torch.cuda.current_device())
    entries = run_graph(args.config, args.layers, tokens, args.steps, args.warmup, args.rounds, dev)
    cfg = bench.BASELINE_CONFIGS[args.config]
    line = {"metric": "moe_layer_stack_graph_ms", "config": bench.config_dict(args.config, cfg, 1), "layers": args.layers,
            "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds, "card": common.card(dev),
            "graph": entries}
    print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
