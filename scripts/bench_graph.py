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
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import torch  # noqa: E402

import bench  # noqa: E402   (configs and their description; bench.py itself is not changed by this script)
from bench_varlen import card, parse_tokens  # noqa: E402


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
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize(dev)
        t0 = time.perf_counter()
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize(dev)
        wall = (time.perf_counter() - t0) * 1e3 / steps
        return wall, e0.elapsed_time(e1) / steps

    entries = []
    for n in tokens:
        graph_n = capture(n, False)
        arms = {"eager": lambda: stack(n, False), "graph_per_n": graph_n.replay, "graph_dev_n": graph_dev.replay}
        n_dev.fill_(n)
        for fn in arms.values():
            for _ in range(warmup):
                fn()
        ctx.synchronize()
        runs = {k: {"wall": [], "device": []} for k in arms}
        for _ in range(rounds):
            for k, fn in arms.items():
                wall, device = window(fn)
                runs[k]["wall"].append(wall)
                runs[k]["device"].append(device)
        ctx.synchronize()   # raises if a launch reported a problem
        e = {"tokens": n}
        for k, r in runs.items():
            for what in ("wall", "device"):
                v = r[what]
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
    ap.add_argument("--tokens", default="1,8,128,4096", metavar="N1,N2,..")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    tokens = parse_tokens(ap, args.tokens, bench.BASELINE_CONFIGS[args.config].S)
    if args.layers < 1:
        ap.error("--layers must be >= 1")
    if args.steps < 1 or args.rounds < 1 or args.warmup < 0:
        ap.error("--steps and --rounds must be >= 1, --warmup >= 0")
    if not torch.cuda.is_available():
        print("bench_graph.py: no CUDA device; the MoE forward path has no CPU fallback", file=sys.stderr)
        return 3
    dev = torch.device("cuda", torch.cuda.current_device())
    entries = run_graph(args.config, args.layers, tokens, args.steps, args.warmup, args.rounds, dev)
    cfg = bench.BASELINE_CONFIGS[args.config]
    line = {"metric": "moe_layer_stack_graph_ms", "config": bench.config_dict(args.config, cfg, 1), "layers": args.layers,
            "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds, "card": card(dev), "graph": entries}
    print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
