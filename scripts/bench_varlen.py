#!/usr/bin/env python
"""Forwards on fewer tokens than the context's size (MoEContext.forward_tokens): device time per token count n.

    python scripts/bench_varlen.py --tokens 1,8,32,128,512,1024,4096 [--config B] [--steps K] [--warmup W] [--rounds R]
    python -m torch.distributed.run --nproc-per-node N ... scripts/bench_varlen.py --tokens ...

For every n (0 <= n <= S of --config) three arms run alternating, `rounds` times `steps` forwards each (medians reported):
  ms                 forward_tokens(n) on the --config context (S tokens at most);
  ms_context_of_n    forward on a context created for S = n (n a multiple of 128 only);
  ms_padded_to_S     the workaround without forward_tokens: n real rows plus zero rows up to S through forward.
Also tokens/s, executed token-expert pairs and an HBM floor: the weights of the experts that received at least one row,
the router weights, x read and out written, over the H100 SXM data-sheet 3.35 TB/s.  Inputs are bench.py's seeded
synthetic tensors.  Prints one JSON line (rank 0) with the card's name and power limit next to the figures; writes no
files.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402   (seeded inputs, rank helpers; bench.py itself is not changed by this script)
from scripts import bench_common as common  # noqa: E402

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet HBM3 bandwidth: the floor is stated against it, not a measured rate


def run_varlen(env, name, tokens, steps, warmup, rounds):
    from flashmoe_b200.runtime import MoEContext

    rank, world, dev = env.rank, env.world, env.dev
    cfg = bench.BASELINE_CONFIGS[name]
    nlx = cfg.num_local_experts(world)
    S, H, P = cfg.S, cfg.H, cfg.P
    ctx = MoEContext(cfg, rank=rank, world=world, device=dev.index, timeout_ms=30000)
    x, wg, we = bench.make_inputs(cfg, nlx, rank)
    xd, wgd, wed = x.to(dev).view(S, H), wg.to(dev), we.to(dev)
    del we

    entries = []
    for n in tokens:
        xn = xd[:n]
        out_n = torch.empty_like(xn)
        arms = {"ms": lambda: ctx.forward_tokens(xn, wgd, wed, out=out_n)}
        x_pad = torch.zeros(1, S, H, dtype=torch.bfloat16, device=dev)
        x_pad.view(S, H)[:n] = xn
        out_pad = torch.empty_like(x_pad)
        arms["ms_padded_to_S"] = lambda: ctx.forward(x_pad, wgd, wed, out=out_pad)
        ctx_n = None
        if n > 0 and n % 128 == 0:
            ctx_n = MoEContext(cfg.replace(sequence_len=n, mini_batch=1), rank=rank, world=world, device=dev.index,
                               timeout_ms=30000)
            xn3, out_n3 = xn.view(1, n, H), torch.empty(1, n, H, dtype=torch.bfloat16, device=dev)
            arms["ms_context_of_n"] = lambda: ctx_n.forward(xn3, wgd, wed, out=out_n3)
        times = common.alternate(arms, warmup, rounds, env.barrier,
                                 lambda fn: env.max_over_ranks(common.device_ms(fn, steps, env.barrier)))
        # work of the forward_tokens call: executed token-expert pairs and the experts that received rows
        ctx.forward_tokens(xn, wgd, wed, out=out_n)
        ctx.synchronize()
        recv = ctx.read("recv_cnt").reshape(world, nlx)
        pairs = env.sum_over_ranks(int(recv.sum()))
        used_local = int((recv.sum(axis=0) > 0).sum())
        floor_bytes = used_local * 2 * P * H * 2 + cfg.E * H * 2 + 2 * n * H * 2
        floor_ms = env.max_over_ranks(floor_bytes / HBM_BYTES_PER_S * 1e3)
        e = {"tokens": n, "ec": cfg.EC_of(n), **common.medians(times)}
        ms = e["ms"]
        e.update({"tokens_per_s": world * n / (ms * 1e-3), "token_expert_pairs_executed": pairs,
                  "experts_with_rows_per_rank": used_local, "hbm_floor_bytes_per_rank": floor_bytes,
                  "hbm_floor_ms": floor_ms, "frac_of_hbm_floor": floor_ms / ms})
        if "ms_context_of_n" in e:
            e["gap_vs_context_of_n"] = ms / e["ms_context_of_n"] - 1.0
        entries.append(e)
        if ctx_n is not None:
            env.barrier()
            ctx_n.close()
        del x_pad, out_pad
        env.barrier()
    ctx.close()
    torch.cuda.empty_cache()
    env.barrier()
    return entries


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--config", default="B", choices=sorted(bench.BASELINE_CONFIGS))
    common.add_run_args(ap, tokens=None, steps=200, warmup=32, rounds=3)
    args = ap.parse_args()
    tokens = common.parse_tokens(ap, args.tokens, bench.BASELINE_CONFIGS[args.config].S)
    common.check_counts(ap, args)
    if not torch.cuda.is_available():
        return common.no_cuda("bench_varlen.py")
    rank, world, local = bench.env_int("RANK", 0), bench.env_int("WORLD_SIZE", 1), bench.env_int("LOCAL_RANK", 0)
    torch.cuda.set_device(local % torch.cuda.device_count())
    dev = torch.device("cuda", torch.cuda.current_device())
    import torch.distributed as dist

    if world > 1:
        dist.init_process_group(backend="cpu:gloo,cuda:nccl", rank=rank, world_size=world, device_id=dev)
    env = bench.Env(rank, world, dev)
    entries = run_varlen(env, args.config, tokens, args.steps, args.warmup, args.rounds)
    line = {"metric": "moe_layer_fwd_varlen_ms", "config": bench.config_dict(args.config, bench.BASELINE_CONFIGS[args.config],
                                                                             world),
            "n_gpus": world, "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds,
            "card": common.card(dev), "hbm_floor_rate_bytes_per_s": HBM_BYTES_PER_S, "varlen": entries}
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
    if rank == 0:
        print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
