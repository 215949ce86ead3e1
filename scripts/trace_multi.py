"""Per-rank phase timeline of one fused forward at world > 1 (launch with torchrun): where the time of an expert-parallel
step goes -- dispatch complete, first tile of a REMOTE packet ready, last tile published, all done flags seen, kernel end.
Usage: torchrun --nproc-per-node N scripts/trace_multi.py [--cfg B] [--slab-out 0|1]"""
import argparse
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np
import torch
import torch.distributed as dist

from flashmoe_b200 import trace_slots as ts
from flashmoe_b200.config import BASELINE_CONFIGS
from flashmoe_b200.runtime import MoEContext, env_rank_world


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cfg", default="B")
    ap.add_argument("--slab-out", type=int, default=1)
    ap.add_argument("--steps", type=int, default=50)
    args = ap.parse_args()
    rank, world, local = env_rank_world()
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group(backend="cpu:gloo,cuda:nccl", rank=rank, world_size=world, device_id=dev)
    cfg = BASELINE_CONFIGS[args.cfg]
    nlx = cfg.num_local_experts(world)
    g = torch.Generator().manual_seed(0x5EED + rank)
    gw = torch.Generator().manual_seed(0x5EED)
    x = torch.randn(1, cfg.S, cfg.H, generator=g).bfloat16().to(dev)
    wg = torch.randn(cfg.H, cfg.E, generator=gw).bfloat16().to(dev)
    we = torch.randn(nlx, 2, cfg.P, cfg.H, generator=g).bfloat16().to(dev)
    ctx = MoEContext(cfg, rank=rank, world=world, device=local, timeout_ms=20000)
    out = ctx.output_buffer() if (args.slab_out and world > 1) else torch.empty_like(x)
    for _ in range(10):
        ctx.forward(x, wg, we, out=out)
    torch.cuda.synchronize()
    dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        ctx.forward(x, wg, we, out=out)
    e1.record()
    torch.cuda.synchronize()
    ms = torch.tensor([e0.elapsed_time(e1) / args.steps], device=dev)
    dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    dist.barrier()
    ctx.set_trace(True)
    for _ in range(3):   # the last launch's stamps are read; a few traced launches so the ranks are in lock-step again
        ctx.forward(x, wg, we, out=out)
    ctx.synchronize()
    tr = ctx.read("trace").astype(np.int64)
    t00 = tr[:, ts.START].min()
    us = lambda a: (a - t00) / 1e3  # noqa: E731
    rec = {}
    for key, col, red in (("start_spread", ts.START, "max"), ("gate_done", ts.GATE_DONE, "med"), ("barrier", ts.BARRIER, "med"),
                          ("disp_prefix", ts.DISP_PREFIX, "med"), ("disp_rows_done", ts.DISP_ROWS_DONE, "med"),
                          ("dispatch_end_max", ts.DISPATCH_END, "max"), ("ffn_end_med", ts.FFN_END, "med"),
                          ("done_flags_seen", ts.DONE_FLAGS, "med"), ("kernel_end", ts.KERNEL_END, "max")):
        v = tr[:, col][tr[:, col] > 0]
        rec[key] = float(us(np.median(v) if red == "med" else v.max())) if len(v) else float("nan")
    first_landed = tr[:, ts.TILE_FIRST_KB][tr[:, ts.TILE_FIRST_KB] > 0]
    rec["first_tile_kb0_landed_min"] = float(us(first_landed.min())) if len(first_landed) else float("nan")
    rec["first_tile_kb0_landed_med"] = float(us(np.median(first_landed))) if len(first_landed) else float("nan")
    rem = tr[:, ts.FIRST_REMOTE][tr[:, ts.FIRST_REMOTE] > 0]
    rec["first_remote_tile_ready_min"] = float(us(rem.min())) if len(rem) else float("nan")
    pub = tr[:, ts.TILE_PUBLISHED:ts.TILE_PUBLISHED + ts.TILES]
    rec["last_tile_published"] = float(us(pub.max())) if (pub > 0).any() else float("nan")
    mma = tr[:, ts.TILE_MMA_DONE:ts.TILE_MMA_DONE + ts.TILES]   # MMA complete, per tile
    rec["last_mma_complete"] = float(us(mma.max())) if (mma > 0).any() else float("nan")
    rec["abs_start_ns"] = int(t00)
    allr = [None] * world
    dist.all_gather_object(allr, rec)
    if rank == 0:
        print(f"=== config {args.cfg} world {world}: {float(ms.item()) * 1e3:.1f} us / step (max over ranks, {args.steps} steps, "
              f"output in {'slab' if args.slab_out and world > 1 else 'caller tensor'})")
        keys = [k for k in rec if k != "abs_start_ns"]
        print("rank " + " ".join(f"{k[:18]:>18s}" for k in keys) + "   start skew vs rank0 (us)")
        for r, d in enumerate(allr):
            print(f"{r:4d} " + " ".join(f"{d[k]:18.1f}" for k in keys) + f"   {(d['abs_start_ns'] - allr[0]['abs_start_ns']) / 1e3:10.1f}")
    np.save(f"gpurun_out/trace_{args.cfg}_w{world}_r{rank}.npy", tr)
    dist.barrier()
    ctx.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
