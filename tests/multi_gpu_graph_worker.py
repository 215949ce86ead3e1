"""Launched by torchrun (one rank per GPU): every rank captures one device-count CUDA graph (MoEContext.forward_tokens
with n_tokens=<int32 tensor>) and replays it with its own token count, different between ranks and between replays,
including a replay where one rank has no tokens and one where every rank has S; rows past n of x hold NaN.  A second
context on every rank runs the same forwards eagerly with host-side counts; each replay's output and routing tables
must equal them bit for bit.  Prints 'RANK r GRAPH ALL OK'."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from flashmoe_b200.config import MoEConfig  # noqa: E402
from flashmoe_b200.runtime import MoEContext, env_rank_world  # noqa: E402
from tests.multi_gpu_varlen_worker import schedule  # noqa: E402

CASES = [
    dict(num_experts=8, expert_top_k=2, sequence_len=512, hidden_size=256, intermediate_size=512),
    dict(num_experts=16, expert_top_k=4, sequence_len=256, hidden_size=128, intermediate_size=256, hidden_act=1),
]
TABLES = ("topk_idx", "topk_w", "slot", "mcw", "counts", "recv_cnt")


def state(ctx, out, n, H):
    ctx.synchronize()
    st = {"out": out.reshape(-1, H)[:n].view(torch.int16).cpu().numpy()}
    for name in TABLES:
        t = ctx.read(name)
        st[name] = t if name in ("counts", "recv_cnt") else t[:n]
    return st


def main():
    rank, world, local = env_rank_world()
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group(backend="cpu:gloo,cuda:nccl", rank=rank, world_size=world, device_id=dev)
    for ci, kw in enumerate(CASES):
        cfg = MoEConfig(**kw)
        if cfg.E % world:
            continue
        nlx = cfg.num_local_experts(world)
        g = torch.Generator().manual_seed(3000 + 31 * ci + rank)
        gw = torch.Generator().manual_seed(1999 + ci)
        wgd = (torch.randn(cfg.H, cfg.E, generator=gw) * cfg.H ** -0.5).bfloat16().to(dev)
        wed = (torch.randn(nlx, 2, cfg.P, cfg.H, generator=g) * cfg.H ** -0.5).bfloat16().to(dev)
        ctx = MoEContext(cfg, rank=rank, world=world, device=local, timeout_ms=20000)
        ref = MoEContext(cfg, rank=rank, world=world, device=local, timeout_ms=20000)
        x_full = torch.empty(cfg.S, cfg.H, dtype=torch.bfloat16, device=dev)
        out_full = torch.empty_like(x_full)
        n_dev = torch.zeros(1, dtype=torch.int32, device=dev)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            ctx.forward_tokens(x_full, wgd, wed, out=out_full, n_tokens=n_dev)
        for it, counts in enumerate(schedule(cfg.S, world)):
            n = counts[rank]
            xn = torch.randn(n, cfg.H, generator=g).bfloat16().to(dev)
            x_full[:n].copy_(xn)
            x_full[n:].view(torch.int16).fill_(-64)   # bf16 NaN
            n_dev.fill_(n)
            graph.replay()
            got = state(ctx, out_full, n, cfg.H)
            want = state(ref, ref.forward_tokens(xn, wgd, wed), n, cfg.H)
            for name in want:
                assert np.array_equal(got[name], want[name]), f"rank {rank} case {ci} replay {it} n={n}: {name}"
            print(f"RANK {rank} case {ci} replay {it} n={n} OK", flush=True)
        dist.barrier()
        ctx.close()
        ref.close()
        dist.barrier()
    dist.destroy_process_group()
    print(f"RANK {rank} GRAPH ALL OK", flush=True)


if __name__ == "__main__":
    main()
