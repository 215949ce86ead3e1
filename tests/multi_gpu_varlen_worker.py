"""Launched by torchrun (one rank per GPU): expert-parallel forwards in which every rank passes its own token count
(MoEContext.forward_tokens), different between ranks and between launches, including a launch where one rank has no
tokens and one where every rank has S.  Each rank checks every launch's output against the oracle on its own rows with
its own capacity EC(n_r) and all experts' weights.  Prints 'RANK r VARLEN ALL OK'."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from flashmoe_b200.config import MoEConfig  # noqa: E402
from flashmoe_b200.runtime import MoEContext, env_rank_world  # noqa: E402
from oracle import moe_oracle as mo  # noqa: E402
from tests.util import check_output, check_topk  # noqa: E402

CASES = [
    dict(num_experts=8, expert_top_k=2, sequence_len=512, hidden_size=256, intermediate_size=512),
    dict(num_experts=16, expert_top_k=4, sequence_len=256, hidden_size=128, intermediate_size=256, hidden_act=1),
]


def schedule(S, world, launches=8):
    """Token counts [launch][rank], the same on every rank: seeded draws, then one launch with rank 1 empty and one
    with every rank at S."""
    rng = np.random.default_rng(4242)
    counts = [[int(rng.integers(1, S + 1)) for _ in range(world)] for _ in range(launches)]
    counts[2][1] = 0
    counts[5] = [S] * world
    counts[6] = [int(rng.integers(1, 32)) for _ in range(world)]   # decode-sized
    return counts


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
        g = torch.Generator().manual_seed(2000 + 31 * ci + rank)
        gw = torch.Generator().manual_seed(999 + ci)
        wg = (torch.randn(cfg.H, cfg.E, generator=gw) * cfg.H ** -0.5).bfloat16()
        we = (torch.randn(nlx, 2, cfg.P, cfg.H, generator=g) * cfg.H ** -0.5).bfloat16()
        ctx = MoEContext(cfg, rank=rank, world=world, device=local, timeout_ms=20000)
        wgd, wed = wg.to(dev), we.to(dev)
        wes = [torch.empty_like(wed) for _ in range(world)]
        dist.all_gather(wes, wed)
        up, down = mo.split_expert_weights(mo.to_bits(torch.cat([w.cpu() for w in wes], dim=0)))
        del wes
        wg_eff = mo.gate_weights_effective(mo.to_bits(wg), cfg.E, cfg.H)
        slab = ctx.output_buffer().view(cfg.S, cfg.H)
        for it, counts in enumerate(schedule(cfg.S, world)):
            n = counts[rank]
            xn = torch.randn(n, cfg.H, generator=g).bfloat16()
            # alternate between a caller tensor and the zero-copy slab output
            out = ctx.forward_tokens(xn.to(dev), wgd, wed, out=slab[:n] if it % 2 else None)
            ctx.synchronize()
            if n > 0:
                ref = mo.forward(mo.to_bits(xn), wg_eff, up, down, k=cfg.k, EC=cfg.EC_of(n), act=cfg.hidden_act)
                mism = check_topk(ctx.read("topk_idx")[:n], ref)
                check_output(mo.to_bits(out.cpu().reshape(n, cfg.H)), ref.out, rows_ok=~mism,
                             what=f"rank {rank} case {ci} launch {it} n={n}")
                if not mism.any():
                    assert (ctx.read("slot")[:n] == ref.slot).all() and (ctx.read("counts") == ref.counts).all()
            print(f"RANK {rank} case {ci} launch {it} n={n} OK", flush=True)
        dist.barrier()
        ctx.close()
        dist.barrier()
    dist.destroy_process_group()
    print(f"RANK {rank} VARLEN ALL OK", flush=True)


if __name__ == "__main__":
    main()
