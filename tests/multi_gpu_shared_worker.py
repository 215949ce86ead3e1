"""Launched by torchrun (one rank per GPU): expert-parallel forwards with a shared expert per rank.  Each rank holds its
own shared weights; in every round all ranks first run without one (out_plain), then rank 0 alone passes its shared
expert, then every rank does.  A rank that passed one must have out = rne(out_plain + shared_y) bit for bit, and a rank
that did not must have out_plain.  Prints 'RANK r SHARED ALL OK'."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from flashmoe_b200.config import MoEConfig  # noqa: E402
from flashmoe_b200.runtime import MoEContext, SharedExpert, env_rank_world  # noqa: E402

CASES = [
    dict(num_experts=8, expert_top_k=2, sequence_len=512, hidden_size=256, intermediate_size=512),
    dict(num_experts=8, expert_top_k=3, sequence_len=256, hidden_size=128, intermediate_size=256, hidden_act=1),
]


def main():
    rank, world, local = env_rank_world()
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group(backend="cpu:gloo,cuda:nccl", rank=rank, world_size=world, device_id=dev)
    for ci, kw in enumerate(CASES):
        cfg = MoEConfig(**kw)
        nlx = cfg.num_local_experts(world)
        ps = 320
        g = torch.Generator().manual_seed(4000 + 31 * ci + rank)
        we = (torch.randn(nlx, 2, cfg.P, cfg.H, generator=g) * cfg.H ** -0.5).bfloat16().to(dev)
        wg = (torch.randn(cfg.H, cfg.E, generator=torch.Generator().manual_seed(90 + ci)) * cfg.H ** -0.5).bfloat16().to(dev)
        se = SharedExpert((torch.randn(2, ps, cfg.H, generator=g) * cfg.H ** -0.5).bfloat16().to(dev),
                          (torch.randn(ps, generator=g) * 0.1).bfloat16().to(dev),
                          (torch.randn(cfg.H, generator=g) * 0.1).bfloat16().to(dev))
        ctx = MoEContext(cfg, rank=rank, world=world, device=local, timeout_ms=20000, shared_inter=ps)
        for it in range(3):
            n = [cfg.S, 1 + 97 * (it + 1) % cfg.S, cfg.S - 5][it] if rank == 0 else [cfg.S, 200, 0][it]
            x = torch.randn(n, cfg.H, generator=g).bfloat16().to(dev)
            plain = ctx.forward_tokens(x, wg, we).clone()
            ctx.synchronize()
            for who in ("rank0", "all"):
                mine = who == "all" or rank == 0
                out = ctx.forward_tokens(x, wg, we, shared_expert=se if mine else None)
                ctx.synchronize()
                if mine:
                    sy = torch.from_numpy(ctx.read("shared_y")[:n].copy()).view(torch.bfloat16).to(dev)
                    want = (plain.float() + sy.float()).bfloat16()
                else:
                    want = plain
                assert torch.equal(out.view(torch.int16), want.view(torch.int16)), f"rank {rank} case {ci} {it} {who}"
                print(f"RANK {rank} case {ci} round {it} {who} n={n} OK", flush=True)
        dist.barrier()
        ctx.close()
        dist.barrier()
    dist.destroy_process_group()
    print(f"RANK {rank} SHARED ALL OK", flush=True)


if __name__ == "__main__":
    main()
