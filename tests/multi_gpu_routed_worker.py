"""Launched by torchrun (one rank per GPU): expert-parallel forwards on the caller's routing (MoEContext.forward_routed),
each rank with its own routing -- global expert ids, -1 and duplicate picks, skew that overflows a capacity -- and its
own token count.  Each rank's out must be bit-identical to a one-GPU context holding all E experts run on that rank's
tokens and routing: the per-(source, expert) capacity EC(n_r) and the slot order are the same in both.  One launch per
case is a router call on every rank, to mix the two kinds of call.  Prints 'RANK r ROUTED ALL OK'."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from flashmoe_b200.config import MoEConfig  # noqa: E402
from flashmoe_b200.runtime import MoEContext, env_rank_world  # noqa: E402
from tests import exact as ex  # noqa: E402

CASES = [
    dict(num_experts=8, expert_top_k=2, sequence_len=512, hidden_size=256, intermediate_size=512),
    dict(num_experts=16, expert_top_k=1, sequence_len=256, hidden_size=128, intermediate_size=256, hidden_act=1),
    dict(num_experts=8, expert_top_k=3, sequence_len=256, hidden_size=128, intermediate_size=256),
]


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
        we_all = (torch.randn(cfg.E, 2, cfg.P, cfg.H, generator=torch.Generator().manual_seed(77 + ci))
                  * cfg.H ** -0.5).bfloat16().to(dev)
        wg = (torch.randn(cfg.H, cfg.E, generator=torch.Generator().manual_seed(78 + ci)) * cfg.H ** -0.5).bfloat16().to(dev)
        ctx = MoEContext(cfg, rank=rank, world=world, device=local, timeout_ms=20000)
        one = MoEContext(cfg, device=local, timeout_ms=20000)   # world 1, all experts
        wed = we_all[rank * nlx:(rank + 1) * nlx].contiguous()
        rng = np.random.default_rng(500 + ci)
        for it in range(6):
            counts = [int(rng.integers(1, cfg.S + 1)) for _ in range(world)]
            if it == 2:
                counts[1] = 0
            if it == 4:
                counts = [cfg.S] * world
            n = counts[rank]
            x = torch.randn(n, cfg.H, generator=g).bfloat16().to(dev)
            if it == 3:   # every rank runs the router this time
                ctx.forward_tokens(x, wg, wed)
                ctx.synchronize()
                print(f"RANK {rank} case {ci} launch {it} router n={n} OK", flush=True)
                continue
            topk, w = ex.routing_case(n, cfg.E, cfg.k, seed=1000 * ci + 10 * it + rank, hot=rank % cfg.E)
            idx_d, w_d = torch.from_numpy(topk).to(dev), torch.from_numpy(w).to(dev)
            out = ctx.forward_routed(x, idx_d, w_d, wed)
            ctx.synchronize()
            got = out.clone()
            want = one.forward_routed(x, idx_d, w_d, we_all)
            one.synchronize()
            assert torch.equal(got.view(torch.int16), want.view(torch.int16)), f"rank {rank} case {ci} launch {it}"
            print(f"RANK {rank} case {ci} launch {it} n={n} OK", flush=True)
        dist.barrier()
        one.close()
        ctx.close()
        dist.barrier()
    dist.destroy_process_group()
    print(f"RANK {rank} ROUTED ALL OK", flush=True)


if __name__ == "__main__":
    main()
