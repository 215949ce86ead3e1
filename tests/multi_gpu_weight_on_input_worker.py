"""Launched by torchrun (one rank per GPU): expert-parallel forwards with the router weight on the input on the even
ranks only (fm_set_weight_on_input; each rank's own setting governs the rows it sends), on the caller's routing and on
the gated Llama 4 rule.  Each rank's out must be bit-identical to a one-GPU context holding all E experts with that
rank's setting, run on that rank's tokens.  Prints 'RANK r WEIGHT ON INPUT ALL OK'."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from flashmoe_b200.config import MoEConfig  # noqa: E402
from flashmoe_b200.router import RouterSpec  # noqa: E402
from flashmoe_b200.runtime import MoEContext, env_rank_world  # noqa: E402
from tests import exact as ex  # noqa: E402

LLAMA4 = RouterSpec("sigmoid", renormalize=False)
CASES = [
    dict(num_experts=8, expert_top_k=1, sequence_len=512, hidden_size=256, intermediate_size=384, hidden_act=2),
    dict(num_experts=16, expert_top_k=1, sequence_len=256, hidden_size=128, intermediate_size=256, hidden_act=0),
]


def main():
    rank, world, local = env_rank_world()
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group(backend="cpu:gloo,cuda:nccl", rank=rank, world_size=world, device_id=dev)
    on = rank % 2 == 0
    for ci, kw in enumerate(CASES):
        cfg = MoEConfig(**kw)
        nlx = cfg.num_local_experts(world)
        m = cfg.expert_mats
        g = torch.Generator().manual_seed(5000 + 31 * ci + rank)
        we_all = (torch.randn(cfg.E, m, cfg.P, cfg.H, generator=torch.Generator().manual_seed(97 + ci))
                  * cfg.H ** -0.5).bfloat16().to(dev)
        wg = (torch.randn(cfg.H, cfg.E, generator=torch.Generator().manual_seed(98 + ci)) * cfg.H ** -0.5).bfloat16().to(dev)
        ctx = MoEContext(cfg, rank=rank, world=world, device=local, timeout_ms=20000, weight_on_input=on)
        one = MoEContext(cfg, device=local, timeout_ms=20000, weight_on_input=on)   # world 1, all experts
        wed = we_all[rank * nlx:(rank + 1) * nlx].contiguous()
        rng = np.random.default_rng(700 + ci)
        for it in range(4):
            counts = [int(rng.integers(1, cfg.S + 1)) for _ in range(world)]
            if it == 3:
                counts = [cfg.S] * world
            n = counts[rank]
            x = torch.randn(n, cfg.H, generator=g).bfloat16().to(dev)
            if it % 2:
                out = ctx.forward_gated(x, wg, wed, LLAMA4)
                ctx.synchronize()
                got = out.clone()
                want = one.forward_gated(x, wg, we_all, LLAMA4)
            else:
                topk, _ = ex.routing_case(n, cfg.E, 1, seed=1000 * ci + 10 * it + rank, hot=rank % cfg.E)
                w = rng.random((n, 1)).astype(np.float32) * 1.5
                idx_d, w_d = torch.from_numpy(topk).to(dev), torch.from_numpy(w).to(dev)
                out = ctx.forward_routed(x, idx_d, w_d, wed)
                ctx.synchronize()
                got = out.clone()
                want = one.forward_routed(x, idx_d, w_d, we_all)
            one.synchronize()
            assert torch.equal(got.view(torch.int16), want.view(torch.int16)), f"rank {rank} case {ci} launch {it}"
            print(f"RANK {rank} case {ci} launch {it} n={n} on={on} OK", flush=True)
        dist.barrier()
        one.close()
        ctx.close()
        dist.barrier()
    dist.destroy_process_group()
    print(f"RANK {rank} WEIGHT ON INPUT ALL OK", flush=True)


if __name__ == "__main__":
    main()
