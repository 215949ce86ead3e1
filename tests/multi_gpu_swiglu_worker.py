"""Launched by torchrun (one rank per GPU): expert-parallel SwiGLU forwards (hidden_act = 2).  Every rank holds its
slice [nLx, 3, P, H] of one set of E experts (the W_down block at matrix 2 of the gated layout, reached through the
dispatched packets of every source rank) and its own tokens and count; on the built-in router, the caller's routing
(-1 picks) and the DeepSeek-V3 rule, with biases and a [3, Ps, H] shared expert.  Each rank's out must equal, bit for
bit, a one-rank context holding all E experts on the same tokens: routing, h, y and the combine are per token and do
not depend on where an expert runs.  Prints 'RANK r SWIGLU ALL OK'."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from flashmoe_b200.config import MoEConfig  # noqa: E402
from flashmoe_b200.router import RouterSpec  # noqa: E402
from flashmoe_b200.runtime import MoEContext, SharedExpert, env_rank_world  # noqa: E402

V3 = RouterSpec("sigmoid", 8, 4, 2, True, 2.5)
CASES = [   # (route, config)
    ("router", dict(num_experts=16, expert_top_k=2, sequence_len=512, hidden_size=320, intermediate_size=320)),
    ("router", dict(num_experts=16, expert_top_k=3, sequence_len=256, hidden_size=256, intermediate_size=192)),
    ("routed", dict(num_experts=16, expert_top_k=2, sequence_len=512, hidden_size=256, intermediate_size=384)),
    ("gated", dict(num_experts=16, expert_top_k=4, sequence_len=256, hidden_size=320, intermediate_size=192)),
]
PS = 192


def main():
    rank, world, local = env_rank_world()
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group(backend="cpu:gloo,cuda:nccl", rank=rank, world_size=world, device_id=dev)
    for ci, (route, kw) in enumerate(CASES):
        cfg = MoEConfig(hidden_act=2, **kw)
        E, k, H, P, S = cfg.E, cfg.k, cfg.H, cfg.P, cfg.S
        nlx = cfg.num_local_experts(world)
        gw = torch.Generator().manual_seed(500 + ci)   # the same weights on every rank
        s = H ** -0.5
        we = (torch.randn(E, 3, P, H, generator=gw) * s).bfloat16().to(dev)
        bu = (torch.randn(E, 2, P, generator=gw) * 0.1).bfloat16().to(dev)
        bd = (torch.randn(E, H, generator=gw) * 0.1).bfloat16().to(dev)
        wg = (torch.randn(H, E, generator=gw) * s).bfloat16().to(dev)
        se = SharedExpert((torch.randn(3, PS, H, generator=gw) * s).bfloat16().to(dev),
                          (torch.randn(2, PS, generator=gw) * 0.1).bfloat16().to(dev),
                          (torch.randn(H, generator=gw) * 0.1).bfloat16().to(dev))
        mine = slice(rank * nlx, (rank + 1) * nlx)
        ctx = MoEContext(cfg, rank=rank, world=world, device=local, timeout_ms=20000, shared_inter=PS)
        one = MoEContext(cfg, rank=0, world=1, device=local, timeout_ms=20000, shared_inter=PS)
        g = torch.Generator().manual_seed(600 + 31 * ci + rank)   # this rank's tokens
        for it, n in enumerate((S, [S - 5, 200][rank % 2], [1, 0][rank % 2])):
            x = torch.randn(n, H, generator=g).bfloat16().to(dev)
            idx = torch.randint(-1, E, (n, k), generator=g, dtype=torch.int32).to(dev)
            w = torch.rand(n, k, generator=g).to(dev)
            for shared in (None, se):
                def call(c, weights, b_up, b_down):
                    kwargs = dict(bias_up=b_up, bias_down=b_down, shared_expert=shared)
                    if route == "routed":
                        return c.forward_routed(x, idx, w, weights, **kwargs)
                    if route == "gated":
                        return c.forward_gated(x, wg, weights, V3, **kwargs)
                    return c.forward_tokens(x, wg, weights, **kwargs)

                got = call(ctx, we[mine].contiguous(), bu[mine].contiguous(), bd[mine].contiguous()).clone()
                ctx.synchronize()
                want = call(one, we, bu, bd)
                one.synchronize()
                assert torch.equal(got.view(torch.int16), want.view(torch.int16)), (
                    f"rank {rank} case {ci} ({route}) round {it} n={n} shared={shared is not None}: out differs from "
                    f"the one-rank context in {int((got.view(torch.int16) != want.view(torch.int16)).sum())} elements")
                print(f"RANK {rank} case {ci} {route} round {it} n={n} shared={shared is not None} OK", flush=True)
        dist.barrier()
        one.close()
        ctx.close()
        dist.barrier()
    dist.destroy_process_group()
    print(f"RANK {rank} SWIGLU ALL OK", flush=True)


if __name__ == "__main__":
    main()
