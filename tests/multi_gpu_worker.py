"""Expert-parallel forwards, one process per GPU: `python -m torch.distributed.run --nproc-per-node=N
tests/multi_gpu_worker.py <scenario>`, a name from SCENARIOS.  Every rank checks its own output; each prints
'RANK r <scenario> ALL OK' at the end.

A world of one rank runs every scenario against a one-rank context.  That checks little of expert parallelism, but it
runs every scenario's code on a one-GPU machine."""
import os
import sys
from dataclasses import dataclass, field

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from flashmoe_b200.config import MoEConfig  # noqa: E402
from flashmoe_b200.router import RouterSpec  # noqa: E402
from flashmoe_b200.runtime import MoEContext, SharedExpert, env_rank_world  # noqa: E402
from oracle import moe_oracle as mo  # noqa: E402
from tests import exact as ex  # noqa: E402
from tests.util import check_output, check_topk  # noqa: E402

V3 = RouterSpec("sigmoid", 8, 4, 2, True, 2.5)
LLAMA4 = RouterSpec("sigmoid", renormalize=False)
GRAPH_TABLES = ("topk_idx", "topk_w", "slot", "mcw", "counts", "recv_cnt")


def config(entry):
    """A case entry's config: its keys that start with `_` are the scenario's, not MoEConfig's."""
    return MoEConfig(**{k: v for k, v in entry.items() if not k.startswith("_")})


def _bits(a):
    """A bf16 tensor as int16 bits on the host; a routing table read from a context as it is."""
    return a.view(torch.int16).cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)


@dataclass
class Case:
    """One case on this rank.  Its seeds derive from `ci`, its position in the scenario's list."""
    ci: int
    cfg: MoEConfig
    entry: dict
    rank: int
    world: int
    dev: torch.device = None
    contexts: list = field(default_factory=list)   # closed by main after the case

    @property
    def nlx(self):
        return self.cfg.num_local_experts(self.world)

    def context(self, one_rank=False, **kw):
        """This rank's context in the world or, with `one_rank`, a one-rank context holding all E experts."""
        rank, world = (0, 1) if one_rank else (self.rank, self.world)
        ctx = MoEContext(self.cfg, rank=rank, world=world, device=self.dev.index, timeout_ms=20000, **kw)
        self.contexts.append(ctx)
        return ctx

    def randn(self, g, *shape, scale=None):
        """Normal draws from `g` times `scale` (default H^-0.5, the weights' scale) as bf16 on this rank's GPU."""
        s = self.cfg.H ** -0.5 if scale is None else scale
        return (torch.randn(*shape, generator=g) * s).bfloat16().to(self.dev)

    def experts(self, g):
        """Seeded weights [E, m, P, H] of all E experts (m = 2, or SwiGLU's 3) and this rank's slice of them."""
        cfg = self.cfg
        we = self.randn(g, cfg.E, cfg.expert_mats, cfg.P, cfg.H)
        return we, we[self.rank * self.nlx:(self.rank + 1) * self.nlx].contiguous()

    def same_bits(self, got, want, it, n, what="out"):
        g, w = _bits(got), _bits(want)
        diff = int((g != w).sum()) if g.shape == w.shape else f"all (shapes {g.shape} and {w.shape})"
        assert g.shape == w.shape and not diff, (
            f"rank {self.rank} case {self.ci} launch {it} n={n}: {what} differs from the reference in {diff} elements")


def oracle_experts(c, wg, we):
    """The oracle's gate and all E experts' weights, gathered from every rank's `we` (other ranks' tokens are
    irrelevant to this rank's)."""
    wes = [torch.empty_like(we) for _ in range(c.world)]
    dist.all_gather(wes, we)
    up, down = mo.split_expert_weights(mo.to_bits(torch.cat([w.cpu() for w in wes], dim=0)))
    return mo.gate_weights_effective(mo.to_bits(wg.cpu()), c.cfg.E, c.cfg.H), up, down


def token_counts(rng, S, world, launches, empty=None, full=None):
    """Token counts [rank] of each launch, drawn from `rng` in [1, S] when the launch comes (a caller may draw from `rng`
    in between); rank 1 has none at launch `empty` (a world of one has no rank 1), every rank has S at launch `full`."""
    for it in range(launches):
        counts = [int(rng.integers(1, S + 1)) for _ in range(world)]
        if it == empty and world > 1:
            counts[1] = 0
        if it == full:
            counts = [S] * world
        yield counts


# ------------------------------------------------------------------ parity, parity_small
PARITY = [
    dict(num_experts=8, expert_top_k=2, sequence_len=512, hidden_size=256, intermediate_size=512),
    dict(num_experts=8, expert_top_k=2, sequence_len=1024, hidden_size=512, intermediate_size=1024, drop_tokens=0),
    dict(num_experts=16, expert_top_k=4, sequence_len=256, hidden_size=128, intermediate_size=256, hidden_act=1),
    # BASELINE config B sharded E/W -- the shape bench.py times at N = 2, 4, 8 (sampled oracle)
    dict(num_experts=8, expert_top_k=2, sequence_len=4096, hidden_size=1024, intermediate_size=4096, _sample=192,
         _launches=20),
    # token-sweep shape D4k: 32 experts, d_model 2048, ffn 2048 (sampled oracle)
    dict(num_experts=32, expert_top_k=2, sequence_len=4096, hidden_size=2048, intermediate_size=2048, _sample=128),
]


def parity_counts(c):
    return [c.cfg.S] * c.entry.get("_launches", 6)


def parity(c):
    """Each rank's [S, H] output against the oracle's world composition (SURVEY.md Appendix A.8).  Back-to-back
    launches on one context take different inputs, so routing, per-packet row counts and drops change from launch to
    launch: a GEMM that read a stale row of the previous launch (recv_x, hidden, recv_meta, the accumulator) would give
    a wrong result.  Full-size cases are checked on a seeded sample of tokens per rank (the oracle's FFN cost is per
    token; routing and capacity drops are still computed over all tokens)."""
    cfg, rank = c.cfg, c.rank
    g = torch.Generator().manual_seed(1000 + 17 * c.ci + rank)
    gw = torch.Generator().manual_seed(777 + c.ci)
    xs = [torch.randn(1, cfg.S, cfg.H, generator=g).bfloat16() for _ in range(3)]
    # the third input routes most tokens to few experts: counts shrink / grow strongly between launches.  (Token 0 plus
    # small noise, not identical copies: with identical rows one borderline element would be replicated S/2 times and
    # decide the ">= 99.9 % of the elements within tolerance" criterion on its own.)
    noise = torch.randn(1, cfg.S // 2, cfg.H, generator=g) * 0.02
    xs[2][:, : cfg.S // 2] = (xs[2][:, :1].float() + noise).bfloat16()
    wg = c.randn(gw, cfg.H, cfg.E)
    we = c.randn(g, c.nlx, 2, cfg.P, cfg.H)
    ctx = c.context()
    wg_eff, up, down = oracle_experts(c, wg, we)
    n_sample = c.entry.get("_sample", 0)
    refs, samples = [], []
    for i, x in enumerate(xs):
        xb = mo.to_bits(x.view(cfg.S, cfg.H))
        if n_sample:
            smp = np.sort(np.random.default_rng(5 + i + rank).choice(cfg.S, size=n_sample, replace=False)).astype(np.int32)
            refs.append(mo.forward_sample(xb, wg_eff, up, down, smp, k=cfg.k, EC=cfg.EC, act=cfg.hidden_act))
        else:
            smp = None
            refs.append(mo.forward(xb, wg_eff, up, down, k=cfg.k, EC=cfg.EC, act=cfg.hidden_act))
        samples.append(smp)
    xds = [x.to(c.dev) for x in xs]
    out_slab = ctx.output_buffer()
    launches = parity_counts(c)
    worst = 0.0
    for it in range(len(launches)):
        i = it % len(xs)
        # alternate between a caller tensor and the zero-copy slab output
        out = ctx.forward(xds[i], wg, we, out=out_slab if it % 2 else None)
        ctx.synchronize()
        ref, smp = refs[i], samples[i]
        mism = check_topk(ctx.read("topk_idx"), ref)
        got = mo.to_bits(out.cpu().view(cfg.S, cfg.H))
        what = f"rank {rank} case {c.ci} launch {it}"
        if smp is not None:
            relf = check_output(got[smp], ref.out, rows_ok=~mism[smp], what=what)
        else:
            relf = check_output(got, ref.out, rows_ok=~mism, what=what)
            if not mism.any():
                assert (ctx.read("slot") == ref.slot).all() and (ctx.read("counts") == ref.counts).all(), what
        worst = max(worst, relf)
    return f"launches={len(launches)} relF_max={worst:.2e} recv_cnt={ctx.read('recv_cnt').tolist()[:16]}"


# ------------------------------------------------------------------ routed
ROUTED = [
    dict(num_experts=8, expert_top_k=2, sequence_len=512, hidden_size=256, intermediate_size=512),
    dict(num_experts=16, expert_top_k=1, sequence_len=256, hidden_size=128, intermediate_size=256, hidden_act=1),
    dict(num_experts=8, expert_top_k=3, sequence_len=256, hidden_size=128, intermediate_size=256),
]


def routed_counts(c):
    counts = token_counts(np.random.default_rng(500 + c.ci), c.cfg.S, c.world, 6, empty=2, full=4)
    return [cs[c.rank] for cs in counts]


def routed(c):
    """The caller's routing (MoEContext.forward_routed), each rank with its own routing -- global expert ids, -1 and
    duplicate picks, skew that overflows a capacity -- and its own token count.  Each rank's out must be bit-identical
    to a one-rank context holding all E experts run on that rank's tokens and routing: the per-(source, expert)
    capacity EC(n_r) and the slot order are the same in both.  Launch 3 is a router call on every rank, to mix the two
    kinds of call."""
    cfg = c.cfg
    g = torch.Generator().manual_seed(3000 + 31 * c.ci + c.rank)
    we_all, we = c.experts(torch.Generator().manual_seed(77 + c.ci))
    wg = c.randn(torch.Generator().manual_seed(78 + c.ci), cfg.H, cfg.E)
    ctx, one = c.context(), c.context(one_rank=True)
    for it, n in enumerate(routed_counts(c)):
        x = c.randn(g, n, cfg.H, scale=1)
        if it == 3:
            ctx.forward_tokens(x, wg, we)
            ctx.synchronize()
            continue
        topk, w = ex.routing_case(n, cfg.E, cfg.k, seed=1000 * c.ci + 10 * it + c.rank, hot=c.rank % cfg.E)
        idx_d, w_d = torch.from_numpy(topk).to(c.dev), torch.from_numpy(w).to(c.dev)
        got = ctx.forward_routed(x, idx_d, w_d, we).clone()
        ctx.synchronize()
        want = one.forward_routed(x, idx_d, w_d, we_all)
        one.synchronize()
        c.same_bits(got, want, it, n)


# ------------------------------------------------------------------ varlen, graph
VARLEN = [
    dict(num_experts=8, expert_top_k=2, sequence_len=512, hidden_size=256, intermediate_size=512),
    dict(num_experts=16, expert_top_k=4, sequence_len=256, hidden_size=128, intermediate_size=256, hidden_act=1),
]


def varlen_counts(c):
    rng = np.random.default_rng(4242)
    counts = list(token_counts(rng, c.cfg.S, c.world, 8, empty=2, full=5))
    counts[6] = [int(rng.integers(1, 32)) for _ in range(c.world)]   # decode-sized
    return [cs[c.rank] for cs in counts]


def varlen(c):
    """Every rank passes its own token count (MoEContext.forward_tokens), different between ranks and between launches,
    including a launch where rank 1 has no tokens and one where every rank has S.  Each rank checks every launch's
    output against the oracle on its own rows with its own capacity EC(n_r) and all experts' weights."""
    cfg = c.cfg
    g = torch.Generator().manual_seed(2000 + 31 * c.ci + c.rank)
    wg = c.randn(torch.Generator().manual_seed(999 + c.ci), cfg.H, cfg.E)
    we = c.randn(g, c.nlx, 2, cfg.P, cfg.H)
    ctx = c.context()
    wg_eff, up, down = oracle_experts(c, wg, we)
    slab = ctx.output_buffer().view(cfg.S, cfg.H)
    for it, n in enumerate(varlen_counts(c)):
        xn = torch.randn(n, cfg.H, generator=g).bfloat16()
        # alternate between a caller tensor and the zero-copy slab output
        out = ctx.forward_tokens(xn.to(c.dev), wg, we, out=slab[:n] if it % 2 else None)
        ctx.synchronize()
        if n > 0:
            ref = mo.forward(mo.to_bits(xn), wg_eff, up, down, k=cfg.k, EC=cfg.EC_of(n), act=cfg.hidden_act)
            mism = check_topk(ctx.read("topk_idx")[:n], ref)
            what = f"rank {c.rank} case {c.ci} launch {it} n={n}"
            check_output(mo.to_bits(out.cpu().reshape(n, cfg.H)), ref.out, rows_ok=~mism, what=what)
            if not mism.any():
                assert (ctx.read("slot")[:n] == ref.slot).all() and (ctx.read("counts") == ref.counts).all(), what


def launch_state(ctx, out, n):
    """The first n rows of `out` and the routing tables of ctx's last launch."""
    ctx.synchronize()
    st = {"out": out.reshape(-1, ctx.cfg.H)[:n]}
    for name in GRAPH_TABLES:
        t = ctx.read(name)
        st[name] = t if name in ("counts", "recv_cnt") else t[:n]
    return st


def graph(c):
    """Every rank captures one device-count CUDA graph (MoEContext.forward_tokens with n_tokens=<int32 tensor>) and
    replays it with its own token count, on varlen's schedule; rows past n of x hold NaN.  A second context on every
    rank runs the same forwards eagerly with host-side counts; each replay's output and routing tables must equal them
    bit for bit."""
    cfg = c.cfg
    g = torch.Generator().manual_seed(3000 + 31 * c.ci + c.rank)
    wg = c.randn(torch.Generator().manual_seed(1999 + c.ci), cfg.H, cfg.E)
    we = c.randn(g, c.nlx, 2, cfg.P, cfg.H)
    ctx, ref = c.context(), c.context()
    x_full = torch.empty(cfg.S, cfg.H, dtype=torch.bfloat16, device=c.dev)
    out_full = torch.empty_like(x_full)
    n_dev = torch.zeros(1, dtype=torch.int32, device=c.dev)
    cuda_graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(cuda_graph):
        ctx.forward_tokens(x_full, wg, we, out=out_full, n_tokens=n_dev)
    for it, n in enumerate(varlen_counts(c)):
        xn = c.randn(g, n, cfg.H, scale=1)
        x_full[:n].copy_(xn)
        x_full[n:].view(torch.int16).fill_(-64)   # bf16 NaN
        n_dev.fill_(n)
        cuda_graph.replay()
        got = launch_state(ctx, out_full, n)
        want = launch_state(ref, ref.forward_tokens(xn, wg, we), n)
        for name in want:
            c.same_bits(got[name], want[name], it, n, name)


# ------------------------------------------------------------------ shared
SHARED = [
    dict(num_experts=8, expert_top_k=2, sequence_len=512, hidden_size=256, intermediate_size=512),
    dict(num_experts=8, expert_top_k=3, sequence_len=256, hidden_size=128, intermediate_size=256, hidden_act=1),
]


def shared_counts(c):
    S = c.cfg.S
    return [S, 1 + 194 % S, S - 5] if c.rank == 0 else [S, 200, 0]


def shared(c):
    """A shared expert per rank, each rank with its own shared weights.  In every round all ranks first run without
    one (plain), then rank 0 alone passes its shared expert, then every rank does.  A rank that passed one must have
    out = rne(plain + shared_y) bit for bit, and a rank that did not must have plain."""
    cfg, ps = c.cfg, 320
    g = torch.Generator().manual_seed(4000 + 31 * c.ci + c.rank)
    we = c.randn(g, c.nlx, 2, cfg.P, cfg.H)
    wg = c.randn(torch.Generator().manual_seed(90 + c.ci), cfg.H, cfg.E)
    se = SharedExpert(c.randn(g, 2, ps, cfg.H), c.randn(g, ps, scale=0.1), c.randn(g, cfg.H, scale=0.1))
    ctx = c.context(shared_inter=ps)
    for it, n in enumerate(shared_counts(c)):
        x = c.randn(g, n, cfg.H, scale=1)
        plain = ctx.forward_tokens(x, wg, we).clone()
        ctx.synchronize()
        for who in ("rank 0", "every rank"):
            mine = who == "every rank" or c.rank == 0
            out = ctx.forward_tokens(x, wg, we, shared_expert=se if mine else None)
            ctx.synchronize()
            if mine:
                sy = torch.from_numpy(ctx.read("shared_y")[:n].copy()).view(torch.bfloat16).to(c.dev)
                want = (plain.float() + sy.float()).bfloat16()
            else:
                want = plain
            c.same_bits(out, want, it, n, f"out (shared expert passed by {who})")


# ------------------------------------------------------------------ swiglu
SWIGLU = [
    dict(_route="router", num_experts=16, expert_top_k=2, sequence_len=512, hidden_size=320, intermediate_size=320,
         hidden_act=2),
    dict(_route="router", num_experts=16, expert_top_k=3, sequence_len=256, hidden_size=256, intermediate_size=192,
         hidden_act=2),
    dict(_route="routed", num_experts=16, expert_top_k=2, sequence_len=512, hidden_size=256, intermediate_size=384,
         hidden_act=2),
    dict(_route="gated", num_experts=16, expert_top_k=4, sequence_len=256, hidden_size=320, intermediate_size=192,
         hidden_act=2),
]


def swiglu_counts(c):
    S = c.cfg.S
    return [S, [S - 5, 200][c.rank % 2], [1, 0][c.rank % 2]]


def swiglu(c):
    """SwiGLU experts (hidden_act = 2).  Every rank holds its slice [nLx, 3, P, H] of one set of E experts (the W_down
    block at matrix 2 of the gated layout, reached through the dispatched packets of every source rank) and its own
    tokens and count; on the built-in router, the caller's routing (-1 picks) or the DeepSeek-V3 rule, with biases,
    without and with a [3, Ps, H] shared expert.  Each rank's out must equal, bit for bit, a one-rank context holding
    all E experts on the same tokens: routing, h, y and the combine are per token and do not depend on where an expert
    runs."""
    cfg, route, ps = c.cfg, c.entry["_route"], 192
    E, k, H = cfg.E, cfg.k, cfg.H
    gw = torch.Generator().manual_seed(500 + c.ci)   # the same weights on every rank
    we_all, we = c.experts(gw)
    bu_all, bd_all = c.randn(gw, E, 2, cfg.P, scale=0.1), c.randn(gw, E, H, scale=0.1)
    bu, bd = (b[c.rank * c.nlx:(c.rank + 1) * c.nlx].contiguous() for b in (bu_all, bd_all))
    wg = c.randn(gw, H, E)
    se = SharedExpert(c.randn(gw, 3, ps, H), c.randn(gw, 2, ps, scale=0.1), c.randn(gw, H, scale=0.1))
    ctx, one = c.context(shared_inter=ps), c.context(one_rank=True, shared_inter=ps)
    g = torch.Generator().manual_seed(600 + 31 * c.ci + c.rank)   # this rank's tokens
    for it, n in enumerate(swiglu_counts(c)):
        x = c.randn(g, n, H, scale=1)
        idx = torch.randint(-1, E, (n, k), generator=g, dtype=torch.int32).to(c.dev)
        w = torch.rand(n, k, generator=g).to(c.dev)
        for shared_expert in (None, se):
            def call(ctx, weights, b_up, b_down):
                kwargs = dict(bias_up=b_up, bias_down=b_down, shared_expert=shared_expert)
                if route == "routed":
                    return ctx.forward_routed(x, idx, w, weights, **kwargs)
                if route == "gated":
                    return ctx.forward_gated(x, wg, weights, V3, **kwargs)
                return ctx.forward_tokens(x, wg, weights, **kwargs)

            got = call(ctx, we, bu, bd).clone()
            ctx.synchronize()
            want = call(one, we_all, bu_all, bd_all)
            one.synchronize()
            c.same_bits(got, want, it, n, f"out ({route}, shared expert: {shared_expert is not None})")


# ------------------------------------------------------------------ weight_on_input
WEIGHT_ON_INPUT = [
    dict(num_experts=8, expert_top_k=1, sequence_len=512, hidden_size=256, intermediate_size=384, hidden_act=2),
    dict(num_experts=16, expert_top_k=1, sequence_len=256, hidden_size=128, intermediate_size=256, hidden_act=0),
]


def weight_on_input_launches(c):
    """This rank's token count per launch, with the caller's weights on the even launches.  Both come from one
    generator, so a rank's later counts depend on its earlier ones."""
    rng = np.random.default_rng(700 + c.ci)
    for it, counts in enumerate(token_counts(rng, c.cfg.S, c.world, 4, full=3)):
        n = counts[c.rank]
        yield n, (rng.random((n, 1)).astype(np.float32) * 1.5 if it % 2 == 0 else None)


def weight_on_input(c):
    """The router weight on the input on the even ranks only (fm_set_weight_on_input; each rank's own setting governs
    the rows it sends), on the caller's routing and on the gated Llama 4 rule.  Each rank's out must be bit-identical
    to a one-rank context holding all E experts with that rank's setting, run on that rank's tokens."""
    cfg, on = c.cfg, c.rank % 2 == 0
    g = torch.Generator().manual_seed(5000 + 31 * c.ci + c.rank)
    we_all, we = c.experts(torch.Generator().manual_seed(97 + c.ci))
    wg = c.randn(torch.Generator().manual_seed(98 + c.ci), cfg.H, cfg.E)
    ctx, one = c.context(weight_on_input=on), c.context(one_rank=True, weight_on_input=on)
    for it, (n, w) in enumerate(weight_on_input_launches(c)):
        x = c.randn(g, n, cfg.H, scale=1)
        if w is None:
            got = ctx.forward_gated(x, wg, we, LLAMA4).clone()
            ctx.synchronize()
            want = one.forward_gated(x, wg, we_all, LLAMA4)
        else:
            topk, _ = ex.routing_case(n, cfg.E, 1, seed=1000 * c.ci + 10 * it + c.rank, hot=c.rank % cfg.E)
            idx_d, w_d = torch.from_numpy(topk).to(c.dev), torch.from_numpy(w).to(c.dev)
            got = ctx.forward_routed(x, idx_d, w_d, we).clone()
            ctx.synchronize()
            want = one.forward_routed(x, idx_d, w_d, we_all)
        one.synchronize()
        c.same_bits(got, want, it, n, f"out (weight on input: {on})")


SCENARIOS = {   # name: (cases, this rank's token count per launch, run)
    "parity": (PARITY, parity_counts, parity),
    "parity_small": ([PARITY[0], PARITY[2]], parity_counts, parity),
    "routed": (ROUTED, routed_counts, routed),
    "varlen": (VARLEN, varlen_counts, varlen),
    "graph": (VARLEN, varlen_counts, graph),
    "shared": (SHARED, shared_counts, shared),
    "swiglu": (SWIGLU, swiglu_counts, swiglu),
    "weight_on_input": (WEIGHT_ON_INPUT, lambda c: [n for n, _ in weight_on_input_launches(c)], weight_on_input),
}


def main():
    name = sys.argv[1]
    cases, _, run = SCENARIOS[name]
    rank, world, local = env_rank_world()
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group(backend="cpu:gloo,cuda:nccl", rank=rank, world_size=world, device_id=dev)
    for ci, entry in enumerate(cases):
        c = Case(ci, config(entry), entry, rank, world, dev)
        if c.cfg.E % world:
            continue
        note = run(c)
        print(f"RANK {rank} {name} case {ci} OK" + (f" {note}" if note else ""), flush=True)
        dist.barrier()
        for ctx in c.contexts:
            ctx.close()
        dist.barrier()
    dist.destroy_process_group()
    print(f"RANK {rank} {name} ALL OK", flush=True)


if __name__ == "__main__":
    main()
