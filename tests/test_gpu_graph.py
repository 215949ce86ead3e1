"""Forwards captured in CUDA graphs and forwards whose token count is in device memory (MoEContext.forward_tokens(...,
n_tokens=<int32 tensor>) -> fm_moe_forward_tokens_dev) on one H100.  Every comparison is bitwise, on `out` and on the
routing tables, against eager host-count calls: graphs captured per n and replayed on changing inputs, eager calls and
replays interleaved on one context, one device-count graph replayed over changing counts with NaN past row n of x,
the training-mode loss, out-of-range counts, the nn.Module wrapper, and one case checked stage by stage on inputs
whose sums are exact (tests/exact.py)."""
import numpy as np
import pytest
import torch

from flashmoe_b200._lib import FlashMoEError
from flashmoe_b200.config import MoEConfig
from tests import exact as ex
from tests.util import make_inputs

pytestmark = pytest.mark.gpu

BASE = MoEConfig(num_experts=8, expert_top_k=2, sequence_len=512, hidden_size=256, intermediate_size=512)
# every kernel path a launch's state or a device-side count could reach differently: router (CUDA cores, tensor cores
# with one and two passes over the experts), combine (fused, gather, k = 3), dense E = 1, bias + GELU
PATHS = {
    "router_cuda_cores": (BASE, {}),
    "router_tensor_cores_E32": (BASE.replace(num_experts=32), {}),
    "router_tensor_cores_E160": (BASE.replace(num_experts=160, intermediate_size=256), {}),
    "gather_combine": (BASE, {"FM_FUSED_COMBINE": "0"}),
    "gather_combine_k3": (BASE.replace(expert_top_k=3), {}),
    "dense_E1": (BASE.replace(num_experts=1, expert_top_k=1), {}),
    "bias_gelu": (BASE.replace(hidden_act=1), {}),
}
TABLES = ("topk_idx", "topk_w", "slot", "mcw", "counts", "recv_cnt")
NAN, SENTINEL = -64, 0x7F7F   # bf16 bit patterns: 0xFFC0 (a NaN) and 3.39e38
DEVICE_COUNTS = (512, 3, 300, 1, 0, 129, 512)


def _ctx(cfg):
    from flashmoe_b200.runtime import MoEContext

    return MoEContext(cfg, timeout_ms=5000)


def _setup(monkeypatch, path, seed):
    cfg, env = PATHS[path]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    bias = path == "bias_gelu"
    x, wg, we, bu, bd = make_inputs(cfg, seed=seed, bias=bias)
    return cfg, x.reshape(cfg.S, cfg.H), (wg, we, bu, bd)


def _weights(w, dev):
    wg, we, bu, bd = w
    return dict(gate_weights=wg.to(dev), expert_weights=we.to(dev), bias_up=None if bu is None else bu.to(dev),
                bias_down=None if bd is None else bd.to(dev))


def _state(ctx, out, n):
    """out's first n rows as bits and the routing tables of the context's last launch (synchronises)."""
    ctx.synchronize()
    st = {"out": out.reshape(-1, ctx.dims["H"])[:n].view(torch.int16).cpu().numpy()}
    for name in TABLES:
        t = ctx.read(name)
        st[name] = t if name in ("counts", "recv_cnt") else t[:n]
    return st


def _assert_same(got, want, what):
    for name in want:
        assert np.array_equal(got[name], want[name]), f"{what}: {name} differs"


def _eager(ctx, xs, n, w):
    """The host-count forward on exactly n rows (no tail): the reference every other form must equal."""
    out = ctx.forward_tokens(xs[:n].contiguous(), **w)
    return _state(ctx, out, n)


def _fill_tail(xs, n):
    xs[n:].view(torch.int16).fill_(NAN)


@pytest.mark.parametrize("path", list(PATHS))
def test_graph_per_token_count_replays_equal_eager_calls(monkeypatch, path):
    """A graph captured per n (host-side count) replays on new contents of its static x, three times per n; each replay
    is followed by the eager call on the same inputs, on the same context."""
    cfg, xs_cpu, w = _setup(monkeypatch, path, seed=1101)
    ctx = _ctx(cfg)
    dev = ctx.device
    wd = _weights(w, dev)
    xs = xs_cpu.to(dev)
    g_in = torch.Generator().manual_seed(1102)
    for n in (1, 300, cfg.S):
        static_x = torch.empty(n, cfg.H, dtype=torch.bfloat16, device=dev)
        static_x.copy_(xs[:n])
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            static_out = ctx.forward_tokens(static_x, **wd)
        for rep in range(3):
            static_x.copy_(torch.randn(n, cfg.H, generator=g_in).bfloat16())
            graph.replay()
            got = _state(ctx, static_out, n)
            _assert_same(got, _eager(ctx, static_x, n, wd), f"{path} n={n} replay {rep}")
    ctx.close()


@pytest.mark.parametrize("fused", [1, 0])
def test_eager_calls_and_replays_interleaved_on_one_context(monkeypatch, fused):
    """About ten launches on one context -- eager host-count calls, replays of a host-count graph, replays of a
    device-count graph, eager device-count calls -- each equal to the same forward on a second context that only ever
    runs eagerly.  A frozen epoch, barrier target or parity buffer would break the launch after a replay."""
    monkeypatch.setenv("FM_FUSED_COMBINE", str(fused))
    cfg = BASE
    _, wg, we, _, _ = make_inputs(cfg, seed=1201)
    ctx, ref = _ctx(cfg), _ctx(cfg)
    dev = ctx.device
    wd = _weights((wg, we, None, None), dev)
    g_in = torch.Generator().manual_seed(1202)
    n_fixed = 200
    x_fixed = torch.empty(n_fixed, cfg.H, dtype=torch.bfloat16, device=dev)
    x_full = torch.zeros(cfg.S, cfg.H, dtype=torch.bfloat16, device=dev)
    out_full = torch.empty_like(x_full)
    n_dev = torch.zeros(1, dtype=torch.int32, device=dev)
    g_fixed, g_dev = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
    with torch.cuda.graph(g_fixed):
        out_fixed = ctx.forward_tokens(x_fixed, **wd)
    with torch.cuda.graph(g_dev):
        ctx.forward_tokens(x_full, out=out_full, n_tokens=n_dev, **wd)
    seq = ["eager", "graph", "graph", "eager", "dev_graph", "eager", "dev_eager", "dev_graph", "graph", "eager"]
    for i, kind in enumerate(seq):
        n = n_fixed if kind == "graph" else (17, 512, 129, 300, 1, 256, 77, 400, 64, 333)[i]
        xn = torch.randn(n, cfg.H, generator=g_in).bfloat16().to(dev)
        if kind == "eager":
            got = _state(ctx, ctx.forward_tokens(xn, **wd), n)
        elif kind == "graph":
            x_fixed.copy_(xn)
            g_fixed.replay()
            got = _state(ctx, out_fixed, n)
        else:
            x_full[:n].copy_(xn)
            _fill_tail(x_full, n)
            n_dev.fill_(n)
            if kind == "dev_graph":
                g_dev.replay()
            else:
                ctx.forward_tokens(x_full, out=out_full, n_tokens=n_dev, **wd)
            got = _state(ctx, out_full, n)
            assert ctx.launch_record()[1] == n
        _assert_same(got, _eager(ref, xn, n, wd), f"launch {i} ({kind}, n={n})")
    launches, _ = ctx.launch_record()
    assert launches == len(seq) and ctx.launch_count == 2 + seq.count("eager") + seq.count("dev_eager")
    ctx.close()
    ref.close()


def _device_count_run(ctx, cfg, xs, wd, counts, replay):
    """x_full holds S rows: the first n from xs, NaN past them; out_full holds a sentinel past row n.  Returns the
    states of the launches (`replay`: one captured device-count graph; otherwise eager device-count calls)."""
    dev = ctx.device
    x_full = torch.empty(cfg.S, cfg.H, dtype=torch.bfloat16, device=dev)
    out_full = torch.empty_like(x_full)
    n_dev = torch.zeros(1, dtype=torch.int32, device=dev)
    graph = None
    if replay:
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            ctx.forward_tokens(x_full, out=out_full, n_tokens=n_dev, **wd)
    states = []
    for n in counts:
        x_full.copy_(xs)
        _fill_tail(x_full, n)
        out_full.view(torch.int16).fill_(SENTINEL)
        n_dev.fill_(n)
        if replay:
            graph.replay()
        else:
            ctx.forward_tokens(x_full, out=out_full, n_tokens=n_dev, **wd)
        st = _state(ctx, out_full, n)
        tail = out_full[n:].view(torch.int16)
        assert bool((tail == SENTINEL).all()), f"n={n}: rows at or past n of out were written"
        assert ctx.launch_record()[1] == n and ctx.last_tokens is None
        states.append(st)
    return states


@pytest.mark.parametrize("path", list(PATHS))
def test_device_count_graph_over_changing_counts(monkeypatch, path):
    """One device-count graph replayed with n = 512, 3, 300, 1, 0, 129, 512 and NaN in x past row n; then the same
    counts as eager device-count calls.  Both equal the host-count forward on the n rows alone."""
    cfg, xs_cpu, w = _setup(monkeypatch, path, seed=1301)
    ctx, ref = _ctx(cfg), _ctx(cfg)
    dev = ctx.device
    wd = _weights(w, dev)
    xs = xs_cpu.to(dev)
    want = [_eager(ref, xs, n, wd) for n in DEVICE_COUNTS]
    for replay in (True, False):
        got = _device_count_run(ctx, cfg, xs, wd, DEVICE_COUNTS, replay)
        for n, g, r in zip(DEVICE_COUNTS, got, want):
            _assert_same(g, r, f"{path} {'replay' if replay else 'eager'} n={n}")
    ctx.close()
    ref.close()


def test_training_mode_aux_loss_after_replays():
    """is_training = 1: the loss buffer read after each replay of a device-count graph is the eager call's.  gML and the
    loss are sums of per-CTA float atomics, whose order varies between launches: they agree to rounding; the routed
    fractions gMeC are exact."""
    cfg = BASE.replace(is_training=1)
    x, wg, we, _, _ = make_inputs(cfg, seed=1401)
    ctx, ref = _ctx(cfg), _ctx(cfg)
    dev = ctx.device
    wd = _weights((wg, we, None, None), dev)
    xs = x.reshape(cfg.S, cfg.H).to(dev)
    x_full = torch.empty_like(xs)
    out_full = torch.empty_like(xs)
    n_dev = torch.zeros(1, dtype=torch.int32, device=dev)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ctx.forward_tokens(x_full, out=out_full, n_tokens=n_dev, **wd)
    E = cfg.E
    for n in (300, 512, 0, 1, 129):
        x_full.copy_(xs)
        _fill_tail(x_full, n)
        n_dev.fill_(n)
        graph.replay()
        got = _state(ctx, out_full, n)
        aux = ctx.read("aux_loss")
        want = _eager(ref, xs, n, wd)
        aux_ref = ref.read("aux_loss")
        _assert_same(got, want, f"n={n}")
        assert np.array_equal(aux[E:2 * E], aux_ref[E:2 * E]), f"n={n}: gMeC"
        np.testing.assert_allclose(aux[:E], aux_ref[:E], rtol=1e-5, atol=1e-7, err_msg=f"n={n}: gML")
        np.testing.assert_allclose(aux[2 * E], aux_ref[2 * E], rtol=1e-5, atol=1e-7, err_msg=f"n={n}: loss")
        if n == 0:
            assert (aux == 0).all()
    ctx.close()
    ref.close()


@pytest.mark.parametrize("bad", [-1, 513], ids=["minus_one", "S_plus_one"])
def test_out_of_range_device_count_is_reported_and_the_context_stays_usable(bad):
    cfg = BASE
    x, wg, we, _, _ = make_inputs(cfg, seed=1501)
    ctx, ref = _ctx(cfg), _ctx(cfg)
    dev = ctx.device
    wd = _weights((wg, we, None, None), dev)
    xs = x.reshape(cfg.S, cfg.H).to(dev)
    out_full = torch.empty_like(xs)
    n_dev = torch.full((1,), bad, dtype=torch.int32, device=dev)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ctx.forward_tokens(xs, out=out_full, n_tokens=n_dev, **wd)
    for replay in (False, True):
        n_dev.fill_(bad)
        out_full.view(torch.int16).fill_(SENTINEL)
        if replay:
            graph.replay()
        else:
            ctx.forward_tokens(xs, out=out_full, n_tokens=n_dev, **wd)
        with pytest.raises(FlashMoEError, match=f"n_tokens = {bad} not in \\[0, S = {cfg.S}\\]"):
            ctx.synchronize()
        ctx.check()   # reported once
        assert ctx.launch_record()[1] == 0
        assert bool((out_full.view(torch.int16) == SENTINEL).all()), "a launch on 0 tokens wrote out"
        # the next valid launch is exact
        n = 300
        n_dev.fill_(n)
        graph.replay()
        _assert_same(_state(ctx, out_full, n), _eager(ref, xs, n, wd), f"after count {bad} ({'replay' if replay else 'eager'})")
    ctx.close()
    ref.close()


def test_layer_captured_in_a_graph():
    """FlashMoELayer.forward(x, n_tokens=...) captured once and replayed over changing counts; `routing(out)` after a
    replay returns that replay's tables, equal to the layer's eager call on the n rows."""
    from flashmoe_b200.layer import FlashMoELayer

    cfg = BASE
    torch.manual_seed(1601)
    layer = FlashMoELayer(cfg)
    dev = layer.ctx.device
    xs = torch.randn(1, cfg.S, cfg.H, device=dev).bfloat16()
    x_full = torch.empty_like(xs)
    n_dev = torch.zeros(1, dtype=torch.int32, device=dev)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = layer(x_full, n_tokens=n_dev)
    assert out.shape == xs.shape
    for n in (100, 512, 7):
        x_full.copy_(xs)
        _fill_tail(x_full.view(cfg.S, cfg.H), n)
        n_dev.fill_(n)
        graph.replay()
        res = layer.routing(out)
        got_out = res.out[0, :n].clone()
        assert res.topk_idx.shape == (n, cfg.k)
        want = layer(xs[:, :n].contiguous(), return_routing=True)
        assert torch.equal(got_out.view(torch.int16), want.out[0].view(torch.int16)), f"n={n}: out"
        for name in ("topk_idx", "topk_weight", "slot"):
            a, b = getattr(res, name), getattr(want, name)
            assert torch.equal(a.view(torch.int16) if a.dtype == torch.bfloat16 else a,
                               b.view(torch.int16) if b.dtype == torch.bfloat16 else b), f"n={n}: {name}"
    layer.ctx.close()


def test_replayed_device_count_graph_exact_stage_by_stage():
    """Inputs whose sums are exact in fp32 (tests/exact.py), through one replayed device-count graph with NaN past row
    n: every stage -- top-k, gate_out, topk_w, mcw, slots, counts, recv_cnt, recv_x, h, out -- checked element by
    element at the capacity of n tokens."""
    cfg = MoEConfig(num_experts=8, expert_top_k=2, sequence_len=512, hidden_size=128, intermediate_size=128)
    inp = ex.exact_inputs(cfg, seed=1701, ties=[(0, cfg.E - 1), (2, 3)], zero_tokens=4, underflow_tokens=8)
    ctx = _ctx(cfg)
    run = ex.Launcher(ctx, "router", inp)
    xs = run.x
    x_full, out_full = torch.empty_like(xs), torch.empty_like(xs)
    n_dev = torch.zeros(1, dtype=torch.int32, device=ctx.device)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        run.launch(cfg.S, out=out_full, n_tokens=n_dev, x=x_full)
    st = ex.Stats()
    for n in (1, 129, 300, 512):
        x_full.copy_(xs)
        _fill_tail(x_full, n)
        n_dev.fill_(n)
        graph.replay()
        ctx.synchronize()
        d, _ = run.read(out_full[:n], n)
        run.check(d, None, n, stats=st)
    ctx.close()
    print(f"\n[device-count graph, exact] {st.line()}")
