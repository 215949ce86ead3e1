"""Forwards on fewer tokens than the context's S (MoEContext.forward_tokens -> fm_moe_forward_tokens) on one H100: parity
with the oracle at the call's own capacity EC(n), bit-identity with a context created for S = n on every kernel path,
changing counts on one context, no writes past row n, training-mode aux loss and the nn.Module wrapper."""
import numpy as np
import pytest
import torch

from flashmoe_b200.config import MoEConfig
from oracle import moe_oracle as mo
from tests.util import check_output, check_topk, make_inputs

pytestmark = pytest.mark.gpu

BASE = MoEConfig(num_experts=8, expert_top_k=2, sequence_len=512, hidden_size=256, intermediate_size=512)


def _ctx(cfg):
    from flashmoe_b200.runtime import MoEContext

    return MoEContext(cfg, timeout_ms=5000)


def _oracle(cfg, xn, wg, we, bu=None, bd=None):
    """The layer over the n rows of xn ([n, H] bf16, CPU) with the capacity of n tokens."""
    n = xn.shape[0]
    up, down = mo.split_expert_weights(mo.to_bits(we))
    return mo.forward(mo.to_bits(xn), mo.gate_weights_effective(mo.to_bits(wg), cfg.E, cfg.H), up, down, k=cfg.k,
                      EC=cfg.EC_of(n), act=cfg.hidden_act, b_up=None if bu is None else mo.to_bits(bu),
                      b_down=None if bd is None else mo.to_bits(bd))


def _tables(ctx, n):
    return {"topk_idx": ctx.read("topk_idx")[:n], "topk_w": ctx.read("topk_w")[:n], "slot": ctx.read("slot")[:n],
            "mcw": ctx.read("mcw")[:n], "counts": ctx.read("counts")}


def _check_against_oracle(ctx, cfg, out, n, ref, what):
    t = _tables(ctx, n)
    mism = check_topk(t["topk_idx"], ref)
    if not mism.any():
        assert (t["slot"] == ref.slot).all(), f"{what}: slots"
        assert (t["counts"] == ref.counts).all(), f"{what}: counts"
    check_output(mo.to_bits(out.cpu().reshape(n, cfg.H)), ref.out, rows_ok=~mism, what=what)


@pytest.mark.parametrize("E", [8, 32, 1], ids=["router_cuda_cores", "router_tensor_cores", "dense_E1"])
def test_parity_with_oracle_over_token_counts(E):
    """Token counts below one box of the maps over x (32 rows for the tensor-core router, 128 for the dense GEMM0) read
    only the caller's n rows: the boxes' missing rows read as zero."""
    cfg = BASE.replace(num_experts=E, expert_top_k=min(2, E))
    x, wg, we, _, _ = make_inputs(cfg, seed=901)
    xs = x.reshape(cfg.S, cfg.H)
    ctx = _ctx(cfg)
    dev = ctx.device
    xd, wgd, wed = xs.to(dev), wg.to(dev), we.to(dev)
    for n in (1, 7, 31, 128, 129, 300, 512):
        out = ctx.forward_tokens(xd[:n], wgd, wed)
        ctx.synchronize()
        assert out.shape == (n, cfg.H) and ctx.last_tokens == n
        _check_against_oracle(ctx, cfg, out, n, _oracle(cfg, xs[:n], wg, we), f"n={n}")
    ctx.close()


# every kernel path that a token count could reach differently: router (CUDA cores / tensor cores, one and two passes
# over d_model), combine (fused / gather, k = 3), the dense E = 1 path, bias + GELU
PATHS = {
    "router_cuda_cores": (BASE, {}),
    "router_tensor_cores_E32": (BASE.replace(num_experts=32), {}),
    "router_tensor_cores_E160": (BASE.replace(num_experts=160, intermediate_size=256), {}),
    "gather_combine": (BASE, {"FM_FUSED_COMBINE": "0"}),
    "gather_combine_k3": (BASE.replace(expert_top_k=3), {}),
    "dense_E1": (BASE.replace(num_experts=1, expert_top_k=1), {}),
    "bias_gelu": (BASE.replace(hidden_act=1), {}),
}


@pytest.mark.parametrize("path", list(PATHS))
def test_bit_identical_to_a_context_created_for_n_tokens(monkeypatch, path):
    cfg, env = PATHS[path]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    bias = path == "bias_gelu"
    x, wg, we, bu, bd = make_inputs(cfg, seed=902, bias=bias)
    ctx = _ctx(cfg)
    dev = ctx.device
    xd, wgd, wed = x.reshape(cfg.S, cfg.H).to(dev), wg.to(dev), we.to(dev)
    bud, bdd = (bu.to(dev), bd.to(dev)) if bias else (None, None)
    for n in (128, 256, 384):
        got = ctx.forward_tokens(xd[:n], wgd, wed, bias_up=bud, bias_down=bdd)
        ctx.synchronize()
        t_got = _tables(ctx, n)
        small = _ctx(cfg.replace(sequence_len=n))
        want = small.forward(xd[:n].reshape(1, n, cfg.H), wgd, wed, bias_up=bud, bias_down=bdd)
        small.synchronize()
        t_want = _tables(small, n)
        small.close()
        assert torch.equal(got.view(torch.int16), want.view(n, cfg.H).view(torch.int16)), f"{path} n={n}: out"
        for name in t_got:
            assert np.array_equal(t_got[name], t_want[name]), f"{path} n={n}: {name}"
    # n = S: the same kernel launch as forward
    a = ctx.forward_tokens(xd, wgd, wed, bias_up=bud, bias_down=bdd).clone()
    ta = _tables(ctx, cfg.S)
    b = ctx.forward(xd.view(1, cfg.S, cfg.H), wgd, wed, bias_up=bud, bias_down=bdd)
    ctx.synchronize()
    assert torch.equal(a.view(torch.int16), b.view(cfg.S, cfg.H).view(torch.int16)), f"{path}: n = S"
    for name, v in _tables(ctx, cfg.S).items():
        assert np.array_equal(ta[name], v), f"{path} n = S: {name}"
    ctx.close()


@pytest.mark.parametrize("fused", [1, 0])
def test_changing_token_counts_on_one_context(monkeypatch, fused):
    """Counts going up and down, including 0: rows, counts or flags left by a larger earlier call cannot hide."""
    monkeypatch.setenv("FM_FUSED_COMBINE", str(fused))
    cfg = BASE
    _, wg, we, _, _ = make_inputs(cfg, seed=903)
    ctx = _ctx(cfg)
    dev = ctx.device
    wgd, wed = wg.to(dev), we.to(dev)
    g = torch.Generator().manual_seed(904)
    for i, n in enumerate((512, 3, 300, 1, 512, 129, 0, 64, 512)):
        xn = torch.randn(n, cfg.H, generator=g).bfloat16()
        out = ctx.forward_tokens(xn.to(dev), wgd, wed)
        ctx.synchronize()
        if n == 0:
            assert out.numel() == 0
            assert (ctx.read("counts") == 0).all() and (ctx.read("recv_cnt") == 0).all()
            continue
        _check_against_oracle(ctx, cfg, out, n, _oracle(cfg, xn, wg, we), f"call {i} (n={n})")
    ctx.close()


@pytest.mark.parametrize("fused", [1, 0])
def test_nothing_is_written_past_row_n(monkeypatch, fused):
    monkeypatch.setenv("FM_FUSED_COMBINE", str(fused))
    cfg = BASE
    x, wg, we, _, _ = make_inputs(cfg, seed=905)
    xs = x.reshape(cfg.S, cfg.H)
    ctx = _ctx(cfg)
    dev = ctx.device
    xd, wgd, wed = xs.to(dev), wg.to(dev), we.to(dev)
    sentinel = torch.full((cfg.S, cfg.H), 0x7F7F, dtype=torch.int16, device=dev)   # bf16 3.39e38, bit pattern checked
    for n in (1, 129, 300):
        big = sentinel.clone().view(torch.bfloat16)
        out = ctx.forward_tokens(xd[:n], wgd, wed, out=big[:n])
        ctx.synchronize()
        assert out.data_ptr() == big.data_ptr()
        assert torch.equal(big.view(torch.int16)[n:], sentinel[n:]), f"n={n}: rows past n were written"
        # rows below n: the same result as into a tensor of exactly n rows (whose oracle parity the tests above check)
        alone = ctx.forward_tokens(xd[:n], wgd, wed)
        ctx.synchronize()
        assert torch.equal(out.view(torch.int16), alone.view(torch.int16)), f"n={n}"
    ctx.close()


def test_training_mode_aux_loss_over_n_tokens():
    cfg = BASE.replace(is_training=1)
    x, wg, we, _, _ = make_inputs(cfg, seed=906)
    xs = x.reshape(cfg.S, cfg.H)
    ctx = _ctx(cfg)
    dev = ctx.device
    xd, wgd, wed = xs.to(dev), wg.to(dev), we.to(dev)
    n = 300
    out = ctx.forward_tokens(xd[:n], wgd, wed)
    ctx.synchronize()
    aux = ctx.read("aux_loss")
    gml, gmec, loss = mo.aux_loss(mo.to_bits(xs[:n]), mo.gate_weights_effective(mo.to_bits(wg), cfg.E, cfg.H), k=cfg.k,
                                  EC=cfg.EC_of(n))
    ref = _oracle(cfg, xs[:n], wg, we)
    mism = check_topk(ctx.read("topk_idx")[:n], ref)
    np.testing.assert_allclose(aux[:cfg.E], gml, rtol=2e-5, atol=1e-7)
    if not mism.any():
        np.testing.assert_allclose(aux[cfg.E:2 * cfg.E], gmec, rtol=1e-6)
        np.testing.assert_allclose(aux[2 * cfg.E], loss, rtol=2e-5)
    check_output(mo.to_bits(out.cpu()), ref.out, rows_ok=~mism)
    ctx.forward_tokens(xd[:0], wgd, wed)   # no tokens: the loss terms are zero
    ctx.synchronize()
    assert (ctx.read("aux_loss") == 0).all()
    ctx.close()


def test_layer_runs_fewer_tokens_than_its_size():
    from flashmoe_b200.layer import FlashMoELayer

    cfg = BASE
    torch.manual_seed(907)
    layer = FlashMoELayer(cfg)
    x = torch.randn(2, 100, cfg.H, device=layer.ctx.device).bfloat16()
    res = layer(x, return_routing=True)
    n = 200
    assert res.out.shape == x.shape
    assert res.topk_idx.shape == (n, cfg.k) and res.topk_weight.shape == (n, cfg.k) and res.slot.shape == (n, cfg.k)
    ref = _oracle(cfg, x.cpu().reshape(n, cfg.H), layer.gate_weight.data.cpu(), layer.expert_weight.data.cpu())
    mism = check_topk(res.topk_idx.numpy(), ref)
    assert (res.slot.numpy()[~mism] == ref.slot[~mism]).all()
    check_output(mo.to_bits(res.out.cpu().reshape(n, cfg.H)), ref.out, rows_ok=~mism)
    with pytest.raises(RuntimeError, match="more than"):
        layer(torch.zeros(1, cfg.S + 1, cfg.H, device=layer.ctx.device, dtype=torch.bfloat16))
    layer.ctx.close()


def test_out_of_range_token_count_is_rejected_by_the_c_abi():
    cfg = BASE
    _, wg, we, _, _ = make_inputs(cfg, seed=908)
    ctx = _ctx(cfg)
    dev = ctx.device
    x = torch.zeros(cfg.S + 128, cfg.H, dtype=torch.bfloat16, device=dev)
    out = torch.empty_like(x)
    wgd, wed = wg.to(dev), we.to(dev)
    for n in (-1, cfg.S + 1):
        rc = ctx._L.fm_moe_forward_tokens(ctx._ctx, x.data_ptr(), n, wgd.data_ptr(), wed.data_ptr(), None, None,
                                          out.data_ptr(), torch.cuda.current_stream(dev).cuda_stream)
        assert rc == -1 and b"n_tokens" in ctx._L.fm_last_error()
    ctx.close()
