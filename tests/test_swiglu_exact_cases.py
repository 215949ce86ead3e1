"""The SwiGLU exact-input reference (tests/exact_swiglu.py) on the CPU: its hand-built corners, agreement with torch's
float64 SwiGLU and with the torch restatement of the whole forward (tests/torch_swiglu.py) on both routes, that
restatement against oracle/torch_moe on a layout-equivalent input, the generator's conditions (g >= -64, exact GEMM
sums), the kernel's partial-tile argument replayed in float64, and the stage checker accepting a correct launch record
and rejecting a planted fault.  CPU only."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from flashmoe_b200.config import MoEConfig
from tests import exact as ex
from tests import exact_swiglu as sw


def _ref(g, u):
    """h's interval for gate and up pre-activations g and u."""
    return sw.silu_mul_rounded(np.atleast_1d(np.asarray(g, np.float64)), np.atleast_1d(np.asarray(u, np.float64)))


def test_corner_g0_is_zero():
    r = _ref([0.0, 0.0], [3.0, -5.0])
    assert (ex.bits_to_f64(r.lo) == 0).all() and (ex.bits_to_f64(r.hi) == 0).all()


def test_corner_large_g_is_rne_of_g_times_u():
    g, u = np.array([100.0, 100.0, 64.0]), np.array([3.0, -1.5, 7.0])
    r = _ref(g, u)
    want = ex.f64_to_bf16(g * u)
    assert np.array_equal(r.lo, want) and np.array_equal(r.hi, want)


@pytest.mark.parametrize("g", [-100.0, -150.0, -1000.0])
def test_corner_very_negative_g_is_zero(g):
    r = _ref([g, g], [4.0, -4.0])
    assert (ex.bits_to_f64(r.lo) == 0).all() and (ex.bits_to_f64(r.hi) == 0).all()   # -0 and +0 both accepted


def test_interval_is_at_most_one_ulp_and_contains_torch_float64():
    rng = np.random.default_rng(3)
    g = rng.integers(-128, 129, 4096) / 16.0
    u = rng.integers(-64, 65, 4096) / 4.0
    r = _ref(g, u)
    assert (ex.order_key(r.hi) - ex.order_key(r.lo) <= 1).all()
    t = (F.silu(torch.from_numpy(g)) * torch.from_numpy(u)).numpy()
    tb = ex.f64_to_bf16(t)
    assert ((ex.order_key(tb) >= ex.order_key(r.lo)) & (ex.order_key(tb) <= ex.order_key(r.hi))).all()
    # the fp32 arithmetic the kernel does, emulated with numpy's exact fp32 steps and a correctly rounded exp2
    g32 = g.astype(np.float32)
    a = (-g32 * ex.LOG2E_F32).astype(np.float32)
    with np.errstate(over="ignore"):
        sig = (np.float32(1) / (np.float32(1) + np.exp2(a.astype(np.float64)).astype(np.float32))).astype(np.float32)
    h32 = ((g32 * sig).astype(np.float32) * u.astype(np.float32)).astype(np.float32)
    hb = ex.f32_to_bf16(h32)
    assert ((ex.order_key(hb) >= ex.order_key(r.lo)) & (ex.order_key(hb) <= ex.order_key(r.hi))).all()


def _cfg(E=4, k=2, S=256, H=128, P=192):
    return MoEConfig(num_experts=E, expert_top_k=k, sequence_len=S, hidden_size=H, intermediate_size=P, hidden_act=2)


def test_generator_keeps_g_above_minus_64_and_sums_exact():
    cfg = _cfg()
    inp = sw.swiglu_inputs(cfg, 11, bias=True)
    xp = inp.experts
    assert tuple(xp.w.shape) == (4, 3, 192, 128) and tuple(xp.bu.shape) == (4, 2, 192)
    for e in range(cfg.E):
        g, _ = xp.pre(e, inp.x64)
        assert g.min() >= sw.G_MIN
        xp.y(e, xp.h(e, inp.x64).lo)   # asserts exact sums


def test_partial_last_tile_reads_stay_in_the_tensor_and_are_not_stored():
    """Replays the kernel's tile mapping for P = 192 (= 64 mod 128) in float64: tile nt of expert e loads B rows
    [b_row, b_row + 128) and [b_row + P, b_row + P + 128) of the [E * 3P, H] view; the stored chunks of the
    accumulator columns are the reference's h, and every row read lies inside the tensor."""
    cfg = _cfg()
    E, P, H = cfg.E, cfg.P, cfg.H
    inp = sw.swiglu_inputs(cfg, 12, bias=True)
    xp = inp.experts
    flat = xp.w.double().numpy().reshape(E * 3 * P, H)
    x = inp.x64[:128]
    tn = -(-P // 128)
    for e in range(E):
        ref = xp.h(e, x)
        bias = xp.bu[e].double().numpy().reshape(-1)   # [gate; up], glu_rows = P apart
        for nt in range(tn):
            b_row, n0 = e * 3 * P + nt * 128, nt * 128
            assert b_row + P + 128 <= flat.shape[0]
            acc = x @ np.concatenate([flat[b_row:b_row + 128], flat[b_row + P:b_row + P + 128]]).T   # [128 rows, 256]
            for c in range(min(2, (P - n0) // 64)):
                cols = slice(64 * c, 64 * c + 64)
                g = acc[:, cols] + bias[n0 + 64 * c:n0 + 64 * c + 64]
                u = acc[:, 128 + 64 * c:128 + 64 * c + 64] + bias[P + n0 + 64 * c:P + n0 + 64 * c + 64]
                np.testing.assert_array_equal(g / (1 + np.exp(-g)) * u, ref.exact[:, n0 + 64 * c:n0 + 64 * c + 64])


def test_checker_accepts_the_reference_and_rejects_a_planted_fault():
    cfg = _cfg()
    inp = sw.swiglu_inputs(cfg, 13, bias=True, zero_tokens=2)
    dev, _ = ex.reference_launch("router", inp, cfg.EC, cfg.S)
    st = ex.Stats()
    ex.check_launch("router", inp, cfg.EC, cfg.S, dev, stats=st)
    h = st.d["hidden"]
    assert h[1] > 0.5 * h[0], "the inputs must make h round"
    e = int(np.flatnonzero(dev.recv_cnt)[0])
    j = int(np.flatnonzero(dev.hidden[e, 0])[0])
    dev.hidden[e, 0, j] += 2   # two bf16 ulps off
    with pytest.raises(AssertionError, match=f"hidden of expert {e}"):
        ex.check_launch("router", inp, cfg.EC, cfg.S, dev)


def _torch_device(res, E, EC):
    """A launch record from tests/torch_swiglu.py's forward (its own routing, h, y and out)."""
    idx = res["topk_idx"].numpy()
    valid = idx >= 0
    counts = np.bincount(idx[valid], minlength=E).astype(np.int32)
    return ex.Device(ex.to_bits(res["out"]), idx, ex.to_bits(res["topk_w"].bfloat16()), res["mcw"].numpy(), None,
                     res["slot"].numpy(), counts, np.minimum(counts, EC).astype(np.int32), None,
                     ex.to_bits(res["hidden"]), ex.to_bits(res["ret_y"]))


@pytest.mark.parametrize("k,bias", [(1, True), (2, True), (4, False)])
def test_reference_agrees_with_torch_swiglu_router(k, bias):
    """The float64 reference against the torch restatement on exact inputs: its routing, every h inside the interval,
    y bit for bit from that h, and out inside the combine's interval."""
    from tests.torch_swiglu import moe_forward_swiglu_cpu

    cfg = _cfg(k=k)
    inp = sw.swiglu_inputs(cfg, 20 + k, bias=bias, zero_tokens=2)
    res = moe_forward_swiglu_cpu(inp.x.reshape(cfg.S, cfg.H), inp.wg, inp.experts.w, k=k, EC=cfg.EC,
                                 bias_up=inp.experts.bu, bias_down=inp.experts.bd)
    dev = _torch_device(res, cfg.E, cfg.EC)
    # gate_out: the reference's own, with the torch forward's weights at its picks (they must lie in the interval)
    dev.gate_out = ex.reference_launch("router", inp, cfg.EC, cfg.S)[0].gate_out
    dev.gate_out[np.arange(cfg.S)[:, None], dev.topk_idx] = dev.topk_w
    st = ex.Stats()
    ex.check_launch("router", inp, cfg.EC, cfg.S, dev, stats=st)
    assert st.d["hidden"][0] > 0 and st.d["ret_y"][0] > 0


@pytest.mark.parametrize("k", [1, 2])
def test_reference_agrees_with_torch_swiglu_routed(k):
    from tests.torch_swiglu import moe_forward_swiglu_routed_cpu

    cfg = _cfg(k=k)
    inp = sw.swiglu_inputs(cfg, 30 + k, bias=True)
    xp = inp.experts
    idx, w = ex.routing_case(cfg.S, cfg.E, k, 30 + k, hot=1, hot_frac=0.4, empty=(3,))
    res = moe_forward_swiglu_routed_cpu(inp.x.reshape(cfg.S, cfg.H), torch.from_numpy(idx), torch.from_numpy(w),
                                        xp.w, EC=cfg.EC, bias_up=xp.bu, bias_down=xp.bd)
    dev = _torch_device(res, cfg.E, cfg.EC)
    ex.check_launch("routed", inp, cfg.EC, cfg.S, dev, routing=(idx, w))


def test_torch_swiglu_relu_equivalent_layout():
    """torch_swiglu reads [e,2] flat as W_down and combines exactly as oracle/torch_moe does with [e,1]: with every
    gate pre-activation 64 (silu(64) is 64 in fp32) and u >= 0, SwiGLU's h = 64 u equals ReLU's h for W_up = 64 up, and
    the two forwards agree bit for bit."""
    from oracle.torch_moe import moe_forward_cpu
    from tests.torch_swiglu import moe_forward_swiglu_cpu

    cfg = _cfg(k=2)
    g = torch.Generator().manual_seed(4)
    x = torch.randint(0, 3, (cfg.S, cfg.H), generator=g).bfloat16()
    wg = (torch.randn(cfg.H, cfg.E, generator=g) * 0.05).bfloat16()
    up = torch.randint(0, 3, (cfg.E, cfg.P, cfg.H), generator=g).bfloat16() * 0.125
    down = torch.randint(-2, 3, (cfg.E, cfg.P, cfg.H), generator=g).bfloat16() * 0.03125
    gate = torch.zeros(cfg.E, cfg.P, cfg.H, dtype=torch.bfloat16)
    gate[:, :, 0] = 1.0
    xg = x.clone()
    xg[:, 0] = 64.0
    relu = moe_forward_cpu(xg, wg, torch.stack([up * 64.0, down], 1), k=2, EC=cfg.EC)
    glu = moe_forward_swiglu_cpu(xg, wg, torch.stack([gate, up, down], 1), k=2, EC=cfg.EC)
    assert torch.equal(relu["topk_idx"], glu["topk_idx"])
    assert torch.equal(relu["out"].view(torch.int16), glu["out"].view(torch.int16))
