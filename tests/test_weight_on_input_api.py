"""The router weight on the input (fm_set_weight_on_input) without a GPU: the header documents the setter and _lib binds
it; MoEContext and FlashMoELayer reject k != 1 and E = 1 before any native call; tests/torch_llama4.py's statement of
Llama4TextMoe agrees with a float64 reference on exact inputs, and so does the Hugging Face layout conversion; the exact
checker (tests/exact_weight_on_input.py) accepts its own reference launches and catches the faults it exists for; the
bench script's argument and device checks."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from flashmoe_b200 import _lib
from flashmoe_b200.config import MoEConfig
from flashmoe_b200.router import RouterSpec
from tests import exact as ex
from tests import exact_weight_on_input as wi
from tests import torch_llama4 as tl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "flashmoe_b200.h")
LLAMA4 = RouterSpec("sigmoid", renormalize=False)


def test_header_declares_and_documents_the_setter():
    text = open(HEADER).read()
    assert re.search(r"FM_API int fm_set_weight_on_input\(fm_ctx_t\* ctx, int enable\);", text)
    doc = text.split("FM_API int fm_set_trace")[1].split("FM_API int fm_set_weight_on_input")[0]
    for phrase in ("rne_bf16(fl32(x[t]) * fl32(w~))", "weight 1", "fm_moe_forward_routed(x', topk_idx, ones)",
                   "FM_BUF_RECV_X holds the scaled rows", "k != 1", "E = 1", "Fixed at capture", "world > 1"):
        assert phrase in doc, phrase
    assert "fm_set_weight_on_input" in _lib.EXPORTED_SYMBOLS


def test_lib_binds_the_setter():
    try:
        L = _lib.load()
    except RuntimeError:
        pytest.skip("native library not built")
    assert L.fm_set_weight_on_input.argtypes is not None
    assert L.fm_set_weight_on_input(None, 1) == -1 and b"null context" in L.fm_last_error()


def _cfg(**kw):
    base = dict(num_experts=16, expert_top_k=1, sequence_len=256, hidden_size=256, intermediate_size=256, hidden_act=2)
    base.update(kw)
    return MoEConfig(**base)


@pytest.mark.parametrize("kw, what", [(dict(expert_top_k=2), "k = 1"), (dict(num_experts=1), "E > 1")])
def test_context_and_layer_reject_before_any_native_call(monkeypatch, kw, what):
    from flashmoe_b200.layer import FlashMoELayer
    from flashmoe_b200.runtime import MoEContext

    def no_native():
        raise AssertionError("a native call was made")

    monkeypatch.setattr(_lib, "load", no_native)
    with pytest.raises(ValueError, match=re.escape(what)):
        MoEContext(_cfg(**kw), device=0, weight_on_input=True)
    with pytest.raises(ValueError, match=re.escape(what)):
        FlashMoELayer(_cfg(**kw), device=0, weight_on_input=True)
    with pytest.raises(ValueError, match="bool"):
        MoEContext(_cfg(), device=0, weight_on_input=2)


# ----------------------------------------------------------------------------- the torch statement of Llama 4
def _hf_tensors(E, H, P, Ps, seed):
    """Hugging Face-layout tensors whose every product is exact: small integers times powers of two."""
    g = np.random.default_rng(seed)
    bf = lambda a: torch.from_numpy(np.ascontiguousarray(a)).bfloat16()   # noqa: E731
    return dict(router_w=bf(g.integers(-4, 5, size=(E, H)) * 2.0 ** -6),
                gate_up=bf(g.integers(-2, 3, size=(E, H, 2 * P)) * 2.0 ** -3),
                down=bf(g.integers(-2, 3, size=(E, P, H)) * 2.0 ** -5),
                sh_gate=bf(g.integers(-2, 3, size=(Ps, H)) * 2.0 ** -3),
                sh_up=bf(g.integers(-2, 3, size=(Ps, H)) * 2.0 ** -3),
                sh_down=bf(g.integers(-2, 3, size=(H, Ps)) * 2.0 ** -5))


def _bf16_64(a):
    return ex.bits_to_f64(ex.f64_to_bf16(a))


def _numpy_llama4(x, t):
    """float64 numpy of Llama4TextMoe with torch's bf16 roundings: every matmul and product rounded once to bf16."""
    f = {k: v.double().numpy() for k, v in t.items()}
    E = f["router_w"].shape[0]
    P = f["down"].shape[1]
    logits = _bf16_64(x @ f["router_w"].T)
    pick = np.argmax(logits, axis=1)   # (the exact inputs below have no ties)
    score = _bf16_64(1 / (1 + np.exp(-logits[np.arange(len(x)), pick].astype(np.float32).astype(np.float64))))
    silu = lambda v: _bf16_64(v / (1 + np.exp(-v)))   # noqa: E731
    routed = np.zeros_like(x)
    for e in range(E):
        xe = _bf16_64(x * np.where(pick == e, score, 0.0)[:, None])
        gu = _bf16_64(xe @ f["gate_up"][e])
        h = _bf16_64(gu[:, P:] * silu(gu[:, :P]))
        routed = routed + _bf16_64(h @ f["down"][e])   # (at most one expert's rows are nonzero per token)
    s = _bf16_64(_bf16_64(silu(_bf16_64(x @ f["sh_gate"].T)) * _bf16_64(x @ f["sh_up"].T)) @ f["sh_down"].T)
    return _bf16_64(s + _bf16_64(routed)), pick


def test_torch_llama4_agrees_with_float64_on_exact_inputs():
    E, H, P, Ps, n = 4, 64, 64, 64, 16
    t = _hf_tensors(E, H, P, Ps, 3)
    g = np.random.default_rng(4)
    x = g.integers(-2, 3, size=(n, H)).astype(np.float64)
    out, picks = tl.llama4_moe(torch.from_numpy(x).bfloat16(), **t)
    want, pick = _numpy_llama4(x, t)
    assert np.array_equal(picks[:, 0].numpy(), pick)
    got = out.double().numpy()
    np.testing.assert_allclose(got, want, rtol=2 ** -7, atol=2 ** -10)
    assert np.mean(got == want) > 0.95


def test_hf_conversion_reproduces_the_expert_outputs():
    """The converted [E, 3, P, H] experts, [3, Ps, H] shared expert and flat-viewed router give the statement's numbers
    through this project's conventions (W_down read flat as [H, P], gate_w read flat as [E, H])."""
    E, H, P, Ps, n = 4, 64, 128, 64, 8
    t = _hf_tensors(E, H, P, Ps, 5)
    we = tl.convert_experts(t["gate_up"], t["down"])
    ws = tl.convert_shared(t["sh_gate"], t["sh_up"], t["sh_down"])
    gw = tl.convert_router(t["router_w"])
    assert we.shape == (E, 3, P, H) and ws.shape == (3, Ps, H) and gw.shape == (H, E)
    assert torch.equal(gw.reshape(-1).view(E, H), t["router_w"])
    x = torch.from_numpy(np.random.default_rng(6).integers(-2, 3, size=(n, H)).astype(np.float32)).bfloat16()
    for e in range(E):
        gu = x @ t["gate_up"][e]
        y_hf = (gu[:, P:] * torch.nn.functional.silu(gu[:, :P])) @ t["down"][e]
        g, u = x @ we[e, 0].t(), x @ we[e, 1].t()
        y = (u * torch.nn.functional.silu(g)) @ we[e, 2].reshape(-1).view(H, P).t()
        assert torch.equal(y, y_hf), e
    s = tl.shared_mlp(x, t["sh_gate"], t["sh_up"], t["sh_down"])
    s2 = (torch.nn.functional.silu(x @ ws[0].t()) * (x @ ws[1].t())) @ ws[2].reshape(-1).view(H, Ps).t()
    assert torch.equal(s, s2)


# ----------------------------------------------------------------------------- the exact checker
def _case(act=2, route="routed", n=200, shared_ps=None, seed=21):
    cfg = MoEConfig(num_experts=8, expert_top_k=1, sequence_len=256, hidden_size=128, intermediate_size=192,
                    hidden_act=act)
    inp = wi.inputs(cfg, seed)
    rt = wi.routing(cfg.S, cfg.E, seed, hot=3, hot_frac=0.3)
    sh = None if shared_ps is None else wi.shared(cfg.H, shared_ps, act, seed + 7)
    EC = cfg.EC_of(n)
    dev, rec = wi.reference_launch(route, inp, EC, n, routing=rt, router=LLAMA4, shared=sh)
    return cfg, inp, rt, sh, EC, n, dev, rec


def _check(c, dev=None, rec=None):
    cfg, inp, rt, sh, EC, n, d, r = c
    return wi.check_launch("routed", inp, EC, n, d if dev is None else dev, r if rec is None else rec, routing=rt,
                           router=LLAMA4, shared=sh)


@pytest.mark.parametrize("act", [0, 1, 2])
@pytest.mark.parametrize("shared_ps", [None, 128])
def test_reference_launch_passes_its_own_checks_and_rounds(act, shared_ps):
    c = _case(act, shared_ps=shared_ps)
    st = ex.Stats()
    cfg, inp, rt, sh, EC, n, dev, rec = c
    wi.check_launch("routed", inp, EC, n, dev, rec, routing=rt, shared=sh, stats=st)
    xb = ex.f64_to_bf16(inp.x64[:n])
    kept = dev.slot[:, 0] < EC
    assert (dev.slot[:, 0] >= EC).any() and (dev.topk_idx[:, 0] < 0).any(), "no capacity drops or -1 picks"
    xs = ex.f64_to_bf16(wi.scaled_rows(inp.x64[:n], dev.topk_w))
    exact = ex.f64_to_bf16(ex.bits_to_f64(xb) * ex.bits_to_f64(dev.topk_w))
    assert (xs[kept] != xb[kept]).any()
    rounds = ex.bits_to_f64(xs) != inp.x64[:n] * ex.bits_to_f64(dev.topk_w)
    assert rounds[kept].sum() > 100, "rne(x * w~) never rounds"
    assert np.array_equal(xs, exact)
    assert st.d["recv_x"][0] > 0 and st.d["hidden"][0] > 0


def test_gated_llama4_reference_passes_its_own_checks():
    cfg, inp, rt, sh, EC, n, dev, rec = _case(route="gated", shared_ps=64)
    assert (ex.bits_to_f64(dev.topk_w) >= 0.5).all()
    wi.check_launch("gated", inp, EC, n, dev, rec, router=LLAMA4, shared=sh)


def _kept_token(dev, EC):
    """A kept token whose weight is neither 0 nor 1, so its scaled row differs from its unscaled one."""
    return next(t for t in np.flatnonzero(dev.slot[:, 0] < EC) if dev.topk_w[t, 0] not in (0x3F80, 0, 0x8000))


def _row(dev, t):
    return int(dev.topk_idx[t, 0]), int(dev.slot[t, 0])


def test_fault_unscaled_row():
    c = _case()
    dev = c[6]
    t = _kept_token(dev, c[4])
    e, s = _row(dev, t)
    dev.recv_x[e, s] = ex.f64_to_bf16(c[1].x64[t])
    with pytest.raises(AssertionError, match=f"recv_x of expert {e}"):
        _check(c)


def test_fault_row_scaled_by_another_tokens_weight():
    c = _case()
    dev = c[6]
    ts = [t for t in np.flatnonzero(dev.slot[:, 0] < c[4])]
    t, u = next((t, u) for t in ts for u in ts if dev.topk_w[t, 0] != dev.topk_w[u, 0] and c[1].x64[t].any())
    e, s = _row(dev, t)
    dev.recv_x[e, s] = ex.f64_to_bf16(wi.scaled_rows(c[1].x64[t:t + 1], dev.topk_w[u:u + 1]))[0]
    with pytest.raises(AssertionError, match=f"recv_x of expert {e}"):
        _check(c)


def test_fault_output_scaled_twice():
    c = _case()
    dev = c[6]
    t = next(t for t in np.flatnonzero(dev.slot[:, 0] < c[4])
             if ex.bits_to_f64(dev.topk_w[t, 0]) not in (0.0, 1.0) and dev.out[t].any())
    dev.out[t] = ex.f64_to_bf16(ex.bits_to_f64(dev.out[t]) * ex.bits_to_f64(dev.topk_w[t, 0]))
    with pytest.raises(AssertionError, match=f"out: .* first at token {t},"):
        _check(c)


def test_fault_shared_term_from_the_scaled_row():
    c = _case(shared_ps=128)
    cfg, inp, rt, sh, EC, n, dev, rec = c
    bad = ex.shared_stage(wi.scaled_rows(inp.x64[:n], dev.topk_w), sh)
    assert not np.array_equal(bad.h_s, rec.h_s)
    with pytest.raises(AssertionError, match="h_s"):
        _check(c, rec=bad)


# ----------------------------------------------------------------------------- the bench script
BENCH = os.path.join(ROOT, "scripts", "bench_llama4.py")


@pytest.mark.parametrize("args", [["--tokens", "-1"], ["--tokens", "x"], ["--steps", "0"]])
def test_bench_rejects_bad_arguments(args):
    r = subprocess.run([sys.executable, BENCH, *args], capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 2, r.stderr


def test_bench_needs_a_cuda_device():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    r = subprocess.run([sys.executable, BENCH, "--tokens", "1", "--steps", "1"], capture_output=True, text=True,
                       cwd=ROOT)
    assert r.returncode == 3, r.stderr
