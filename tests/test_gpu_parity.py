"""Parity tests proper: the CUDA path, called through the C-ABI (MoEContext -> ctypes -> libflashmoe_b200.so), against
the CPU oracle on the same seeded inputs, against the committed golden fixtures, and -- at BASELINE.json's full
single-GPU size -- through size-independent properties.  Needs an H100 (pytest -m gpu)."""
import glob
import os

import numpy as np
import pytest
import torch

from flashmoe_b200.config import BASELINE_CONFIGS, MoEConfig
from oracle import moe_oracle as mo
from tests.exact import slots_from_topk
from tests.test_oracle import load_golden
from tests.util import check_output, check_topk, make_inputs, run_oracle

pytestmark = pytest.mark.gpu
GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "*.npz")))


def _ctx(cfg, **kw):
    from flashmoe_b200.runtime import MoEContext

    return MoEContext(cfg, timeout_ms=5000, **kw)


def _run(cfg, x, wg, we, bu=None, bd=None):
    ctx = _ctx(cfg)
    dev = ctx.device
    args = [t.to(dev) for t in (x, wg, we)]
    out = ctx.forward(*args, bias_up=None if bu is None else bu.to(dev), bias_down=None if bd is None else bd.to(dev))
    ctx.synchronize()
    got = {"out": mo.to_bits(out.cpu().reshape(cfg.S, cfg.H)), "topk_idx": ctx.read("topk_idx"), "slot": ctx.read("slot"),
           "counts": ctx.read("counts"), "mcw": ctx.read("mcw"), "gate_out": ctx.read("gate_out"),
           "topk_w": ctx.read("topk_w"), "recv_cnt": ctx.read("recv_cnt")}
    ctx.close()
    return got


def _compare(cfg, got, ref, mcw_rtol=2e-6):
    mism = check_topk(got["topk_idx"], ref)
    # integer bookkeeping is exact given the device's own routing, whether or not an ambiguous token routed differently
    slot, counts, recv_cnt, _ = slots_from_topk(got["topk_idx"], cfg.E, cfg.EC)
    assert (got["slot"] == slot).all()
    assert (got["counts"] == counts).all()
    if "recv_cnt" in got:
        assert (got["recv_cnt"] == recv_cnt).all()
    np.testing.assert_allclose(got["mcw"][~mism], ref.mcw[~mism], rtol=mcw_rtol)
    assert (got["gate_out"] == ref.gate_out).mean() > 0.995  # bf16 probabilities; rare 1-ulp flips from ex2.approx
    return check_output(got["out"], ref.out, rows_ok=~mism)


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_matches_committed_golden_vectors(path):
    cfg, z = load_golden(path)
    x, wg, we, bu, bd = make_inputs(cfg, seed=int(z["seed"]), scaled=bool(z["scaled"]), bias=bool(z["bias"]))
    got = _run(cfg, x, wg, we, bu, bd)
    amb = z["ambiguous"]
    mism = (got["topk_idx"] != z["topk_idx"]).any(axis=1)
    assert not (mism & ~amb).any()
    if not mism.any():
        assert (got["slot"] == z["slot"]).all() and (got["counts"] == z["counts"]).all()
    check_output(got["out"], z["out"], rows_ok=~mism, what="out vs golden")


CASES = {
    "tiny": MoEConfig(num_experts=4, expert_top_k=2, sequence_len=128, hidden_size=64, intermediate_size=256),
    "small_drop": MoEConfig(num_experts=8, expert_top_k=2, sequence_len=512, hidden_size=256, intermediate_size=512),
    "small_nodrop": MoEConfig(num_experts=8, expert_top_k=2, sequence_len=512, hidden_size=256, intermediate_size=512,
                              drop_tokens=0),
    "configA_top1": BASELINE_CONFIGS["A"],
    "gelu_cf2": MoEConfig(num_experts=8, expert_top_k=2, sequence_len=256, hidden_size=128, intermediate_size=384,
                          hidden_act=1, capacity_factor=2),
    "ragged_dims": MoEConfig(num_experts=6, expert_top_k=3, sequence_len=384, hidden_size=320, intermediate_size=448),
    "E32_k2": MoEConfig(num_experts=32, expert_top_k=2, sequence_len=1024, hidden_size=512, intermediate_size=512),
    "E64_k4": MoEConfig(num_experts=64, expert_top_k=4, sequence_len=512, hidden_size=256, intermediate_size=256),
    "E128_k2": MoEConfig(num_experts=128, expert_top_k=2, sequence_len=1024, hidden_size=256, intermediate_size=256),
    # more than 128 experts: the tensor-core router takes a second pass over d_model for experts 128..E-1
    "E160_k2": MoEConfig(num_experts=160, expert_top_k=2, sequence_len=2048, hidden_size=256, intermediate_size=256),
    "E256_k2": MoEConfig(num_experts=256, expert_top_k=2, sequence_len=2048, hidden_size=256, intermediate_size=256),
    # 139 tokens per CTA: the tensor-core router walks two sub-chunks (128 + 11 tokens) with different numbers of x boxes
    # (the 64k-token sweep point has four; a stage layout that followed the sub-chunk's row count broke its last one)
    "E32_router_subchunks": MoEConfig(num_experts=32, expert_top_k=2, sequence_len=20480, hidden_size=128,
                                      intermediate_size=128),
    "E64_router_subchunks": MoEConfig(num_experts=64, expert_top_k=2, sequence_len=40960, hidden_size=128,
                                      intermediate_size=64),
    "E1_dense": MoEConfig(num_experts=1, expert_top_k=1, sequence_len=256, hidden_size=128, intermediate_size=512),
    "k8": MoEConfig(num_experts=16, expert_top_k=8, sequence_len=256, hidden_size=128, intermediate_size=256),
    "multi_seq": MoEConfig(num_experts=8, expert_top_k=2, sequence_len=256, mini_batch=3, hidden_size=128,
                           intermediate_size=256),
}


@pytest.mark.parametrize("name", list(CASES))
def test_parity_with_oracle(name):
    cfg = CASES[name]
    x, wg, we, _, _ = make_inputs(cfg, seed=100 + len(name))
    _compare(cfg, _run(cfg, x, wg, we), run_oracle(cfg, x, wg, we))


@pytest.mark.parametrize("g1_lag,fused", [(0, 1), (1, 0), (0, 0), (2, 1), (2, 0)])
@pytest.mark.parametrize("name", ["small_drop", "odd_row_blocks", "configA_top1", "ragged_dims"])
def test_alternate_kernel_modes(monkeypatch, name, g1_lag, fused):
    """The work order with GEMM1 of an expert interleaved g1_lag experts behind its GEMM0 (FM_G1_LAG=1, 2; 0 = the
    default, all GEMM0 tiles first; a lag of at least E, as 2 at configA_top1's two experts, keeps the default) and the
    gather-combine path (FM_FUSED_COMBINE=0; the default for k <= 2 is the fused GEMM1 -> combine epilogue) stay
    parity-green."""
    cases = dict(CASES)
    cases["odd_row_blocks"] = MoEConfig(num_experts=4, expert_top_k=2, sequence_len=768, hidden_size=256,
                                        intermediate_size=512)  # TCM = 3: an odd number of row blocks per packet
    cfg = cases[name]
    if g1_lag:
        monkeypatch.setenv("FM_G1_LAG", str(g1_lag))
    monkeypatch.setenv("FM_FUSED_COMBINE", str(fused))
    x, wg, we, _, _ = make_inputs(cfg, seed=300 + g1_lag * 2 + fused)
    _compare(cfg, _run(cfg, x, wg, we), run_oracle(cfg, x, wg, we))


def test_parity_with_bias_and_gelu():
    cfg = MoEConfig(num_experts=8, expert_top_k=2, sequence_len=256, hidden_size=256, intermediate_size=512, hidden_act=1)
    x, wg, we, bu, bd = make_inputs(cfg, seed=7, bias=True)
    _compare(cfg, _run(cfg, x, wg, we, bu, bd), run_oracle(cfg, x, wg, we, bu, bd))


def test_unscaled_weights_like_the_reference_harness():
    # torch.randn weights without scaling (reference worker.py:56-58): near-one-hot softmax, |y| ~ 1e3
    cfg = MoEConfig(num_experts=8, expert_top_k=2, sequence_len=512, hidden_size=256, intermediate_size=512)
    x, wg, we, _, _ = make_inputs(cfg, seed=8, scaled=False)
    _compare(cfg, _run(cfg, x, wg, we), run_oracle(cfg, x, wg, we))


def test_exp_underflow_corner_matches_reference_semantics():
    # Appendix A.4 on the GPU: all but one probability flush to zero; picks continue in index order
    cfg = MoEConfig(num_experts=4, expert_top_k=3, sequence_len=128, hidden_size=64, intermediate_size=64)
    x = torch.zeros(1, 128, 64)
    x[..., 0] = 1.0
    wg_eff = torch.zeros(4, 64)
    wg_eff[:, 0] = torch.tensor([100.0, -200.0, -150.0, -120.0])
    wg = wg_eff.reshape(-1).view(64, 4)  # the [H,E] tensor whose flat view is wg_eff
    g = torch.Generator().manual_seed(9)
    we = torch.randn(4, 2, 64, 64, generator=g) * 0.1
    got = _run(cfg, x.bfloat16(), wg.bfloat16(), we.bfloat16())
    assert (got["topk_idx"] == np.array([0, 1, 2])).all()
    _compare(cfg, got, run_oracle(cfg, x.bfloat16(), wg.bfloat16(), we.bfloat16()))


def test_all_tokens_to_one_expert_capacity_drop():
    cfg = MoEConfig(num_experts=4, expert_top_k=1, sequence_len=256, hidden_size=64, intermediate_size=128)
    x = torch.ones(1, 256, 64) * 0.5
    wg_eff = torch.zeros(4, 64)
    wg_eff[2] = 1.0
    wg = wg_eff.reshape(-1).view(64, 4)
    g = torch.Generator().manual_seed(10)
    we = (torch.randn(4, 2, 128, 64, generator=g) * 0.2).bfloat16()
    got = _run(cfg, x.bfloat16(), wg.bfloat16(), we)
    assert got["counts"].tolist() == [0, 0, 256, 0]
    assert (got["slot"][:, 0] == np.arange(256)).all()
    out = mo.bits_to_f32(got["out"])
    assert (out[cfg.EC:] == 0).all() and (out[:cfg.EC] != 0).any()
    _compare(cfg, got, run_oracle(cfg, x.bfloat16(), wg.bfloat16(), we))


def test_full_size_config_B_parity_and_properties():
    """BASELINE.json configs[1] (8 experts, top-2, seq 4096, d_model 1024, ffn 4096) at full size."""
    cfg = BASELINE_CONFIGS["B"]
    x, wg, we, _, _ = make_inputs(cfg, seed=1)
    ctx = _ctx(cfg)
    dev = ctx.device
    xd, wgd, wed = x.to(dev), wg.to(dev), we.to(dev)
    out1 = ctx.forward(xd, wgd, wed).clone()
    ctx.synchronize()
    topk = ctx.read("topk_idx")
    slot = ctx.read("slot")
    counts = ctx.read("counts")
    # property: idempotence / determinism across launches (epoch-tagged flags, no stale state)
    for _ in range(3):
        out2 = ctx.forward(xd, wgd, wed)
    ctx.synchronize()
    assert torch.equal(out1, out2)
    # property: capacity accounting -- slots of each expert are a permutation of 0..count-1, kept = min(count, EC)
    for e in range(cfg.E):
        s = np.sort(slot[topk == e])
        assert (s == np.arange(len(s))).all() and len(s) == counts[e]
    assert counts.sum() == cfg.S * cfg.k
    recv = ctx.read("recv_cnt")
    assert (recv == np.minimum(counts, cfg.EC)).all()
    # property: dispatch is an exact row copy (checksum of checksums over the received rows)
    rx = ctx.read("recv_x").astype(np.uint64)
    xb = mo.to_bits(x.reshape(cfg.S, cfg.H)).astype(np.uint64)
    row_sum = xb.sum(axis=1)
    kept = slot < cfg.EC
    want = sum(int(row_sum[t]) for t, j in zip(*np.nonzero(kept)))
    have = sum(int(rx[e, :recv[e]].sum()) for e in range(cfg.E))
    assert want == have
    # property: a token routed twice to dropped slots yields an all-zero row, never garbage
    both_dropped = ~kept.any(axis=1)
    o = mo.to_bits(out1.cpu().reshape(cfg.S, cfg.H))
    assert (o[both_dropped] == 0).all()
    # full-size oracle comparison (~1.5 s of CPU)
    ref = run_oracle(cfg, x, wg, we)
    mism = check_topk(topk, ref)
    check_output(o, ref.out, rows_ok=~mism)
    # permutation property: permuting tokens permutes routing decisions and (un-dropped) outputs
    perm = torch.randperm(cfg.S, generator=torch.Generator().manual_seed(3))
    xp = x.reshape(cfg.S, cfg.H)[perm].reshape(x.shape).contiguous()
    ctx.forward(xp.to(dev), wgd, wed)
    ctx.synchronize()
    assert (ctx.read("topk_idx") == topk[perm.numpy()]).all()
    ctx.close()


def test_host_buffer_entry_point_equals_device_path():
    cfg = CASES["small_drop"]
    x, wg, we, _, _ = make_inputs(cfg, seed=21)
    ctx = _ctx(cfg)
    dev = ctx.device
    out_dev = ctx.forward(x.to(dev), wg.to(dev), we.to(dev))
    ctx.synchronize()
    out_host = ctx.forward_host(x.pin_memory(), wg.to(dev), we.to(dev))
    assert torch.equal(out_host, out_dev.cpu())
    ctx.close()


@pytest.mark.parametrize("name", ["small_drop", "ragged_dims", "E64_k4", "E128_k2", "E160_k2"])
def test_router_cuda_core_path(monkeypatch, name):
    """The router's logits come from wgmma by default (17 <= E <= 256); FM_TC_GATE=0 selects the register-blocked
    CUDA-core GEMV (the only path for E > 256), which must stay parity-green too."""
    monkeypatch.setenv("FM_TC_GATE", "0")
    cfg = CASES[name]
    x, wg, we, _, _ = make_inputs(cfg, seed=400 + len(name))
    _compare(cfg, _run(cfg, x, wg, we), run_oracle(cfg, x, wg, we))


@pytest.mark.parametrize("name", ["tiny", "small_drop", "ragged_dims", "configA_top1", "multi_seq"])
def test_router_tensor_core_path_small_expert_counts(monkeypatch, name):
    """FM_TC_GATE=1 forces the wgmma router where the default (E <= 16) is the CUDA-core GEMV: padded expert columns
    (E = 2, 4, 6, 8 -> 64), chunks of fewer than 32 tokens."""
    monkeypatch.setenv("FM_TC_GATE", "1")
    cfg = CASES[name]
    x, wg, we, _, _ = make_inputs(cfg, seed=500 + len(name))
    _compare(cfg, _run(cfg, x, wg, we), run_oracle(cfg, x, wg, we))


def test_router_many_experts_general_path():
    """E = 320 > 256: beyond one tensor-core accumulator, the CUDA-core router is used automatically."""
    cfg = MoEConfig(num_experts=320, expert_top_k=2, sequence_len=1024, hidden_size=128, intermediate_size=128)
    x, wg, we, _, _ = make_inputs(cfg, seed=71)
    _compare(cfg, _run(cfg, x, wg, we), run_oracle(cfg, x, wg, we))


@pytest.mark.parametrize("E,k,tc_gate", [(4, 3, None), (6, 3, None), (8, 2, None), (16, 2, None), (64, 4, None),
                                         (8, 2, 1)])
def test_router_nan_token(monkeypatch, E, k, tc_gate):
    """A NaN in a token's x row makes all its logits NaN: no expert compares greater than -inf in any top-k round, and
    the token picks expert 0 every time, as the oracle does.  Every index stays in range (E = 6: idle lanes in the
    lane groups), and the other tokens route, count and combine as usual."""
    if tc_gate is not None:
        monkeypatch.setenv("FM_TC_GATE", str(tc_gate))
    cfg = MoEConfig(num_experts=E, expert_top_k=k, sequence_len=512, hidden_size=256, intermediate_size=512)
    x, wg, we, _, _ = make_inputs(cfg, seed=600 + E + k)
    rows = x.view(cfg.S, cfg.H)
    nan_tokens = [1, 2, 301]
    rows[1] = float("nan")          # a whole row
    rows[2, 17] = float("nan")      # one element, in the neighbour of a NaN row
    rows[301, 0] = float("nan")
    got = _run(cfg, x, wg, we)
    ref = run_oracle(cfg, x, wg, we)
    topk = got["topk_idx"]
    assert ((topk >= 0) & (topk < E)).all()
    assert (topk[nan_tokens] == 0).all() and (ref.topk_idx[nan_tokens] == 0).all()
    slot, counts, recv_cnt, _ = slots_from_topk(topk, E, cfg.EC)
    assert (got["slot"] == slot).all()
    assert (got["counts"] == counts).all()
    assert (got["recv_cnt"] == recv_cnt).all()
    rows_ok = ~check_topk(topk, ref)
    rows_ok[nan_tokens] = False
    check_output(got["out"], ref.out, rows_ok=rows_ok)


@pytest.mark.parametrize("fused", [1, 0])
def test_relaunch_with_changing_inputs_every_launch_checked(monkeypatch, fused):
    """Back-to-back launches on ONE context with different activations (routing, per-expert counts and drops change,
    including counts that shrink so the previous launch's rows lie beyond the new count): every launch's output is
    compared with the oracle, so a read of stale recv_x / hidden / recv_meta / accumulator state cannot hide."""
    monkeypatch.setenv("FM_FUSED_COMBINE", str(fused))
    cfg = MoEConfig(num_experts=8, expert_top_k=2, sequence_len=1024, hidden_size=256, intermediate_size=512, drop_tokens=0)
    g = torch.Generator().manual_seed(77)
    xs = [torch.randn(1, cfg.S, cfg.H, generator=g).bfloat16() for _ in range(3)]
    # half of the tokens near-identical (token 0 + small noise): two experts get most rows
    xs[1][:, : cfg.S // 2] = (xs[1][:, :1].float() + torch.randn(1, cfg.S // 2, cfg.H, generator=g) * 0.02).bfloat16()
    _, wg, we, _, _ = make_inputs(cfg, seed=78)
    refs = [run_oracle(cfg, x, wg, we) for x in xs]
    ctx = _ctx(cfg)
    dev = ctx.device
    wgd, wed = wg.to(dev), we.to(dev)
    for it in range(9):
        i = (it * 2) % 3
        out = ctx.forward(xs[i].to(dev), wgd, wed)
        ctx.synchronize()
        mism = check_topk(ctx.read("topk_idx"), refs[i])
        check_output(mo.to_bits(out.cpu().reshape(cfg.S, cfg.H)), refs[i].out, rows_ok=~mism, what=f"launch {it}")
        if not mism.any():
            assert (ctx.read("counts") == refs[i].counts).all()
    ctx.close()


def test_pipelined_host_entry_point_matches_device_path():
    """fm_host_submit / fm_host_wait: three steps in flight with different inputs; every result equals the device path."""
    cfg = CASES["small_drop"]
    g = torch.Generator().manual_seed(31)
    xs = [torch.randn(1, cfg.S, cfg.H, generator=g).bfloat16() for _ in range(5)]
    _, wg, we, _, _ = make_inputs(cfg, seed=32)
    ctx = _ctx(cfg)
    dev = ctx.device
    wgd, wed = wg.to(dev), we.to(dev)
    want = []
    for x in xs:
        want.append(ctx.forward(x.to(dev), wgd, wed).cpu())
    ctx.synchronize()
    pins = [x.pin_memory() for x in xs]
    outs = [torch.empty_like(x).pin_memory() for x in xs]
    tickets = []
    for i in range(5):
        if len(tickets) == 3:
            ctx.wait_host(tickets.pop(0))
        tickets.append(ctx.submit_host(pins[i], wgd, wed, outs[i]))
    with pytest.raises(RuntimeError):  # tickets complete in submission order
        ctx.wait_host(tickets[-1])
    for t in tickets:
        ctx.wait_host(t)
    for i in range(5):
        assert torch.equal(outs[i], want[i]), f"step {i}"
    ctx.close()


def test_misaligned_tensor_is_rejected():
    cfg = CASES["tiny"]
    x, wg, we, _, _ = make_inputs(cfg, seed=33)
    ctx = _ctx(cfg)
    dev = ctx.device
    buf = torch.empty(x.numel() + 8, dtype=torch.bfloat16, device=dev)
    x_off = buf[1: 1 + x.numel()].view(x.shape)   # contiguous, but starts 2 bytes into the allocation
    x_off.copy_(x)
    with pytest.raises(RuntimeError, match="16-byte"):
        ctx.forward(x_off, wg.to(dev), we.to(dev))
    ctx.close()


@pytest.mark.parametrize("name", ["small_drop", "E32_k2", "E128_k2"])
def test_training_mode_aux_loss_matches_oracle(name):
    """is_training = 1 (SURVEY.md section 8f rank 3): gML / gMeC / loss accumulated in the router, read back through
    FM_BUF_AUX_LOSS; two launches with different inputs on one context (the buffers are cleared per launch)."""
    cfg = CASES[name].replace(is_training=1)
    ctx = _ctx(cfg)
    dev = ctx.device
    for seed in (51, 52):
        x, wg, we, _, _ = make_inputs(cfg, seed=seed)
        out = ctx.forward(x.to(dev), wg.to(dev), we.to(dev))
        ctx.synchronize()
        aux = ctx.read("aux_loss")
        gml, gmec, loss = mo.aux_loss(mo.to_bits(x.reshape(cfg.S, cfg.H)),
                                      mo.gate_weights_effective(mo.to_bits(wg), cfg.E, cfg.H), k=cfg.k, EC=cfg.EC)
        ref = run_oracle(cfg, x, wg, we)
        mism = check_topk(ctx.read("topk_idx"), ref)
        np.testing.assert_allclose(aux[:cfg.E], gml, rtol=2e-5, atol=1e-7)
        if not mism.any():
            np.testing.assert_allclose(aux[cfg.E:2 * cfg.E], gmec, rtol=1e-6)
            np.testing.assert_allclose(aux[2 * cfg.E], loss, rtol=2e-5)
        check_output(mo.to_bits(out.cpu().reshape(cfg.S, cfg.H)), ref.out, rows_ok=~mism)   # the forward itself is unchanged
    ctx.close()


def test_dense_single_expert_general_path_still_works(monkeypatch):
    """E = 1 takes the dense fast path by default (no router GEMV, no dispatch copy; test E1_dense above);
    FM_DENSE_E1=0 sends it through the general router / dispatch path, which must agree too."""
    monkeypatch.setenv("FM_DENSE_E1", "0")
    cfg = CASES["E1_dense"]
    x, wg, we, _, _ = make_inputs(cfg, seed=61)
    _compare(cfg, _run(cfg, x, wg, we), run_oracle(cfg, x, wg, we))


def test_dense_single_expert_with_bias_gelu_and_capacity_factor():
    cfg = MoEConfig(num_experts=1, expert_top_k=1, sequence_len=384, hidden_size=128, intermediate_size=256, hidden_act=1,
                    capacity_factor=2)
    x, wg, we, bu, bd = make_inputs(cfg, seed=62, bias=True)
    _compare(cfg, _run(cfg, x, wg, we, bu, bd), run_oracle(cfg, x, wg, we, bu, bd))


def test_reference_style_argument_checks_raise_runtime_error():
    cfg = CASES["tiny"]
    x, wg, we, _, _ = make_inputs(cfg, seed=22)
    ctx = _ctx(cfg)
    dev = ctx.device
    with pytest.raises(RuntimeError, match="CUDA"):
        ctx.forward(x, wg.to(dev), we.to(dev))
    with pytest.raises(RuntimeError, match="compiled S"):
        ctx.forward(x[:, :64].contiguous().to(dev), wg.to(dev), we.to(dev))
    with pytest.raises(RuntimeError, match="Gate weights"):
        ctx.forward(x.to(dev), wg.t().contiguous().to(dev), we.to(dev))
    with pytest.raises(RuntimeError, match="Expert count"):
        ctx.forward(x.to(dev), wg.to(dev), we[:2].contiguous().to(dev))
    with pytest.raises(RuntimeError, match="bfloat16"):
        ctx.forward(x.float().to(dev), wg.to(dev), we.to(dev))
    with pytest.raises(RuntimeError, match="contiguous"):
        ctx.forward(x.to(dev).transpose(0, 1).expand(128, 1, 64).transpose(0, 1)[:, :, ::1].as_strided((1, 128, 64), (1, 64, 1)),
                    wg.to(dev), we.to(dev)) if False else ctx.forward(x.to(dev), wg.to(dev), we.to(dev).transpose(2, 3))
    ctx.close()


def test_module_level_C_api_single_process():
    """flashmoe._C (the COMPILED pybind11 extension, csrc/python_bindings.cu) initialize / moe_forward / finalize on the
    compiled configuration (config B), output checked against the oracle."""
    import flashmoe
    from flashmoe import _C

    assert _C.__file__.endswith(".so")
    _C.initialize()
    try:
        cc = flashmoe.get_compiled_config()
        assert cc["S"] == 4096 and cc["Element_size"] == 2 and _C.get_bookkeeping() == {"nLx": 8}
        assert _C.get_num_local_experts() == 8
        cfg = BASELINE_CONFIGS["B"]
        x, wg, we, _, _ = make_inputs(cfg, seed=23)
        out = _C.moe_forward(input=x.cuda(), gate_weights=wg.cuda(), expert_weights=we.cuda())
        assert out.shape == x.shape and out.dtype == torch.bfloat16 and torch.isfinite(out.float()).all()
        ref = run_oracle(cfg, x, wg, we)
        # the extension does not expose the routing tables: compare all rows, allowing for the (rare) ambiguous tokens
        check_output(mo.to_bits(out.cpu().reshape(cfg.S, cfg.H)), ref.out, rows_ok=~ref.ambiguous)
        with pytest.raises(RuntimeError, match="compiled S"):
            _C.moe_forward(x[:, :64].contiguous().cuda(), wg.cuda(), we.cuda())
        with pytest.raises(RuntimeError):
            _C.initialize()
    finally:
        _C.finalize()
