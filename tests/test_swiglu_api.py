"""The SwiGLU surface (hidden_act = 2) without a GPU: the schema, MoEConfig and the C-ABI's validate_config accept 2 and
reject 3; the Python argument checks take [nLx, 3, P, H] expert weights, [nLx, 2, P] bias_up and a [3, Ps, H] shared
expert in a SwiGLU context and reject the ReLU / GELU layout there, and the reverse; the pybind11 binding's shape check
follows the compiled configuration.  CPU only."""
import ctypes
import json
import os
import re

import pytest
import torch

from flashmoe_b200 import _build, _lib
from flashmoe_b200 import config as C

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPU = torch.device("cpu")
NLX, P, H = 2, 192, 128


@pytest.fixture(scope="module")
def lib():
    try:
        _build.find_nvcc()
        _build.build()
    except RuntimeError:
        if not _lib.LIB_PATH.exists():
            pytest.skip("nvcc not available and no prebuilt library")
    return _lib.load()


def test_schema_and_config_accept_swiglu_and_reject_3():
    schema = json.load(open(os.path.join(ROOT, "csrc", "flashmoe_config.schema.json")))
    assert schema["properties"]["hidden_act"]["enum"] == [0, 1, 2]
    raw = json.load(open(C.DEFAULT_CONFIG_PATH))
    cfg = C.from_dict({**raw, "hidden_act": C.ACT_SWIGLU})
    cfg.check_hot_path()
    assert C.ACT_SWIGLU == 2 and cfg.expert_mats == 3
    assert C.MoEConfig(hidden_act=C.ACT_RELU).expert_mats == C.MoEConfig(hidden_act=C.ACT_GELU).expert_mats == 2
    with pytest.raises(C.ConfigError):
        C.from_dict({**raw, "hidden_act": 3})


def test_header_documents_the_layout():
    header = open(os.path.join(ROOT, "include", "flashmoe_b200.h")).read()
    assert "2 swiglu" in header and "[nLx, 3, P, H]" in header and "h = silu(g)*u" in header
    assert "torch.stack([w_gate, w_up," in header


def test_validate_config(lib):
    ctx = ctypes.c_void_p()
    bad = _lib.FmConfig.from_config(C.load_config().replace(hidden_act=3))
    assert lib.fm_create(ctypes.byref(bad), 0, 1, 0, ctypes.byref(ctx)) == -1 and not ctx.value
    assert b"hidden_act must be 0 (relu), 1 (gelu) or 2 (swiglu)" in lib.fm_last_error()
    if torch.cuda.is_available():
        pytest.skip("a GPU is present: fm_create would create the context")
    good = _lib.FmConfig.from_config(C.load_config().replace(hidden_act=2))
    assert lib.fm_create(ctypes.byref(good), 0, 1, 0, ctypes.byref(ctx)) < 0   # past validation, at CUDA
    assert b"hidden_act" not in lib.fm_last_error()


def _ctx(act):
    """A MoEContext's argument checks on the CPU, without a native context."""
    from flashmoe_b200.runtime import MoEContext

    ctx = MoEContext.__new__(MoEContext)
    ctx.cfg = C.MoEConfig(hidden_act=act, hidden_size=H, intermediate_size=P, num_experts=NLX)
    ctx.dims = {"num_local_experts": NLX, "P": P, "H": H, "E": NLX, "S": 4096}
    ctx.device = CPU
    ctx.shared_inter = 256
    return ctx


def _z(*shape):
    return torch.zeros(*shape, dtype=torch.bfloat16)


@pytest.mark.parametrize("act,mats", [(0, 2), (1, 2), (2, 3)])
def test_expert_weights_layout_per_activation(act, mats):
    ctx = _ctx(act)
    ctx._validate_weights(None, _z(NLX, mats, P, H))
    if mats == 2:
        with pytest.raises(RuntimeError, match=re.escape("Expert weights must have up and down projections [nLx, 2, P, H]")):
            ctx._validate_weights(None, _z(NLX, 3, P, H))
        with pytest.raises(RuntimeError, match=re.escape(f"Expert weights must be [*, 2, P={P}, H={H}]. Got [*, 2, 64, {H}]")):
            ctx._validate_weights(None, _z(NLX, 2, 64, H))
    else:
        with pytest.raises(RuntimeError, match=re.escape("gate, up and down projections [nLx, 3, P, H]; got 2")):
            ctx._validate_weights(None, _z(NLX, 2, P, H))
        with pytest.raises(RuntimeError, match=re.escape(f"Expert weights must be [*, 3, P={P}, H={H}]")):
            ctx._validate_weights(None, _z(NLX, 3, 64, H))


def test_bias_shapes():
    relu, glu = _ctx(0), _ctx(2)
    bu, bd = _z(NLX, P), _z(NLX, H)
    assert relu._bias_ptrs(bu, bd) == (bu.data_ptr(), bd.data_ptr())
    bu2 = _z(NLX, 2, P)
    assert glu._bias_ptrs(bu2, bd) == (bu2.data_ptr(), bd.data_ptr())
    with pytest.raises(RuntimeError, match=re.escape(f"bias_up must be [nLx={NLX}, gate/up=2, P={P}]")):
        glu._bias_ptrs(bu, None)
    with pytest.raises(RuntimeError, match=re.escape(f"bias_up must be [nLx={NLX}, P={P}]")):
        relu._bias_ptrs(bu2, None)
    with pytest.raises(RuntimeError, match=re.escape(f"bias_down must be [nLx={NLX}, H={H}]")):
        glu._bias_ptrs(None, _z(NLX, 2, H))


def test_shared_expert_shapes():
    from flashmoe_b200.runtime import SharedExpert, shared_expert_struct

    w3, w2, bu2 = _z(3, 192, H), _z(2, 192, H), _z(2, 192)
    st = shared_expert_struct(SharedExpert(w3, bu2), CPU, H, 256, swiglu=True)
    assert (st.w, st.bias_up, st.inter) == (w3.data_ptr(), bu2.data_ptr(), 192)
    with pytest.raises(RuntimeError, match=re.escape("shared_expert.w must be [gate/up/down=3, Ps=192, H=128]")):
        shared_expert_struct(SharedExpert(w2), CPU, H, 256, swiglu=True)
    with pytest.raises(RuntimeError, match=re.escape("shared_expert.w must be [up/down=2, Ps=192, H=128]")):
        shared_expert_struct(SharedExpert(w3), CPU, H, 256)
    with pytest.raises(RuntimeError, match=re.escape("shared_expert.bias_up must be [gate/up=2, Ps=192]")):
        shared_expert_struct(SharedExpert(w3, _z(192)), CPU, H, 256, swiglu=True)
    with pytest.raises(RuntimeError, match=re.escape("must be a 3-D tensor [3, Ps, H]")):
        shared_expert_struct(SharedExpert(_z(192, H)), CPU, H, 256, swiglu=True)


def test_binding_shape_check_source():
    """A source check: `_C.moe_forward` runs on the compiled configuration, so its SwiGLU branch is reachable only in
    a build whose csrc/flashmoe_config.json has hidden_act = 2.  tests/test_gpu_swiglu.py calls the compiled check of
    the default (ReLU) build."""
    src = open(os.path.join(ROOT, "csrc", "python_bindings.cu")).read()
    assert "cfg.hidden_act == 2 ? 3 : 2" in src
    assert '"Expert weights must have up and down projections [nLx, 2, P, H]"' in src   # the ReLU / GELU message


def test_layer_repr_names_the_activation():
    from flashmoe_b200.layer import FlashMoELayer

    layer = FlashMoELayer.__new__(FlashMoELayer)
    torch.nn.Module.__init__(layer)
    layer.cfg = C.MoEConfig(hidden_act=2)
    layer.ctx = type("Ctx", (), {"rank": 0, "world": 1})()
    layer.shared_inter = None
    assert "act=swiglu" in layer.extra_repr()
