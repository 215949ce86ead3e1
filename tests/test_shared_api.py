"""The shared-expert surface without a GPU: the header declares fm_shared_reserve / fm_moe_forward_shared and the
binding exports them; fm_shared_expert_t's layout matches the header; both functions reject a null context; the Python
argument checks reject every bad shared-expert argument.  CPU only."""
import ctypes
import os
import re

import pytest
import torch

from flashmoe_b200 import _build, _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = open(os.path.join(ROOT, "include", "flashmoe_b200.h")).read()


@pytest.fixture(scope="module")
def lib():
    try:
        _build.find_nvcc()
        _build.build()
    except RuntimeError:
        if not _lib.LIB_PATH.exists():
            pytest.skip("nvcc not available and no prebuilt library")
    return _lib.load()


def test_header_declares_and_binding_exports():
    for name in ("fm_shared_reserve", "fm_moe_forward_shared"):
        assert re.search(rf"FM_API\s+int\s+{name}\s*\(", HEADER), name
        assert name in _lib.EXPORTED_SYMBOLS
    assert re.search(r"FM_BUF_SHARED_Y\s*=\s*12\b", HEADER) and _lib.BUF_SHARED_Y == 12
    assert re.search(r"FM_BUF_SHARED_HIDDEN\s*=\s*13\b", HEADER) and _lib.BUF_SHARED_HIDDEN == 13


def test_struct_matches_header():
    body = HEADER.split("typedef struct fm_shared_expert {")[1].split("} fm_shared_expert_t;")[0]
    fields = re.findall(r"^\s*(const void\*|int32_t)\s+(\w+);", body, flags=re.M)
    assert [n for _, n in fields] == [n for n, _ in _lib.FmSharedExpert._fields_] == ["w", "bias_up", "bias_down", "inter"]
    ctype = {"const void*": ctypes.c_void_p, "int32_t": ctypes.c_int32}
    assert [ctype[t] for t, _ in fields] == [t for _, t in _lib.FmSharedExpert._fields_]
    # C layout on LP64: three pointers, then the int32, padded to pointer alignment
    assert [getattr(_lib.FmSharedExpert, n).offset for _, n in fields] == [0, 8, 16, 24]
    assert ctypes.sizeof(_lib.FmSharedExpert) == 32


def test_null_context_rejected(lib):
    assert lib.fm_shared_reserve(None, 64) == -1
    assert b"null context" in lib.fm_last_error()
    assert lib.fm_moe_forward_shared(None, None, 0, None, None, None, None, None, None, None, None, None, None, None,
                                     None) == -1
    assert b"null context" in lib.fm_last_error()


def _se(w, bu=None, bd=None):
    from flashmoe_b200.runtime import SharedExpert

    return SharedExpert(w, bu, bd)


CPU = torch.device("cpu")
H = 128


def _w(ps=128, dtype=torch.bfloat16):
    return torch.zeros(2, ps, H, dtype=dtype)


@pytest.mark.parametrize("se,reserved,pattern", [
    (lambda: _w(), 256, r"must be a SharedExpert"),
    (lambda: _se(_w()), None, r"create it with shared_inter"),
    (lambda: _se(torch.zeros(128, H, dtype=torch.bfloat16)), 256, r"must be a 3-D tensor"),
    (lambda: _se(_w(dtype=torch.float32)), 256, r"must be torch.bfloat16"),
    (lambda: _se(torch.zeros(3, 128, H, dtype=torch.bfloat16)), 256, r"must be \[up/down=2, Ps=128, H=128\]"),
    (lambda: _se(torch.zeros(2, 128, 64, dtype=torch.bfloat16)), 256, r"must be \[up/down=2, Ps=128, H=128\]"),
    (lambda: _se(_w().transpose(1, 2).contiguous().transpose(1, 2)), 256, r"must be contiguous"),
    (lambda: _se(_w(96)), 256, r"Ps = 96 must be a positive multiple of 64"),
    (lambda: _se(_w(320)), 256, r"Ps = 320 is above the context's shared_inter = 256"),
    (lambda: _se(_w(), torch.zeros(64, dtype=torch.bfloat16)), 256, r"shared_expert.bias_up must be \[Ps=128\]"),
    (lambda: _se(_w(), None, torch.zeros(H, dtype=torch.float32)), 256, r"shared_expert.bias_down must be torch.bfloat16"),
    (lambda: _se(_w(), None, torch.zeros(H + 1, dtype=torch.bfloat16)[1:]), 256, r"16-byte boundary"),
], ids=["not_shared_expert", "not_reserved", "w_2d", "w_dtype", "w_shape0", "w_shape_H", "w_strided", "ps_96",
        "ps_above_reserved", "bias_up_shape", "bias_down_dtype", "bias_down_misaligned"])
def test_python_checks_reject(se, reserved, pattern):
    from flashmoe_b200.runtime import shared_expert_struct

    with pytest.raises((RuntimeError, TypeError), match=pattern):
        shared_expert_struct(se(), CPU, H, reserved)


def test_python_checks_accept_and_fill_the_struct():
    from flashmoe_b200.runtime import shared_expert_struct

    w, bu = _w(192), torch.zeros(192, dtype=torch.bfloat16)
    st = shared_expert_struct(_se(w, bu), CPU, H, 256)
    assert (st.w, st.bias_up, st.bias_down, st.inter) == (w.data_ptr(), bu.data_ptr(), None, 192)
