"""The C-ABI shared library loads and exports every symbol include/flashmoe_b200.h declares; the host-side mirror of
the reference API is importable; nothing computes on the CPU (no GPU => loud failure).  CPU only."""
import ctypes
import os
import re
import subprocess
import sys

import pytest

from flashmoe_b200 import _build, _lib, config as C

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "flashmoe_b200.h")


@pytest.fixture(scope="module")
def lib():
    try:
        _build.find_nvcc()
        _build.build()  # no-op when the in-tree .so matches sources + config
    except RuntimeError:
        if not _lib.LIB_PATH.exists():
            pytest.skip("nvcc not available and no prebuilt library")
    return _lib.load()


def declared_symbols():
    text = open(HEADER).read()
    return sorted(set(re.findall(r"FM_API\s+[\w\s\*]+?\b(fm_\w+)\s*\(", text)))


def test_header_declares_the_expected_entry_points():
    syms = declared_symbols()
    for must in ("fm_create", "fm_destroy", "fm_moe_forward", "fm_moe_forward_host", "fm_compiled_config",
                 "fm_num_local_experts", "fm_symm_export", "fm_symm_attach_ipc", "fm_last_error"):
        assert must in syms
    assert sorted(_lib.EXPORTED_SYMBOLS) == syms, "python binding table out of sync with the header"


def test_library_exports_every_declared_symbol(lib):
    for name in declared_symbols():
        assert hasattr(lib, name), f"{name} not exported by {_lib.LIB_PATH}"


def test_compiled_config_is_the_json(lib):
    assert _lib.compiled_config().raw() == C.load_config().raw()


def test_struct_layouts_match_header():
    assert ctypes.sizeof(_lib.FmConfig) == 15 * 4 and ctypes.sizeof(_lib.FmDims) == 16 * 4
    text = open(HEADER).read()
    cfg_fields = re.findall(r"int32_t\s+(\w+);", text.split("typedef struct fm_config")[1].split("} fm_config_t")[0])
    assert cfg_fields == [f for f, _ in _lib.FmConfig._fields_]


def test_sass_contains_hopper_tensor_and_tma_instructions(lib):
    cuobjdump = "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", str(_lib.LIB_PATH)], capture_output=True, text=True).stdout
    assert "sm_90a" in sass
    for mnemonic in ("HGMMA", "UTMALDG"):  # wgmma, TMA tensor load
        assert mnemonic in sass, f"{mnemonic} missing from SASS"
    assert "HMMA.16816" not in sass  # no legacy mma.sync path


def test_create_without_gpu_fails_loudly_with_message(lib):
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    ctx = ctypes.c_void_p()
    rc = lib.fm_create(None, 0, 1, 0, ctypes.byref(ctx))
    assert rc < 0 and not ctx.value
    assert len(lib.fm_last_error()) > 0


def test_invalid_arguments_are_reported_not_fatal(lib):
    bad = _lib.FmConfig.from_config(C.load_config().replace(hidden_size=1000))
    ctx = ctypes.c_void_p()
    assert lib.fm_create(ctypes.byref(bad), 0, 1, 0, ctypes.byref(ctx)) == -1  # FM_EINVAL before touching CUDA
    assert b"hidden_size" in lib.fm_last_error()
    assert lib.fm_create(None, 3, 2, 0, ctypes.byref(ctx)) == -1
    assert lib.fm_moe_forward(None, None, None, None, None, None, None, None) == -1
    assert lib.fm_destroy(None) == 0


def test_reference_api_surface_is_mirrored():
    import flashmoe
    import flashmoe_b200
    import inspect

    assert flashmoe.__all__ == ["run_moe", "get_compiled_config"] == flashmoe_b200.__all__
    sig = inspect.signature(flashmoe.run_moe)
    assert list(sig.parameters) == ["n_processes", "processes_per_node", "hostfile", "config_path"]
    assert sig.parameters["n_processes"].default == 1 and sig.parameters["hostfile"].default is None
    from flashmoe import _C

    for fn in ("moe_forward", "initialize", "finalize", "get_compiled_config", "get_bookkeeping", "get_num_local_experts"):
        assert callable(getattr(_C, fn))
    # compiled extension: the keyword names are in the pybind11 docstring signature; the ctypes fallback has a Python signature
    from flashmoe_b200 import _C as _C_ctypes

    assert list(inspect.signature(_C_ctypes.moe_forward).parameters) == ["input", "gate_weights", "expert_weights"]
    assert "moe_forward(input: object, gate_weights: object, expert_weights: object)" in _C.moe_forward.__doc__
    assert set(_C.get_compiled_config()) == {"S", "H", "E", "P", "PX", "Element_size"}
    with pytest.raises(RuntimeError, match="initialize"):
        _C.moe_forward(None, None, None)


def test_launcher_command_and_errors(tmp_path):
    from flashmoe_b200 import launcher

    cmd = launcher.build_command(str(C.DEFAULT_CONFIG_PATH), 1, 1)
    assert cmd[0] == sys.executable and cmd[-1].endswith("flashmoe_config.json") and "worker.py" in cmd[-2]
    cmd = launcher.build_command(str(C.DEFAULT_CONFIG_PATH), 4, 4)
    assert "--nproc-per-node=4" in cmd and "127.0.0.1" in cmd
    with pytest.raises(FileNotFoundError):
        launcher.build_command(str(tmp_path / "kleos_config.json"), 1, 1)
    with pytest.raises(NotImplementedError):
        launcher.build_command(str(C.DEFAULT_CONFIG_PATH), 16, 8, hostfile="hosts.txt")


def test_product_does_not_import_the_oracle():
    for root, _, files in os.walk(os.path.join(ROOT, "flashmoe_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                text = open(os.path.join(root, f)).read()
                assert "import oracle" not in text and "from oracle" not in text and "moe_oracle" not in text, f


def test_flashmoe_C_is_the_compiled_extension_with_the_reference_signatures():
    """`flashmoe._C` is built from csrc/python_bindings.cu (reference csrc/python_bindings.cu:194-217): six functions,
    the reference's keyword names, RuntimeError (not exit) when used before initialize()."""
    from flashmoe_b200 import _build

    _build.build_bindings()
    import importlib

    import flashmoe

    ext = importlib.import_module("flashmoe._C")
    assert ext.__file__.endswith(".so")
    for fn in ("moe_forward", "initialize", "finalize", "get_compiled_config", "get_bookkeeping", "get_num_local_experts"):
        assert callable(getattr(ext, fn))
    doc = ext.moe_forward.__doc__
    assert "input" in doc and "gate_weights" in doc and "expert_weights" in doc
    cc = ext.get_compiled_config()
    assert cc == C.load_config().compiled_dict() and set(cc) == {"S", "H", "E", "P", "PX", "Element_size"}
    with pytest.raises(RuntimeError, match="initialize"):
        ext.moe_forward(input=None, gate_weights=None, expert_weights=None)
    with pytest.raises(RuntimeError):
        ext.get_num_local_experts()
    assert flashmoe.get_compiled_config() == cc
