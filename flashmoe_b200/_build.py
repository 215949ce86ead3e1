"""In-tree build of the native library: csrc/flashmoe_config.json -> -DFM_CFG_* -> nvcc (sm_90a) ->
flashmoe_b200/libflashmoe_b200.so.

Replaces the reference's setup.py / CMake JSON->macro plumbing (reference setup.py:227-292, csrc/CMakeLists.txt:114-237):
no network downloads, reads the file the reference's CMake reads (csrc/flashmoe_config.json, not the dangling
kleos_config.json), emits sm_90a only.  The .so is a build product (git-ignored); build() writes it into the package.
"""
from __future__ import annotations

import hashlib
import json
import os
import shutil
import subprocess
import sys
from pathlib import Path
from typing import List, Optional

from . import config as _config

PKG_DIR = Path(__file__).resolve().parent
REPO_ROOT = PKG_DIR.parent
CSRC = PKG_DIR / "csrc"
LIB_PATH = PKG_DIR / "libflashmoe_b200.so"
STAMP_PATH = PKG_DIR / ".build_stamp.json"
SOURCES = [CSRC / "flashmoe_b200.cu"]
HEADERS = [CSRC / "fm_kernel.cuh", CSRC / "fm_ptx.cuh", REPO_ROOT / "include" / "flashmoe_b200.h"]

# the compiled `flashmoe._C` extension (csrc/python_bindings.cu: pybind11 over the C-ABI; no device code, no torch headers)
BINDINGS_SRC = REPO_ROOT / "csrc" / "python_bindings.cu"


def ext_path() -> Path:
    import sysconfig

    return REPO_ROOT / "flashmoe" / ("_C" + sysconfig.get_config_var("EXT_SUFFIX"))


NVCC_FLAGS = [
    "-std=c++17", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
    "--compiler-options", "-fPIC,-fvisibility=hidden", "-shared",
]


def find_nvcc() -> str:
    for cand in (os.environ.get("CUDA_HOME", "/usr/local/cuda") + "/bin/nvcc", shutil.which("nvcc")):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found (set CUDA_HOME)")


def config_macros(cfg: _config.MoEConfig) -> List[str]:
    return [f"-DFM_CFG_{k.upper()}={v}" for k, v in cfg.raw().items()]


def _fingerprint(cfg: _config.MoEConfig) -> str:
    h = hashlib.sha256()
    for f in SOURCES + HEADERS:
        h.update(f.read_bytes())
    h.update(json.dumps(cfg.raw(), sort_keys=True).encode())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(config_path: Optional[os.PathLike] = None, force: bool = False, verbose: bool = False) -> Path:
    """Compile the library for sm_90a with the given (default: csrc/flashmoe_config.json) config baked in."""
    cfg = _config.load_config(config_path)
    cfg.check_hot_path()
    fp = _fingerprint(cfg)
    if not force and LIB_PATH.exists() and STAMP_PATH.exists():
        try:
            if json.loads(STAMP_PATH.read_text()).get("fingerprint") == fp:
                return LIB_PATH
        except (OSError, ValueError):
            pass
    cmd = [find_nvcc(), *NVCC_FLAGS, *config_macros(cfg), f"-I{REPO_ROOT / 'include'}", "-o", str(LIB_PATH),
           *[str(s) for s in SOURCES]]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
        print(" ".join(cmd), file=sys.stderr)
    # the image exports CC/CXX=/opt/gcc/...; nvcc must use the system host compiler
    ccbin = "/usr/bin/g++" if Path("/usr/bin/g++").exists() else None
    if ccbin:
        cmd[1:1] = ["-ccbin", ccbin]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"nvcc failed ({res.returncode}):\n{res.stdout}\n{res.stderr}")
    if verbose:
        print(res.stderr, file=sys.stderr)
    STAMP_PATH.write_text(json.dumps({"fingerprint": fp, "config": cfg.raw()}))
    return LIB_PATH


def build_bindings(force: bool = False, verbose: bool = False) -> Path:
    """Compile csrc/python_bindings.cu into flashmoe/_C<ext suffix>, linked against the in-tree libflashmoe_b200.so
    (found at run time through an $ORIGIN-relative rpath).  Needs pybind11 (present in this image)."""
    import sysconfig

    import pybind11

    out = ext_path()
    stamp = out.with_suffix(".stamp")
    h = hashlib.sha256(BINDINGS_SRC.read_bytes() + (REPO_ROOT / "include" / "flashmoe_b200.h").read_bytes()).hexdigest()
    if not force and out.exists() and stamp.exists() and stamp.read_text() == h and LIB_PATH.exists():
        return out
    if not LIB_PATH.exists():
        raise RuntimeError("build libflashmoe_b200.so first")
    cmd = [find_nvcc(), "-std=c++17", "-O2", "-x", "cu", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
           "--compiler-options", "-fPIC,-fvisibility=hidden", "-shared",
           f"-I{pybind11.get_include()}", f"-I{sysconfig.get_paths()['include']}", f"-I{REPO_ROOT / 'include'}",
           "-o", str(out), str(BINDINGS_SRC), f"-L{PKG_DIR}", "-lflashmoe_b200",
           "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN/../flashmoe_b200"]
    if Path("/usr/bin/g++").exists():
        cmd[1:1] = ["-ccbin", "/usr/bin/g++"]
    if verbose:
        print(" ".join(cmd), file=sys.stderr)
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"nvcc failed on python_bindings.cu ({res.returncode}):\n{res.stdout}\n{res.stderr}")
    stamp.write_text(h)
    return out


def lib_is_current(config_path: Optional[os.PathLike] = None) -> bool:
    try:
        cfg = _config.load_config(config_path)
        return LIB_PATH.exists() and json.loads(STAMP_PATH.read_text()).get("fingerprint") == _fingerprint(cfg)
    except (OSError, ValueError):
        return False


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
    print(build_bindings(force="--force" in sys.argv, verbose=True))
