"""The GEMM0 epilogue hands h to TMA tensor stores: the kernel's SASS contains UTMASTG.  CPU only."""
import os
import subprocess

import pytest

from flashmoe_b200 import _lib
from tests.test_abi import lib  # noqa: F401  (fixture: the in-tree library, built if needed)


def test_sass_contains_tma_tensor_store(lib):  # noqa: F811
    cuobjdump = "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", str(_lib.LIB_PATH)], capture_output=True, text=True).stdout
    assert "UTMASTG" in sass, "UTMASTG (TMA tensor store) missing from SASS"
