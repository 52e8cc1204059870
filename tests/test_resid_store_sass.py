"""CPU: the residual + store GEMM (resid_store_gemm<BN, BF16>, the attention cache's store step) read from the built
library's SASS.  Like every gemm_kernel instance (tests/test_gemm_sass.py, tests/test_gemm_epilogue_sass.py) it keeps its
k-loop pipelined (`WARPGROUP.DEPBAR.LE gsb0, 0x1`), hands registers to its consumers (`USETMAXREG`) and keeps them out of
local memory.  Its two outputs leave by TMA: the residual by `cp.reduce.async.bulk.tensor .add` (`UTMAREDG.2D.ADD`), the
16-bit acc + bias by `cp.async.bulk.tensor` (`UTMASTG.2D`).  It runs whole-K tiles only, so it has no stream-K flag and
no global store at all."""
import os
import re
import shutil
import subprocess

import pytest

from latte_b200 import _lib


@pytest.fixture(scope="module")
def store_functions():
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    _lib.load()
    sass = subprocess.run([cuobjdump, "-sass", _lib.lib_path()], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for chunk in sass.split("Function : ")[1:]:
        name, body = chunk.split("\n", 1)
        if "resid_store_gemm" in name:
            m = re.search(r"resid_store_gemmILi(\d+)ELb([01])EE", name)
            assert m, f"unexpected resid_store_gemm signature: {name}"
            funcs[tuple(int(g) for g in m.groups())] = body
    return funcs


def test_instances(store_functions):
    assert sorted(store_functions) == [(bn, bf16) for bn in (128, 192, 256) for bf16 in (0, 1)]


def test_both_outputs_leave_by_tma(store_functions):
    for k, body in store_functions.items():
        assert re.search(r"\bUTMAREDG\.2D\.ADD\b", body), f"{k}: no TMA reduce-add"
        assert re.search(r"\bUTMASTG\.2D\b", body), f"{k}: no TMA store"
        assert not re.search(r"\bSTG(?:\.[\w]+)*", body), f"{k}: per-thread global store"


def test_pipeline_and_registers(store_functions):
    for k, body in store_functions.items():
        assert re.search(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x1\b", body), f"{k}: no wgmma wait<1>"
        assert "USETMAXREG" in body, f"{k}: no setmaxnreg"
        assert not re.search(r"HGMMA\.\S+ RZ, gdesc\[URZ\]", body), f"{k}: injected empty wgmma group"
        assert not re.search(r"\b(LDL|STL)\b", body), f"{k}: local-memory traffic"
