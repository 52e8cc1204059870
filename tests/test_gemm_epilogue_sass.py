"""CPU: the GEMM epilogues leave through TMA, read from the built library's SASS.

Every gemm_kernel instantiation stages its output tile in shared memory and one thread per warpgroup hands it to TMA:
- a 16-bit output (every epilogue but gate+residual) is written by `cp.async.bulk.tensor` stores (`UTMASTG`), never by a
  plain per-thread global store (`STG`);
- the gate+residual epilogue adds its increment into the fp32 residual stream with `cp.reduce.async.bulk.tensor .add`
  (`UTMAREDG.2D.ADD`) and never loads or stores x itself: its only `STG` is the stream-K ordering flag's 64-bit release
  store (`STG.E.64.STRONG.GPU`).
Every instantiation also keeps its accumulators in registers (no local-memory traffic)."""
import os
import re
import shutil
import subprocess

import pytest

from latte_b200 import _lib

EPI_GATE_RESIDUAL = 2


@pytest.fixture(scope="module")
def gemm_functions():
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    _lib.load()
    sass = subprocess.run([cuobjdump, "-sass", _lib.lib_path()], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for chunk in sass.split("Function : ")[1:]:
        name, body = chunk.split("\n", 1)
        if "gemm_kernel" in name:
            m = re.search(r"gemm_kernelILi(\d+)ELi(\d+)ELb([01])ELi(\d+)EE", name)
            assert m, f"unexpected gemm_kernel signature: {name}"
            funcs[tuple(int(g) for g in m.groups())] = body
    assert funcs, "no gemm_kernel in the library's SASS"
    return funcs


def _global_stores(body):
    return re.findall(r"\bSTG(?:\.[\w]+)*", body)


def test_16bit_outputs_leave_by_tma_store(gemm_functions):
    sixteen = {k: b for k, b in gemm_functions.items() if k[1] != EPI_GATE_RESIDUAL}
    # five epilogues (bias, bias+GELU, +16-bit shortcut, x16-bit factor, GELU-both) with K-major operands at BN 128 / 192 / 256,
    # plus dgrad's bias (W read [K, N]) at BN 128 / 256, each for fp16 and bf16
    assert len(sixteen) == 5 * 3 * 2 + 2 * 2
    no_tma = [k for k, b in sixteen.items() if not re.search(r"\bUTMASTG\.2D\b", b)]
    assert no_tma == [], f"no TMA store in {no_tma}"
    stg = {k: _global_stores(b) for k, b in sixteen.items() if _global_stores(b)}
    assert stg == {}, f"per-thread global stores in 16-bit epilogues: {stg}"


def test_residual_epilogue_is_a_tma_reduce_add(gemm_functions):
    resid = {k: b for k, b in gemm_functions.items() if k[1] == EPI_GATE_RESIDUAL}
    assert len(resid) == 3 * 2 + 2 * 2      # forward: BN 128 / 192 / 256; wgrad (both operands transposed): BN 128 / 256
    no_red = [k for k, b in resid.items() if not re.search(r"\bUTMAREDG\.2D\.ADD\b", b)]
    assert no_red == [], f"no TMA reduce-add in {no_red}"
    other = {k: s for k, b in resid.items() for s in [[x for x in _global_stores(b) if x != "STG.E.64.STRONG.GPU"]] if s}
    assert other == {}, f"global stores other than the stream-K flag release: {other}"


def test_no_local_memory(gemm_functions):
    bad = [k for k, b in gemm_functions.items() if re.search(r"\b(LDL|STL)\b", b)]
    assert bad == [], f"local-memory accesses in {bad}"
