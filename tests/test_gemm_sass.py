"""CPU: the shape of the wgmma GEMM's machine code, read from the built library's SASS.

Every gemm_kernel instantiation must keep its k-loop pipelined and warp-specialized:
- no empty `HGMMA ... gdesc[URZ]`: ptxas injects one when the loop holds several wgmma variants behind a run-time branch,
  and it turns the loop's "at most one k-block in flight" wait into a full drain;
- the k-loop waits with `WARPGROUP.DEPBAR.LE gsb0, 0x1` (the previous k-block may still run);
- `USETMAXREG`: the producer warpgroup hands its registers to the two consumer warpgroups.
The forward instantiations (bias, bias+GELU, gate+residual with K-major operands, every tile width and dtype) must also
keep their accumulators in registers: no local-memory traffic under the consumers' register budget."""
import os
import re
import shutil
import subprocess

import pytest

from latte_b200 import _lib

FORWARD_EPILOGUES = {0, 1, 2}   # B200_EPI_BIAS, B200_EPI_BIAS_GELU, B200_EPI_GATE_RESIDUAL


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
            funcs[name.strip()] = body
    assert funcs, "no gemm_kernel in the library's SASS"
    return funcs


def _template_args(name):
    """(BN, epilogue, bf16, operand layout) from the mangled name gemm_kernel<BN, EPI, BF16, MN>."""
    m = re.search(r"gemm_kernelILi(\d+)ELi(\d+)ELb([01])ELi(\d+)EE", name)
    assert m, f"unexpected gemm_kernel signature: {name}"
    return tuple(int(g) for g in m.groups())


def test_no_empty_wgmma_group(gemm_functions):
    bad = [n for n, body in gemm_functions.items() if re.search(r"HGMMA\.\S+ RZ, gdesc\[URZ\]", body)]
    assert bad == [], f"injected empty wgmma groups in {len(bad)} kernels, e.g. {bad[:2]}"


def test_kloop_keeps_one_group_in_flight(gemm_functions):
    bad = [n for n, body in gemm_functions.items() if not re.search(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x1\b", body)]
    assert bad == [], f"no wgmma wait<1> in {len(bad)} kernels, e.g. {bad[:2]}"


def test_register_budget_is_redistributed(gemm_functions):
    bad = [n for n, body in gemm_functions.items() if "USETMAXREG" not in body]
    assert bad == [], f"no setmaxnreg in {len(bad)} kernels, e.g. {bad[:2]}"


def test_forward_instantiations_have_no_local_memory(gemm_functions):
    forward = {n: b for n, b in gemm_functions.items()
               if _template_args(n)[1] in FORWARD_EPILOGUES and _template_args(n)[3] == 0}
    assert len(forward) == 3 * 3 * 2      # BN 128 / 192 / 256 x three epilogues x fp16 / bf16
    bad = [n for n, body in forward.items() if re.search(r"\b(LDL|STL)\b", body)]
    assert bad == [], f"local-memory accesses in forward GEMMs: {bad}"
