"""CPU: the FP8 (e4m3) GEMM of the sampling path, read from the built library's SASS, and its host-side argument checks.

fp8_linear_kernel<EPI, BF16> (bias and bias+GELU, fp16 / bf16 output) must multiply on the e4m3 tensor cores (`QGMMA`,
no 16-bit `HGMMA`), keep one k-block of MMAs in flight while it folds the previous k-block's partial sums into its fp32
total (`WARPGROUP.DEPBAR.LE gsb0, 0x1`), hand the producer's registers to the consumers (`USETMAXREG`) and keep its three
accumulator fragments in registers (no local memory)."""
import os
import re
import shutil
import subprocess

import pytest

from latte_b200 import _lib


@pytest.fixture(scope="module")
def fp8_functions():
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    _lib.load()
    sass = subprocess.run([cuobjdump, "-sass", _lib.lib_path()], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for chunk in sass.split("Function : ")[1:]:
        name, body = chunk.split("\n", 1)
        if "fp8_linear_kernel" in name:
            m = re.search(r"fp8_linear_kernelILi(\d+)ELb([01])EE", name)
            assert m, f"unexpected fp8_linear_kernel signature: {name}"
            funcs[tuple(int(g) for g in m.groups())] = body
    return funcs


def test_fp8_kernel_instances(fp8_functions):
    assert sorted(fp8_functions) == [(0, 0), (0, 1), (1, 0), (1, 1)]     # B200_EPI_BIAS / BIAS_GELU x fp16 / bf16 output


def test_fp8_kernel_uses_e4m3_wgmma(fp8_functions):
    for k, body in fp8_functions.items():
        assert re.search(r"\bQGMMA\.64x128x32\.F32\.E4M3\.E4M3\b", body), f"{k}: no e4m3 wgmma"
        assert "HGMMA" not in body, f"{k}: 16-bit wgmma in the FP8 kernel"


def test_fp8_kloop_pipelined_without_local_memory(fp8_functions):
    for k, body in fp8_functions.items():
        assert re.search(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x1\b", body), f"{k}: no wgmma wait<1> in the k-loop"
        assert "USETMAXREG" in body, f"{k}: no setmaxnreg"
        assert not re.search(r"\b(LDL|STL)\b", body), f"{k}: local-memory traffic"
        assert re.search(r"\bUTMASTG\.2D\b", body) and not re.search(r"\bSTG\b", body), f"{k}: output not stored by TMA"


def test_fp8_entry_points_check_arguments():
    """Shape checks run on the host before any CUDA call: rows that are not a multiple of 16 bytes are unsupported."""
    lib = _lib.load()
    rc = lib.b200_linear_e4m3(None, None, None, None, None, 128, 128, 72, _lib.FP16, _lib.EPI_BIAS, None, None)
    assert rc == -7 and "16 bytes" in _lib.last_error()
    rc = lib.b200_linear_e4m3(None, None, None, None, None, 128, 128, 64, _lib.FP16, _lib.EPI_GATE_RESIDUAL, None, None)
    assert rc == -7 and "epilogue" in _lib.last_error()
    rc = lib.b200_linear_e4m3(None, None, None, None, None, 128, 128, 64, 5, _lib.EPI_BIAS, None, None)
    assert rc == -2
    assert lib.b200_quantize_rows_e4m3(None, 4, 40, None, None, None) == -7
    assert lib.b200_ln_modulate_e4m3(None, None, None, 0, 1, None, None, 4, 40, None) == -1
