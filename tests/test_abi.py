"""CPU: the C-ABI library builds, loads without a GPU / libcuda, and exports every symbol the header declares."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from latte_b200 import _lib
    return _lib.load()


def _header_symbols():
    text = open(os.path.join(ROOT, "include", "latte_b200.h")).read()
    return sorted(set(re.findall(r"B200_API\s+[\w\s\*]+?\b(b200_\w+)\s*\(", text)))


def test_header_symbols_are_exported(lib):
    syms = _header_symbols()
    assert len(syms) >= 7 and "b200_latte_forward" in syms
    from latte_b200 import _lib
    assert sorted(_lib.EXPORTS) == syms, "ctypes binding table and include/latte_b200.h disagree"
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in the header but not exported by the .so"


def test_no_libcuda_dependency():
    """The driver API is resolved at run time so the library loads on the CPU-only build box."""
    import subprocess
    from latte_b200 import _lib
    out = subprocess.run(["ldd", _lib.lib_path()], capture_output=True, text=True).stdout
    assert "libcuda.so" not in out and "libtorch" not in out and "libc10" not in out, out


def test_sass_is_hopper_native():
    """The shipped cubin must be sm_90a and contain warpgroup MMA and TMA instructions (HGMMA, UTMALDG)."""
    import shutil
    import subprocess
    from latte_b200 import _lib
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", _lib.lib_path()], capture_output=True, text=True).stdout
    assert "sm_90a" in sass
    assert "HGMMA" in sass, "no wgmma in SASS"
    assert "UTMALDG" in sass
    # Legacy mma.sync (HMMA) is allowed in exactly one place: the attention BACKWARD of the training step (csrc/train.cu,
    # ~2 % of the backward FLOPs, first version on register fragments).  Every forward / sampling kernel and every GEMM of the
    # backward must be wgmma.
    legacy = set()
    for chunk in sass.split("Function : ")[1:]:
        name = chunk.split("\n", 1)[0]
        if re.search(r"(?<!G)HMMA", chunk):
            legacy.add(name)
    assert all("attn_bwd" in n for n in legacy), f"legacy mma.sync outside the attention backward: {sorted(legacy)[:4]}"


def test_exports_are_exactly_the_header(lib):
    """The library's dynamic symbol table holds exactly the b200_* entry points the header declares: nothing removed from
    the ABI lingers in the binary."""
    import shutil
    import subprocess
    from latte_b200 import _lib
    nm = shutil.which("nm")
    if nm is None:
        pytest.skip("nm not available")
    out = subprocess.run([nm, "-D", "--defined-only", _lib.lib_path()], capture_output=True, text=True, check=True).stdout
    exported = sorted({line.split()[-1] for line in out.splitlines() if line.split() and line.split()[-1].startswith("b200_")})
    assert exported == _header_symbols()


def test_library_reads_no_environment():
    """No code path of the library or the training engine is selected by an environment variable."""
    csrc = os.path.join(ROOT, "latte_b200", "csrc")
    readers = [f for f in sorted(os.listdir(csrc)) if os.path.isfile(os.path.join(csrc, f)) and
               "getenv" in open(os.path.join(csrc, f), encoding="utf-8", errors="replace").read()]
    assert readers == []
    assert "os.environ" not in open(os.path.join(ROOT, "latte_b200", "training.py")).read()


def test_abi_version_and_error_text(lib):
    from latte_b200 import _lib
    assert lib.b200_abi_version() == _lib.ABI_VERSION
    # host-side validation runs before any CUDA call: a bad shape must come back as an error code + message
    rc = lib.b200_linear(None, None, None, 128, 128, 65, 0, 0, None, None, None, 0, 1, 0, None, None)
    assert rc == -1 and "multiple of 64" in _lib.last_error()
    rc = lib.b200_linear(None, None, None, 128, 128, 64, 7, 0, None, None, None, 0, 1, 0, None, None)
    assert rc == -2
    rc = lib.b200_attention(None, None, 1, 16, 256, 4, 48, 0, 0, None)
    assert rc == -7 and "head_dim" in _lib.last_error()


def test_vae_layer_argument_checks(lib):
    """The single-layer VAE entry points validate shapes and pointers on the host, before any CUDA call."""
    from latte_b200 import _lib
    rc = lib.b200_vae_conv(None, None, None, None, None, None, 1, 16, 8, 96, 64, _lib.VAE_CONV3X3, _lib.FP16, None)
    assert rc == -7 and "multiple of 64" in _lib.last_error()
    rc = lib.b200_vae_conv(None, None, None, None, None, None, 1, 16, 8, 64, 128, _lib.VAE_CONV_T3, _lib.FP16, None)
    assert rc == -7 and "C -> C" in _lib.last_error()
    rc = lib.b200_vae_conv(None, None, None, None, None, None, 1, 16, 8, 64, 64, 9, _lib.FP16, None)
    assert rc == -7 and "kind" in _lib.last_error()
    assert lib.b200_vae_conv(None, None, None, None, None, None, 1, 16, 8, 64, 64, _lib.VAE_CONV_DOWN2, _lib.BF16, None) == -3
    assert lib.b200_group_norm(None, None, None, None, None, 1, 128, 64, 16, 1e-6, 0, 5, None) == -2
    assert lib.b200_group_norm(None, None, None, None, None, 1, 128, 64, 0, 1e-6, 0, 0, None) == -1
    assert lib.b200_vae_mid_attention_workspace_bytes(1, 8, 16, 96, 32) == 0 and "multiple of 64" in _lib.last_error()
    n, hw, C, G = 2, 128, 128, 32
    ws = lib.b200_vae_mid_attention_workspace_bytes(n, 8, 16, C, G)
    lower = 3 * n * hw * C * 2 + C * hw * 2 + hw * hw * (2 + 4) + hw * 4 + n * G * 8    # o, q, k, v^T, P, scores, ones, stats
    assert lower <= ws < lower + 8 * 1024


def test_workspace_size_formula(lib):
    from latte_b200 import _lib
    s = _lib.LatteShape(depth=28, hidden=1152, heads=16, mlp_hidden=4608, patch=2, in_channels=4, out_channels=8,
                        input_size=32, frames=16, num_embed=102, dtype=_lib.FP16)
    n = lib.b200_latte_workspace_bytes(C.byref(s), 2)
    T, D = 2 * 16 * 256, 1152
    lower = T * D * 4 + T * D * 2 + T * 3 * D * 2 + T * 4 * D * 2 + T * 32 * 4     # x, h, qkv, mlp hidden, head output
    assert lower <= n < lower + (1 << 21)       # + conditioning rows, stream-K flags, alignment
    s.heads = 10  # 1152/10 not an integer
    assert lib.b200_latte_workspace_bytes(C.byref(s), 2) == 0 and "heads" in _lib.last_error()
    s.heads = 16
    s.patch = 4
    assert lib.b200_latte_workspace_bytes(C.byref(s), 2) == 0 and "patch" in _lib.last_error()


def test_every_export_is_documented():
    """INTEGRATION.md section 1 maps each exported symbol to the reference code it replaces; the header declares all of them."""
    from latte_b200 import _lib
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    doc = open(os.path.join(root, "INTEGRATION.md")).read()
    hdr = open(os.path.join(root, "include", "latte_b200.h")).read()
    assert [n for n in _lib.EXPORTS if n not in doc] == []
    assert [n for n in _lib.EXPORTS if n not in hdr] == []
