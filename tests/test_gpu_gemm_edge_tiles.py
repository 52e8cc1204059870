"""GEMM epilogues on edge tiles in both directions: N not a multiple of the tile width (the last tile is partly past N, and
for 16-bit outputs its last 64-column chunk can be half past N) and M not a multiple of 8.  The output leaves through TMA
stores / reduce-adds, which clip rows past M and columns past N: the live part must match a plain fp32 restatement and the
rows behind the output must come back untouched, for the 16-bit store and for the residual reduce-add, with and without
the stream-K split."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu


def _close(got, ref, tol):
    err = (got.float() - ref.float()).abs()
    assert not torch.isnan(got.float()).any()
    bad = err > tol + tol * ref.float().abs()
    assert not bad.any(), f"max err {err.max().item():.3e}, {bad.float().mean().item() * 100:.3f}% outside tol {tol}"


def _linear_into(out, A, W, bias, gelu, bn):
    """b200_linear writing into `out` (a view whose rows are followed by guard rows)."""
    from latte_b200 import _lib, ops
    M, K = A.shape
    N = W.shape[0]
    rc = _lib.load().b200_linear(A.data_ptr(), W.data_ptr(), bias.data_ptr(), M, N, K, ops._dt(A),
                                 _lib.EPI_BIAS_GELU if gelu else _lib.EPI_BIAS, out.data_ptr(), None, None, 0, 1, bn,
                                 None, ops._stream(A))
    _lib.check(rc, "b200_linear")


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("M", [77, 1001])
@pytest.mark.parametrize("N", [96, 416, 480])
@pytest.mark.parametrize("bn", [128, 192, 256])
def test_ragged_n_and_m(dt, M, N, bn):
    from latte_b200 import ops
    dev = torch.device("cuda:0")
    K = 192
    g = torch.Generator().manual_seed(M * 31 + N * 7 + bn)
    A = torch.randn(M, K, generator=g).to(dev).to(dt)
    W = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev).to(dt)
    bias = torch.randn(N, generator=g).to(dev)
    ref = A.float() @ W.float().t() + bias
    tol16 = 4e-3 if dt == torch.float16 else 3e-2

    for gelu in (False, True):
        buf = torch.randn(M + 16, N, generator=g).to(dev).to(dt)
        guard = buf[M:].clone()
        _linear_into(buf[:M], A, W, bias, gelu, bn)
        torch.cuda.synchronize()
        _close(buf[:M], torch.nn.functional.gelu(ref, approximate="tanh") if gelu else ref, tol16)
        assert torch.equal(buf[M:], guard)

    B = 2
    rpb = (M + B - 1) // B
    gate = torch.randn(B, N, generator=g).to(dev)
    buf = torch.randn(M + 16, N, generator=g).to(dev)
    guard = buf[M:].clone()
    want = buf[:M] + gate[torch.arange(M, device=dev) // rpb] * ref
    ops.linear_gate_residual_(buf[:M], A, W, bias, gate, rpb, block_n=bn)
    torch.cuda.synchronize()
    _close(buf[:M], want, 2e-4)
    assert torch.equal(buf[M:], guard)


@pytest.mark.parametrize("bn", [128, 192, 256])
def test_streamk_reduce_add_on_ragged_tiles(bn):
    """Long K and more tiles than CTA pairs: the last waves are split along K and the segments of a tile are reduce-added
    in k order.  Reruns are bit-identical, the flags come back zero and the guard rows are untouched."""
    from latte_b200 import _lib, ops
    dev = torch.device("cuda:0")
    M, N, K = 16001, 416, 2560
    g = torch.Generator().manual_seed(bn)
    A = torch.randn(M, K, generator=g).to(dev).half()
    W = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev).half()
    bias = torch.randn(N, generator=g).to(dev)
    B = 3
    rpb = (M + B - 1) // B
    gate = torch.randn(B, N, generator=g).to(dev)
    x0 = torch.randn(M + 16, N, generator=g).to(dev)
    streamk = ctypes.c_int()
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    _lib.load().b200_gemm_schedule(M, N, K, _lib.EPI_GATE_RESIDUAL, bn, sms, None, None, ctypes.byref(streamk), None, 0)
    assert streamk.value == 1, "this shape is meant to take the stream-K schedule"
    want = x0[:M] + gate[torch.arange(M, device=dev) // rpb] * (A.float() @ W.float().t() + bias)
    outs = []
    for _ in range(3):
        x = x0.clone()
        ops.linear_gate_residual_(x[:M], A, W, bias, gate, rpb, block_n=bn)
        outs.append(x)
    torch.cuda.synchronize()
    _close(outs[0][:M], want, 3e-4)
    assert torch.equal(outs[0][M:], x0[M:])
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])
    assert int(ops._sk_flags(dev).abs().sum()) == 0
