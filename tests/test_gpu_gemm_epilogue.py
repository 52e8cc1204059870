"""GEMM epilogues on tiles that lie wholly inside N but only partly inside M (M not a multiple of 8, so one warp holds both
live rows and rows past M): the chunked full-tile paths of gemm.cu must update exactly the live rows, with the same
numbers as a plain fp32 restatement, and leave memory past row M untouched."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _close(got, ref, tol):
    err = (got.float() - ref.float()).abs()
    assert not torch.isnan(got.float()).any()
    bad = err > tol + tol * ref.float().abs()
    assert not bad.any(), f"max err {err.max().item():.3e}, {bad.float().mean().item() * 100:.3f}% outside tol {tol}"


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("M", [100, 203, 1001])
@pytest.mark.parametrize("N,bn", [(384, 128), (384, 192), (512, 256)])
def test_epilogues_with_ragged_rows(dt, M, N, bn):
    from latte_b200 import ops
    dev = torch.device("cuda:0")
    K = 256
    g = torch.Generator().manual_seed(M * 7 + N + bn)
    A = torch.randn(M, K, generator=g).to(dev).to(dt)
    W = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev).to(dt)
    bias = torch.randn(N, generator=g).to(dev)
    ref = A.float() @ W.float().t() + bias
    tol16 = 4e-3 if dt == torch.float16 else 3e-2

    _close(ops.linear(A, W, bias, block_n=bn), ref, tol16)
    _close(ops.linear(A, W, bias, gelu=True, block_n=bn), torch.nn.functional.gelu(ref, approximate="tanh"), tol16)

    # residual stream with guard rows behind row M: they must come back unchanged
    B = 2
    rpb = (M + B - 1) // B
    gate = torch.randn(B, N, generator=g).to(dev)
    buf = torch.randn(M + 16, N, generator=g).to(dev)
    guard = buf[M:].clone()
    resid = buf[:M]
    want = resid + gate[torch.arange(M, device=dev) // rpb] * ref
    ops.linear_gate_residual_(resid, A, W, bias, gate, rpb, block_n=bn)
    torch.cuda.synchronize()
    _close(resid, want, 2e-4)
    assert torch.equal(buf[M:], guard)
