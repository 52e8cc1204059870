"""Per-kernel timings at the Latte-XL/2 (B_model=2) shapes through the C ABI: CUDA events, L2 flushed between
iterations (a 256 MB memset), best-of / mean.  Usage: python tools/gpu_microbench.py [gemm] [attn] [ln]"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from latte_b200 import ops  # noqa: E402

dev = torch.device("cuda:0")
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)


def bench(fn, iters=20, do_flush=True):
    ts = []
    for i in range(iters + 3):
        if do_flush:
            flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        if i >= 3:
            ts.append(e0.elapsed_time(e1) * 1e3)
    ts.sort()
    return ts[0], sum(ts) / len(ts)


def gemm():
    T, D = 8192, 1152
    g = torch.Generator().manual_seed(0)
    for name, (M, N, K), mode in [("qkv", (T, 3 * D, D), "bias"), ("proj", (T, D, D), "resid"), ("fc1", (T, 4 * D, D), "gelu"), ("fc2", (T, D, 4 * D), "resid")]:
        A = torch.randn(M, K, generator=g).to(dev).half()
        W = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev).half()
        bias = torch.randn(N, generator=g).to(dev)
        gate = torch.randn(2, N, generator=g).to(dev)
        resid = torch.randn(M, N, generator=g).to(dev)
        fl = 2.0 * M * N * K
        # library yardstick (cuBLAS through torch; never on the product path): the plain GEMM without any epilogue
        Wt = W.t().contiguous()
        for fl_on in (True, False):
            best, mean = bench(lambda: torch.matmul(A, Wt), do_flush=fl_on)
            print(f"cublas {name:4s} {M}x{N}x{K}       {'cold' if fl_on else 'warm'}: best {best:7.1f} us mean {mean:7.1f} us -> {fl / best / 1e6:7.1f} TFLOP/s (best)", flush=True)
        best, mean = bench(lambda: torch.nn.functional.linear(A, W), do_flush=True)
        print(f"cublas {name:4s} linear(A, W[N,K])        cold: best {best:7.1f} us mean {mean:7.1f} us -> {fl / best / 1e6:7.1f} TFLOP/s (best)", flush=True)
        for bn in (128, 192, 256):
            if mode == "resid":
                fn = lambda: ops.linear_gate_residual_(resid, A, W, bias, gate, M // 2, block_n=bn)
            else:
                fn = lambda: ops.linear(A, W, bias, gelu=(mode == "gelu"), block_n=bn)
            for fl_on in (True, False):
                best, mean = bench(fn, do_flush=fl_on)
                print(f"gemm {name:4s} {M}x{N}x{K} bn{bn} {'cold' if fl_on else 'warm'}: best {best:7.1f} us mean {mean:7.1f} us -> {fl / best / 1e6:7.1f} TFLOP/s (best)", flush=True)
            if mode == "resid":
                # the same shape and tile width with the 16-bit bias epilogue instead: the difference to the line above is
                # what the gated-residual epilogue (fp32 x read + written in place) costs over the mainloop
                best, mean = bench(lambda: ops.linear(A, W, bias, block_n=bn), do_flush=True)
                print(f"gemm {name:4s} {M}x{N}x{K} bn{bn} bias-epilogue cold: best {best:7.1f} us mean {mean:7.1f} us -> {fl / best / 1e6:7.1f} TFLOP/s (best)", flush=True)


def attn():
    g = torch.Generator().manual_seed(1)
    b, f, n, h, hd = 2, 16, 256, 16, 72
    qkv = torch.randn(b * f * n, 3 * h * hd, generator=g).to(dev).half()
    for temporal in (False, True):
        for fl_on in (True, False):
            best, mean = bench(lambda: ops.attention(qkv, b, f, n, h, temporal), do_flush=fl_on)
            byts = qkv.numel() * 2 + b * f * n * h * hd * 2
            flops = 4.0 * (f * f * n if temporal else n * n * f) * h * hd * b
            print(f"attn {'temporal' if temporal else 'spatial '} {'cold' if fl_on else 'warm'}: best {best:7.1f} us mean {mean:7.1f} -> {byts / best / 1e3:7.1f} GB/s, {flops / best / 1e6:6.1f} TFLOP/s", flush=True)


def attn_long():
    """LatteT2V @512 px: spatial attention over N = 1024 tokens per frame (B_model = 2, 16 frames, 16 heads x 72)."""
    g = torch.Generator().manual_seed(3)
    b, f, n, h, hd = 2, 16, 1024, 16, 72
    qkv = torch.randn(b * f * n, 3 * h * hd, generator=g).to(dev).half()
    best, mean = bench(lambda: ops.attention(qkv, b, f, n, h, False), iters=10)
    flops = 4.0 * n * n * f * h * hd * b
    print(f"attn N=1024: best {best:7.1f} us mean {mean:7.1f} -> {flops / best / 1e6:6.1f} TFLOP/s", flush=True)


def ln():
    g = torch.Generator().manual_seed(2)
    T, D = 8192, 1152
    x = torch.randn(T, D, generator=g).to(dev)
    mod = torch.randn(2, 6 * D, generator=g).to(dev)
    for fl_on in (True, False):
        best, mean = bench(lambda: ops.ln_modulate(x, mod[:, :D], mod[:, D:2 * D], T // 2), do_flush=fl_on)
        print(f"ln_modulate {'cold' if fl_on else 'warm'}: best {best:6.1f} us mean {mean:6.1f} -> {(T * D * 6) / best / 1e3:7.1f} GB/s", flush=True)


if __name__ == "__main__":
    which = sys.argv[1:] or ["gemm", "attn", "ln"]
    print(torch.cuda.get_device_name(0), flush=True)
    for w in which:
        {"gemm": gemm, "attn": attn, "ln": ln, "attn_long": attn_long}[w]()
