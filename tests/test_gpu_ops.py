"""GPU parity of each C-ABI op against a plain fp32 torch restatement of the reference op on the same
(16-bit-rounded) inputs.  Tolerances: fp16 operands 4e-3, bf16 3e-2 (abs + rel) — one rounding of the 16-bit
output dominates (2^-11 resp. 2^-8 of |value| <= ~8)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

TOL = {torch.float16: 4e-3, torch.bfloat16: 3e-2}


def _close(got, ref, tol):
    got, ref = got.float(), ref.float()
    err = (got - ref).abs()
    assert not torch.isnan(got).any()
    bad = err > tol + tol * ref.abs()
    assert not bad.any(), f"max err {err.max().item():.3e}, {bad.float().mean().item() * 100:.3f}% outside tol {tol}"


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("shape", [(128, 128, 64), (200, 192, 192), (256, 384, 1152), (640, 4608, 1152), (512, 1152, 4608), (4096, 3456, 1152)])
def test_linear_epilogues(dev, dt, shape):
    """nn.Linear (+GELU tanh | +gate*., +residual) — latte.py:50,75,169-171,179-180 — every tile width."""
    from latte_b200 import ops
    M, N, K = shape
    g = torch.Generator().manual_seed(M + N + K)
    A = torch.randn(M, K, generator=g).to(dev).to(dt)
    W = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev).to(dt)
    bias = torch.randn(N, generator=g).to(dev)
    ref = A.float() @ W.float().t() + bias
    for bn in (0, 128, 192, 256):
        _close(ops.linear(A, W, bias, block_n=bn), ref, TOL[dt])
    _close(ops.linear(A, W, None), ref - bias, TOL[dt])
    _close(ops.linear(A, W, bias, gelu=True), torch.nn.functional.gelu(ref, approximate="tanh"), TOL[dt])
    B = 2
    rpb = (M + B - 1) // B
    gate = torch.randn(B, N, generator=g).to(dev)
    resid = torch.randn(M, N, generator=g).to(dev)
    want = resid + gate[torch.arange(M, device=dev) // rpb] * ref
    ops.linear_gate_residual_(resid, A, W, bias, gate, rpb)
    _close(resid, want, 2e-4 if dt == torch.float16 else 2e-4)  # fp32 residual stream: only accumulation-order noise


@pytest.mark.parametrize("shape", [(8192, 1152, 4608), (8192 + 128, 1152, 2048), (4096 * 5, 384, 4096)])
def test_residual_linear_streamk(dev, shape):
    """The last partial wave of the gated-residual GEMM is split along K across all CTA pairs and the partial sums are
    reduce-added into x in k order (gemm.cu TileSched): same numbers as the unsplit restatement, bit-identical reruns."""
    from latte_b200 import ops
    M, N, K = shape
    g = torch.Generator().manual_seed(M + K)
    A = torch.randn(M, K, generator=g).to(dev).half()
    W = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev).half()
    bias = torch.randn(N, generator=g).to(dev)
    B = 2
    rpb = (M + B - 1) // B
    gate = torch.randn(B, N, generator=g).to(dev)
    x0 = torch.randn(M, N, generator=g).to(dev)
    want = x0 + gate[torch.arange(M, device=dev) // rpb] * (A.float() @ W.float().t() + bias)
    for bn in (0, 128, 192, 256):
        outs = []
        for _ in range(3):
            x = x0.clone()
            ops.linear_gate_residual_(x, A, W, bias, gate, rpb, block_n=bn)
            outs.append(x)
        _close(outs[0], want, 3e-4)
        assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])
        # the ordering flags live in the caller's buffer and every launch leaves them zero (no host-side launch counter:
        # that is what makes the step CUDA-graph replayable)
        torch.cuda.synchronize()
        assert int(ops._sk_flags(A.device).abs().sum()) == 0
        x = x0.clone()
        ops.linear_gate_residual_(x, A, W, bias, gate, rpb, block_n=bn, stream_k=False)   # data-parallel schedule
        _close(x, want, 3e-4)


def test_linear_is_linear_and_deterministic(dev):
    """Size-independent properties at the full XL/2 fc1 shape: f(a) + f(b) == f(a + b) (no bias) up to rounding; reruns are bit-identical."""
    from latte_b200 import ops
    g = torch.Generator().manual_seed(0)
    M, N, K = 8192, 4608, 1152
    a = (torch.randint(-4, 5, (M, K), generator=g).float() / 4).to(dev).half()   # exactly representable: sums are exact in fp32
    b = (torch.randint(-4, 5, (M, K), generator=g).float() / 4).to(dev).half()
    W = (torch.randint(-8, 9, (N, K), generator=g).float() / 64).to(dev).half()
    fa, fb, fab = ops.linear(a, W), ops.linear(b, W), ops.linear(a + b, W)
    assert torch.equal(ops.linear(a, W), fa)
    _close(fab, fa.float() + fb.float(), 4e-3)


def _attn_ref(qkv, batch, frames, tokens, heads, temporal):
    """Attention.forward 'math' (latte.py:50-70) on the regrouped tokens (latte.py:355,368), fp32."""
    T, D3 = qkv.shape
    D = D3 // 3
    hd = D // heads
    x = qkv.float().reshape(batch, frames, tokens, 3, heads, hd)
    x = x.permute(3, 0, 2, 4, 1, 5) if temporal else x.permute(3, 0, 1, 4, 2, 5)
    q, k, v = x[0], x[1], x[2]
    a = torch.softmax(q @ k.transpose(-1, -2) * hd ** -0.5, dim=-1)
    o = a @ v
    o = o.permute(0, 3, 1, 2, 4) if temporal else o.permute(0, 1, 3, 2, 4)
    return o.reshape(T, D)


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("case", [
    (2, 16, 256, 16, 72, False), (2, 16, 256, 16, 72, True),      # XL/2 spatial / temporal
    (2, 16, 256, 6, 64, False), (2, 16, 256, 6, 64, True),        # S/2
    (1, 4, 128, 2, 64, False), (2, 4, 64, 8, 72, False), (1, 2, 16, 2, 64, False),   # N = 128, packed N = 64, 16
    (2, 8, 64, 2, 64, True), (4, 4, 64, 8, 72, True), (1, 32, 32, 2, 80, True),      # F = 8, 4, 32; head_dim 80
    (1, 2, 512, 2, 64, False), (1, 2, 1024, 4, 72, False), (2, 16, 1024, 2, 72, True),  # LatteT2V @512px: N = 1024 (online softmax)
])
def test_attention(dev, dt, case):
    from latte_b200 import ops
    b, f, n, h, hd, temporal = case
    g = torch.Generator().manual_seed(b * 1000 + f * 10 + n + hd)
    qkv = (torch.randn(b * f * n, 3 * h * hd, generator=g) * 1.5).to(dev).to(dt)
    _close(ops.attention(qkv, b, f, n, h, temporal), _attn_ref(qkv, b, f, n, h, temporal), TOL[dt])


def test_attention_properties(dev):
    """V = 1 -> out = 1; Q = 0 -> out = mean of V over the sequence; permuting the keys of a sequence leaves the output unchanged."""
    from latte_b200 import ops
    b, f, n, h, hd = 1, 16, 256, 16, 72
    D = h * hd
    g = torch.Generator().manual_seed(9)
    qkv = torch.randn(b * f * n, 3 * D, generator=g).to(dev).half()
    one = qkv.clone(); one[:, 2 * D:] = 1
    for temporal in (False, True):
        _close(ops.attention(one, b, f, n, h, temporal), torch.ones(b * f * n, D, device=dev), 1e-3)
    q0 = qkv.clone(); q0[:, :D] = 0
    v = qkv[:, 2 * D:].float().reshape(b, f, n, D)
    _close(ops.attention(q0, b, f, n, h, False), v.mean(2, keepdim=True).expand(b, f, n, D).reshape(-1, D), 2e-3)
    _close(ops.attention(q0, b, f, n, h, True), v.mean(1, keepdim=True).expand(b, f, n, D).reshape(-1, D), 2e-3)
    # key/value permutation invariance within each frame (spatial): permute k and v rows, keep q
    perm = torch.randperm(n, generator=g).to(dev)
    x = qkv.reshape(b * f, n, 3 * D)
    xp = x.clone()
    xp[:, :, D:] = x[:, perm, D:]
    _close(ops.attention(xp.reshape(-1, 3 * D).contiguous(), b, f, n, h, False), ops.attention(qkv, b, f, n, h, False), 2e-3)


def test_attention_rejects_unsupported(dev):
    from latte_b200 import ops
    with pytest.raises(RuntimeError, match="UNSUPPORTED"):
        ops.attention(torch.zeros(384, 3 * 2 * 64, device=dev, dtype=torch.float16), 1, 1, 384, 2, False)   # N = 384: not 2^k <= 256 nor a multiple of 256
    with pytest.raises(RuntimeError, match="UNSUPPORTED"):
        ops.attention(torch.zeros(256, 3 * 2 * 48, device=dev, dtype=torch.float16), 1, 1, 256, 2, False)     # head_dim 48


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("D", [128, 384, 576, 1152])
def test_ln_modulate(dev, dt, D):
    """LayerNorm(no affine, eps 1e-6) + modulate — latte.py:28-29,166-168."""
    from latte_b200 import ops
    g = torch.Generator().manual_seed(D)
    rows, B = 96, 3
    x = (torch.randn(rows, D, generator=g) * 2 + 0.5).to(dev)
    mod = torch.randn(B, 6 * D, generator=g).to(dev)
    shift, scale = mod[:, :D], mod[:, D:2 * D]
    xn = torch.nn.functional.layer_norm(x, (D,), eps=1e-6)
    bidx = torch.arange(rows, device=dev) // (rows // B)
    _close(ops.ln_modulate(x, shift, scale, rows // B, dt), xn * (1 + scale[bidx]) + shift[bidx], TOL[dt])


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("case", [(2, 256, 120, 4, 72), (1, 1024, 20, 2, 64), (3, 128, 128, 2, 80), (2, 512, 1, 4, 72)])
def test_cross_attention(dev, dt, case):
    """diffusers Attention (attn2) with text keys (latte_t2v.py:862-870): q from the video tokens, k/v from <=128 text tokens."""
    from latte_b200 import ops
    b, rows, L, h, hd = case
    D = h * hd
    g = torch.Generator().manual_seed(rows + L)
    q = (torch.randn(b * rows, D, generator=g) * 1.5).to(dev).to(dt)
    kv = (torch.randn(b * L, 2 * D, generator=g) * 1.5).to(dev).to(dt)
    out = ops.cross_attention(q, kv, b, rows, L, h)
    qf = q.float().reshape(b, rows, h, hd).transpose(1, 2)
    kf = kv.float()[:, :D].reshape(b, L, h, hd).transpose(1, 2)
    vf = kv.float()[:, D:].reshape(b, L, h, hd).transpose(1, 2)
    ref = (torch.softmax(qf @ kf.transpose(-1, -2) * hd ** -0.5, dim=-1) @ vf).transpose(1, 2).reshape(b * rows, D)
    _close(out, ref, TOL[dt])


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("case", [(2, 256, 120, 4, 72, (12, 120)), (3, 128, 20, 2, 64, (1, 20, 7)), (2, 1024, 128, 2, 80, (128, 3))])
def test_cross_attention_key_bias(dev, dt, case):
    """Padded prompts (latte_t2v.py:766-771): the keep-mask becomes the additive bias (1 - m) * -10000 on the scores."""
    from latte_b200 import ops
    b, rows, L, h, hd, valid = case
    D = h * hd
    g = torch.Generator().manual_seed(rows + L + 1)
    q = (torch.randn(b * rows, D, generator=g) * 1.5).to(dev).to(dt)
    kv = (torch.randn(b * L, 2 * D, generator=g) * 1.5).to(dev).to(dt)
    mask = torch.zeros(b, L)
    for i in range(b):
        mask[i, : valid[i]] = 1
    bias = torch.zeros(b, 128)
    bias[:, :L] = (1 - mask) * -10000.0
    bias[:, L:] = 123.0                 # columns >= kv_len must be ignored
    out = ops.cross_attention(q, kv, b, rows, L, h, key_bias=bias.to(dev))
    qf = q.float().reshape(b, rows, h, hd).transpose(1, 2)
    kf = kv.float()[:, :D].reshape(b, L, h, hd).transpose(1, 2)
    vf = kv.float()[:, D:].reshape(b, L, h, hd).transpose(1, 2)
    sc = qf @ kf.transpose(-1, -2) * hd ** -0.5 + bias[:, :L].to(dev)[:, None, None, :]
    ref = (torch.softmax(sc, dim=-1) @ vf).transpose(1, 2).reshape(b * rows, D)
    _close(out, ref, TOL[dt])
    # an all-ones mask is the unmasked result (the bias path rounds s * scale once more: not bit-identical)
    zero = torch.zeros(b, 128, device=dev)
    _close(ops.cross_attention(q, kv, b, rows, L, h, key_bias=zero), ops.cross_attention(q, kv, b, rows, L, h), 2e-3 if dt == torch.float16 else 2e-2)
