"""GPU: the forward kernels against fp64, element by element -- the GEMM epilogues, attention, cross-attention, LayerNorm +
modulate, and the conditioning, patch-embedding, output-head and guidance kernels reached through `Latte`.

The reference of each op is its forward expression in fp64 on the GPU, evaluated on the same 16-bit and fp32 tensors the
kernel reads.  Every output element must satisfy (tests/fp64_bounds.py, A = 2, B = 4, F = 3)

    |got - ref| <= A * u_out * |ref| + B * u_op * mag + floor

  * u_out: unit roundoff of the output (fp16 2^-11, bf16 2^-8, fp32 2^-24); floor: one fp16 subnormal spacing (2^-24) for a
    16-bit output, 0 in bf16.
  * GEMM (`linear`, three epilogues).  mag = |a| |w|^T + |bias|; u_op = ACC * sqrt(K) * 2^-24, the probabilistic growth of
    the fp32 tensor-core accumulation over K (Higham & Mary).  The wgmma accumulator does not round every add to nearest
    (products are aligned to the largest exponent of a group and truncated), so ACC is measured, not assumed: worst
    err / (2^-24 mag) of the fp32 accumulation (gated-residual epilogue, gate 1, zero residual, no bias, data-parallel
    schedule, M = 8192, N = 1152, three +-60 outliers per row) on an H100 80GB HBM3 at a 700 W power limit:

        K                                64      192     1152    4608
        fp16 err / (2^-24 mag)           8.47    13.0    18.9    22.4     / sqrt(K): 1.06  0.94  0.56  0.33
        bf16 err / (2^-24 mag)           6.27    9.67    17.1    19.4     / sqrt(K): 0.78  0.70  0.50  0.29

    The error grows more slowly than sqrt(K) (the ratio to sqrt(K) falls as K grows), so no K-linear term is needed: ACC = 1
    keeps the sqrt(K) form, and the worst case, 1.06 sqrt(K) at K = 64, sits at a quarter of B * sqrt(K).
      - bias (qkv): one rounding of the 16-bit output; the fp32 bias add is inside u_op * mag.
      - GELU (fc1): gelu_tanh(pre) with |gelu'(pre)| * u_op * mag for the accumulation, plus tanh.approx.f32 (relative
        error 2^-11 of t = tanh(u)) times 0.5 |pre|, plus the four fp32 roundings of u = k0 (x + k1 x^3) times
        0.5 |pre| (1 - t^2) |u|.  For pre <~ -2 the 1 + t cancels: the result is tiny, the tanh.approx term is not, and a
        bound without it fails on correct code.  The same term is as large as the difference between GELU-tanh and
        GELU-erf (under 5e-4 in absolute value), so this bound cannot tell the two apart.
      - gated residual (proj / fc2 / the N = 32 head): x += gate[b] * (acc + bias), fp32 throughout; mag = |x| +
        |gate| (|a| |w| + |bias|).  The add, the product, the bias add and (stream-K) one extra add per K segment are at
        most 4 roundings of values below mag: 4 * 2^-24 <= sqrt(K) * 2^-24 for every K >= 16.
  * Attention (spatial, temporal, cross).  mag = sum_j p_j |v_j| (p the softmax); u_op per query row = 2^-11 / 2^-8 (P
    is rounded to 16 bits before the PV product; its sum l stays fp32) + 2 * 2^-24 * log2(e) * max|s| (the fp32 exp2
    argument s * scale * log2(e), natural-log scores s, +-30 logits, -10000 key biases; the max runs over the keys with
    nonzero probability, tests/fp64_bounds.softmax_fwd_terms) + 2^-22 (ex2.approx.f32) +
    ACC * sqrt(hd) * 2^-24 * max_j |q| |k_j| * scale (the fp32 QK^T) + sqrt(S) * 2^-24 (the fp32 PV and l sums).  fp16
    floor: 2^-24 plus F * p_max * sqrt(sum_j (min(2^-24, P_j) |v_j|)^2) with P_j = p_j / p_max the unnormalised
    probability the kernel rounds (its subnormals are off by up to half a spacing each, independently).
  * ln_modulate: y = xh (1 + scale[b]) + shift[b], xh = (x - mean) rstd; the fp32 statistics are off by sqrt(D) * 2^-24 *
    (rstd mean|x| + |xh|) in xh (a row with mean 8 and spread 0.05 loses digits in the mean), plus 3 roundings of xh and
    one of 1 + scale and of the fma.
  * Conditioning (t_embedder, y_embedder, every adaLN row): a first-order error vector is carried through the chain in
    fp64 -- sinusoid 2^-24 (|t freq| + 1) (the fp32 argument, computed in fp32 by the reference too, and cosf / sinf);
    each gemv sqrt(K) * 2^-24 * (|W| |in| + |bias| + |label row|) plus |W| times the input's error; SiLU |silu'(x)|
    times the input's error plus the __expf error (2 + 1.173 |x| ulp, CUDA C Programming Guide) and two roundings.
    The adaLN gemv reads the module's 16-bit weights, and so does the reference.
  * Embedding and head: patch_embed + pos_embed (+ temp_embed, block 0's epilogue) carries sqrt(K + 2) * 2^-24 of its
    magnitude; LayerNorm propagates it (rstd (e + mean e + |xh| mean(|xh| e))) and adds its own fp32 term as above; the
    modulated row is rounded to 16 bits for the tensor-core head (n_out = 32: u16 |y| |w|, plus the fp16 subnormal
    floor) and kept fp32 for final_layer_kernel (n_out = 16); the head adds sqrt(D) * 2^-24 (|y| |w| + |bias|).
  * Guidance: forward_with_cfg's eps channels equal u + s * (c - u) evaluated in fp32 (the product rounded, then the sum)
    on the halves of a plain forward of the same batch, bit for bit.

Every op runs in fp16 and bf16.  For each op the file also shows that its bound rejects a plausible wrong result built from
the kernel's own output (the bias added after the GELU, a dropped bias on the last partial N tile, the neighbouring sample's gate
on a boundary row, a dropped last key, an ignored key bias, LayerNorm with eps 1e-5, the previous sample's shift/scale,
the label of another sample, a transposed patch in unpatchify, an fma in the guidance).  The worst err / bound of each op
and dtype is printed at the end of the module (pytest -s)."""
import math

import pytest
import torch
import torch.nn.functional as Fn

from fp64_bounds import A, ACC, B, DTS, GELU_K0, GELU_K1, SUB, U16, U32, Checker, report_worst, sqfloor  # noqa: E402
from fp64_bounds import edge_rows, gelu_fwd_terms, silu_err, softmax_fwd_terms, to_rows, to_seq  # noqa: E402

pytestmark = pytest.mark.gpu

_WORST = {}
_ACC_TABLE = {}


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    if _ACC_TABLE:
        print("\nfp32 tensor-core accumulation: worst err / (2^-24 mag), and that / sqrt(K):")
        for (dt, K), r in sorted(_ACC_TABLE.items()):
            print(f"  {dt:<9} K = {K:5d}   {r:8.3g}   {r / math.sqrt(K):8.3g}")
    report_worst(_WORST)


def _chk(dt):
    return Checker(dt, _WORST)


def _rejects(dt, op, got, ref, bound):
    """The bound must reject a wrong result."""
    m = Checker(dt)
    m.add(op, "wrong result", got, ref, bound, lambda i: str(i))
    assert m.bad, f"{op}: the bound accepts a wrong result"


def _rc(idx):
    return f"row {idx[0]}, column {idx[1]}"


def _outliers(x, g, per_row=3, value=60.0):
    """A few +-value entries per row (activations after LayerNorm + modulate with a large scale)."""
    M, K = x.shape
    cols = torch.randint(0, K, (M, per_row), device=x.device, generator=g)
    sign = torch.randint(0, 2, (M, per_row), device=x.device, generator=g).to(x.dtype) * 2 - 1
    x.scatter_(1, cols, value * sign)
    return x


# ------------------------------------------------------------------------------------------------ GEMM
def _linear_into(out, a, w, bias, gelu, bn):
    """b200_linear writing into `out` (a view whose rows are followed by guard rows)."""
    from latte_b200 import _lib, ops
    M, K = a.shape
    rc = _lib.load().b200_linear(a.data_ptr(), w.data_ptr(), bias.data_ptr(), M, w.shape[0], K, ops._dt(a),
                                 _lib.EPI_BIAS_GELU if gelu else _lib.EPI_BIAS, out.data_ptr(), None, None, 0, 1, bn,
                                 None, ops._stream(a))
    _lib.check(rc, "b200_linear")


def _gemm_inputs(dev, dt, M, N, K, seed):
    """Activations with three +-60 outliers per row; Xavier-uniform weights with one block of 32 output rows at the
    adaLN-Zero scale (1e-4), whose biases are as small, so those outputs are small."""
    g = torch.Generator(device=dev).manual_seed(seed)
    a = _outliers(torch.randn(M, K, device=dev, generator=g), g).to(dt)
    lim = math.sqrt(6.0 / (K + N))
    w = (torch.rand(N, K, device=dev, generator=g) * 2 - 1) * lim
    blk = slice(N // 2, min(N, N // 2 + 32))
    w[blk] *= 1e-4 / lim
    w = w.to(dt)
    bias = torch.randn(N, device=dev, generator=g) * 0.5
    bias[blk] *= 1e-4
    return g, a, w, bias, blk


def _gelu64(u):
    return 0.5 * u * (1 + torch.tanh(GELU_K0 * (u + GELU_K1 * u ** 3)))


GEMM_SHAPES = {  # (N, K) of the model GEMMs
    "XL/2 qkv": (3456, 1152), "XL/2 proj": (1152, 1152), "XL/2 fc1": (4608, 1152), "XL/2 fc2": (1152, 4608),
    "S/2 qkv": (1152, 384), "S/2 proj": (384, 384), "S/2 fc1": (1536, 384), "S/2 fc2": (384, 1536),
    "head XL/2": (32, 1152), "head S/2": (32, 384),
}


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("M", [77, 1001, 8192, 16001])
@pytest.mark.parametrize("shape", list(GEMM_SHAPES))
def test_linear(dev, dt, M, shape):
    """All three epilogues at block_n 0 (the planner's choice), 128, 192 and 256; the gated residual with and without
    stream-K; 16 guard rows behind M in every output; three samples whose boundaries fall inside a 128-row tile, gates
    read from a strided adaLN-row view."""
    from latte_b200 import ops
    N, K = GEMM_SHAPES[shape]
    chk = _chk(dt)
    g, a, w, bias, blk = _gemm_inputs(dev, dt, M, N, K, M * 7 + N * 3 + K)
    Bb = 3
    rpb = -(-M // Bb)
    mod = torch.randn(Bb, 6 * N, device=dev, generator=g) * 0.5
    gate = mod[:, 2 * N:3 * N]
    x0 = torch.randn(M + 16, N, device=dev, generator=g) * 4
    buf0 = torch.randn(M + 16, N, device=dev, generator=g).to(dt)

    a64, w64, b64 = a.double(), w.double(), bias.double()
    pre = a64 @ w64.t() + b64
    mag = a64.abs() @ w64.abs().t() + b64.abs()
    del a64, w64
    uacc = ACC * math.sqrt(K) * U32
    tag = f"{shape} M={M}"
    sub = SUB[dt]

    # bias epilogue (qkv)
    bnd_bias = A * U16[dt] * pre.abs() + B * uacc * mag + sub
    # GELU epilogue (fc1)
    ref_gelu, term = gelu_fwd_terms(pre, uacc, mag)
    bnd_gelu = A * U16[dt] * ref_gelu.abs() + term + sub
    del term
    # gated residual (proj / fc2 / head)
    bidx = torch.arange(M, device=dev) // rpb
    g64 = gate.double()[bidx]
    ref_res = x0[:M].double() + g64 * pre
    bnd_res = A * U32 * ref_res.abs() + B * uacc * (x0[:M].double().abs() + g64.abs() * mag)

    outs = {}
    for bn in (0, 128, 192, 256):
        for gelu in (False, True):
            buf = buf0.clone()
            _linear_into(buf[:M], a, w, bias, gelu, bn)
            torch.cuda.synchronize()
            assert torch.equal(buf[M:], buf0[M:]), f"{tag} bn={bn}: rows past M written"
            name = "linear bias+gelu" if gelu else "linear bias"
            chk.add(name, f"{tag} bn={bn}", buf[:M], ref_gelu if gelu else pre, bnd_gelu if gelu else bnd_bias, _rc)
            outs[(bn, gelu)] = buf[:M]
        for sk in (True, False):
            x = x0.clone()
            ops.linear_gate_residual_(x[:M], a, w, bias, gate, rpb, block_n=bn, stream_k=sk)
            torch.cuda.synchronize()
            assert torch.equal(x[M:], x0[M:]), f"{tag} bn={bn}: residual rows past M written"
            chk.add("linear gate+residual", f"{tag} bn={bn} stream-K={sk}", x[:M], ref_res, bnd_res, _rc)
            outs[(bn, "res")] = x[:M]
    chk.done()

    # the bounds reject plausible wrong results built from the kernel's own output
    got = outs[(0, True)].double()
    late = _gelu64(pre - b64) + b64
    _rejects(dt, "GELU applied before the bias", (got + late - ref_gelu).to(dt), ref_gelu, bnd_gelu)
    for bn in (256, 192, 128):
        if N % bn:
            c0 = N - N % bn
            wrong = outs[(bn, False)].double()
            wrong[:, c0:] -= b64[c0:]
            _rejects(dt, "bias dropped on the last partial N tile", wrong.to(dt), pre, bnd_bias)
            break
    wrong = outs[(0, "res")].clone()
    wrong[rpb] += ((gate[0] - gate[1]).double() * pre[rpb]).float()
    _rejects(dt, "neighbouring sample's gate on the boundary row", wrong, ref_res, bnd_res)


@pytest.mark.parametrize("dt", DTS)
def test_gemm_accumulation(dev, dt):
    """The fp32 accumulation alone: x = 0 + 1 * (a w^T) through the gated-residual epilogue on the data-parallel schedule
    (one exact add into a zero residual), M = 8192, N = 1152, at K = 64, 192, 1152 and 4608.  Records worst
    err / (2^-24 mag) per K (the numbers behind ACC) and holds it to B * ACC * sqrt(K)."""
    from latte_b200 import ops
    chk = _chk(dt)
    M, N = 8192, 1152
    for K in (64, 192, 1152, 4608):
        _, a, w, _, _ = _gemm_inputs(dev, dt, M, N, K, K)
        x = torch.zeros(M, N, device=dev)
        ones = torch.ones(1, N, device=dev)
        ops.linear_gate_residual_(x, a, w, None, ones, M, stream_k=False)
        a64, w64 = a.double(), w.double()
        ref = a64 @ w64.t()
        mag = a64.abs() @ w64.abs().t()
        del a64, w64
        r = float(((x.double() - ref).abs() / (U32 * mag).clamp_min(1e-300)).max())
        _ACC_TABLE[(str(dt).replace("torch.", ""), K)] = r
        chk.add("gemm fp32 accumulation", f"K={K}", x, ref, A * U32 * ref.abs() + B * ACC * math.sqrt(K) * U32 * mag, _rc)
    chk.done()


# ------------------------------------------------------------------------------------------------ attention
def _attention_case(dev, dt, Bb, Fr, N, H, hd, temporal):
    from latte_b200 import ops
    chk = _chk(dt)
    kind = "temporal" if temporal else "spatial"
    S, nseq = (Fr, Bb * N) if temporal else (N, Bb * Fr)
    g = torch.Generator(device=dev).manual_seed(Bb * 100003 + Fr * 1009 + N * 7 + hd)
    x = torch.randn(nseq, 3, H, S, hd, device=dev, generator=g)
    edge_rows(x)
    qkv = to_rows(x, Bb, Fr, N, H, hd, temporal).to(dt).contiguous()
    del x
    got = to_seq(ops.attention(qkv, Bb, Fr, N, H, temporal), Bb, Fr, N, 1, H, hd, temporal)[:, 0]
    qs = to_seq(qkv, Bb, Fr, N, 3, H, hd, temporal).double()
    step = max(1, (1 << 24) // (H * S * S))           # sequences per fp64 reference chunk: <= 2^24 scores per tensor
    tag = f"B={Bb} F={Fr} N={N} H={H} hd={hd}"

    def where(c0):
        def f(i):
            sq, h, pos, d = c0 + i[0], i[1], i[2], i[3]
            row = ((sq // N) * Fr + pos) * N + sq % N if temporal else sq * N + pos
            return f"{kind} sequence {sq}, head {h}, position {pos} (row {row}), dim {d}"
        return f

    for c0 in range(0, nseq, step):
        c1 = min(nseq, c0 + step)
        q, k, v = qs[c0:c1, 0], qs[c0:c1, 1], qs[c0:c1, 2]
        ref, term, _ = softmax_fwd_terms(q, k, v, None, dt)
        bnd = A * U16[dt] * ref.abs() + term
        chk.add(f"attention {kind}", tag, got[c0:c1], ref, bnd, where(c0))
        if c0 == 0 and S > 1:       # a kernel that drops the last key of every sequence
            short = torch.softmax(q @ k[..., :-1, :].transpose(-1, -2) * hd ** -0.5, -1) @ v[..., :-1, :]
            _rejects(dt, f"attention {kind}: last key dropped", (got[c0:c1].double() + short - ref).to(dt), ref, bnd)
        del ref, term, bnd
    chk.done()


HEADS = [(16, 72), (6, 64), (4, 80)]


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("H,hd", HEADS)
@pytest.mark.parametrize("N,Bf", [(16, (2, 8)), (32, (2, 4)), (64, (2, 4)), (128, (1, 4)), (256, (2, 2)), (512, (1, 2)),
                                  (1024, (1, 2))])
def test_attention_spatial(dev, dt, H, hd, N, Bf):
    """N <= 64: sequences packed 128 / N per tile; N = 128: one tile; N >= 256: key chunks with the online softmax."""
    _attention_case(dev, dt, Bf[0], Bf[1], N, H, hd, False)


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("H,hd", HEADS)
@pytest.mark.parametrize("Fr", [1, 2, 15, 16, 17, 33, 64, 100, 128])
def test_attention_temporal(dev, dt, H, hd, Fr):
    """F a power of two: the xor-masked full tile; any other F: the partial tile; five tokens per frame, so the last token
    group of a sequence is partial unless it divides 5."""
    _attention_case(dev, dt, 2, Fr, 5, H, hd, True)


XCASES = [  # (samples, query rows per sample, kv_len, heads, hd, mask)
    (2, 128, 1, 16, 72, None), (2, 256, 20, 16, 72, "partial"), (1, 1024, 120, 16, 72, "partial"),
    (2, 1024, 128, 16, 72, None), (3, 128, 128, 6, 64, "all"), (2, 256, 120, 4, 80, "partial"),
    (3, 256, 20, 6, 64, None), (2, 128, 128, 16, 72, "partial"),
]


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("case", XCASES, ids=lambda c: "-".join(str(v) for v in c))
def test_cross_attention(dev, dt, case):
    """Queries of each sample against its kv_len text keys; key_bias None, or padded prompts: keys past a per-sample
    prompt length get -10000 (sample 0 keeps L/2 + 1 keys, one sample keeps 1 key), and "all" masks the last sample
    entirely; columns >= kv_len of key_bias hold 123 and must be ignored."""
    from latte_b200 import ops
    Bn, rows, L, H, hd, mask = case
    D = H * hd
    chk = _chk(dt)
    g = torch.Generator(device=dev).manual_seed(rows + L + hd + Bn)
    q = torch.randn(Bn * rows, D, device=dev, generator=g)
    kv = torch.randn(Bn * L, 2 * D, device=dev, generator=g)
    q[::7] *= 4                                                      # logits up to ~+-30
    q, kv = q.to(dt), kv.to(dt)
    bias = None
    if mask is not None:
        bias = torch.zeros(Bn, 128, device=dev)
        bias[:, L:] = 123.0
        bias[0, L // 2 + 1:L] = -10000.0
        if Bn > 1:
            bias[1, 1:L] = -10000.0
        if mask == "all":
            bias[Bn - 1, :L] = -10000.0
    got = ops.cross_attention(q, kv, Bn, rows, L, H, key_bias=bias).reshape(Bn, rows, H, hd).transpose(1, 2)
    q4 = q.double().reshape(Bn, rows, H, hd).transpose(1, 2)
    kv5 = kv.double().reshape(Bn, L, 2, H, hd)
    k4, v4 = kv5[:, :, 0].transpose(1, 2), kv5[:, :, 1].transpose(1, 2)
    for n0 in range(Bn):
        b4 = bias[n0:n0 + 1, None, None, :L].double() if bias is not None else None
        ref, term, _ = softmax_fwd_terms(q4[n0:n0 + 1], k4[n0:n0 + 1], v4[n0:n0 + 1], b4, dt)
        bnd = A * U16[dt] * ref.abs() + term

        def where(i, n0=n0):
            return f"sample {n0}, head {i[1]}, query {i[2]}, dim {i[3]}"
        chk.add(f"cross_attention {'key_bias' if bias is not None else 'no bias'}", f"{case}", got[n0:n0 + 1], ref, bnd, where)
        if bias is not None and n0 == 0:
            free, _, _ = softmax_fwd_terms(q4[:1], k4[:1], v4[:1], None, dt)
            _rejects(dt, "cross_attention: key_bias ignored", (got[:1].double() + free - ref).to(dt), ref, bnd)
    chk.done()


# ------------------------------------------------------------------------------------------------ ln_modulate
LN_CASES = [(3, 37, 5), (3, 4095, 1000), (5, 1023, 0)]     # (samples, rows_per_batch, rows missing from the last sample)


def _ln_ref(x64, shift, scale, bidx, eps=1e-6):
    mean = x64.mean(1, keepdim=True)
    rstd = (((x64 - mean) ** 2).mean(1, keepdim=True) + eps).rsqrt()
    xh = (x64 - mean) * rstd
    return xh, rstd, xh * (1 + scale.double()[bidx]) + shift.double()[bidx]


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("D", [384, 576, 768, 1024, 1152, 1536])     # ln_modulate's NV = 3, 6, 6, 9, 9, 12 variants
def test_ln_modulate(dev, dt, D):
    """LayerNorm(x) (1 + scale[b]) + shift[b] (eps 1e-6) -> 16-bit, shift / scale strided views of adaLN rows.  Sample
    boundaries fall inside a block's rows (37, 4095 and 1023 are not multiples of the 4 warps x rows-per-warp of a block),
    so one block reads the staged shift / scale for its first sample and the global ones after the boundary; the last
    sample is short.  Every third row has mean 8 and spread 0.05."""
    from latte_b200 import ops
    chk = _chk(dt)
    g = torch.Generator(device=dev).manual_seed(D + 1)
    for Bb, rpb, short in LN_CASES:
        T = Bb * rpb - short
        x = torch.randn(T, D, device=dev, generator=g) * 3 + 1
        x[::3] = 8 + 0.05 * torch.randn(x[::3].shape, device=dev, generator=g)
        mod = torch.randn(Bb, 6 * D, device=dev, generator=g) * 0.5
        shift, scale = mod[:, 3 * D:4 * D], mod[:, 4 * D:5 * D]
        got = ops.ln_modulate(x, shift, scale, rpb, dt)
        bidx = torch.arange(T, device=dev) // rpb
        x64 = x.double()
        xh, rstd, ref = _ln_ref(x64, shift, scale, bidx)
        c1 = (1 + scale.double()[bidx]).abs()
        e_xh = U32 * (math.sqrt(D) * (rstd * x64.abs().mean(1, keepdim=True) + xh.abs()) + 3 * xh.abs())
        e_y = c1 * e_xh + U32 * (2 * xh.abs() * c1 + shift.double()[bidx].abs())
        bnd = A * U16[dt] * ref.abs() + B * e_y + SUB[dt]
        tag = f"B={Bb} rpb={rpb} T={T}"
        chk.add("ln_modulate", tag, got, ref, bnd, _rc)
        wrong = got.double().clone()
        first = torch.arange(rpb, T, rpb, device=dev)
        wrong[first] = (xh[first] * (1 + scale.double()[bidx[first] - 1]) + shift.double()[bidx[first] - 1])
        _rejects(dt, "ln_modulate: previous sample's shift/scale after a boundary", wrong.to(dt), ref, bnd)
        if dt == torch.float16:
            _, _, eps5 = _ln_ref(x64, shift, scale, bidx, 1e-5)
            _rejects(dt, "ln_modulate: eps 1e-5", (got.double() + eps5 - ref).to(dt), ref, bnd)
        del x64, xh, rstd, ref, e_xh, e_y, bnd
    chk.done()


# ------------------------------------------------------------------------------------------------ glue through Latte
def _latte(dev, dt, D, heads, extras, learn_sigma, depth=2, frames=4, input_size=16, seed=0, zero_gates=False):
    """A small Latte with the oracle's seeded weights (every path carries signal), on the GPU with `dt` operands."""
    from latte_b200 import Latte
    from oracle import latte_oracle as O
    cfg = O.LatteConfig(input_size=input_size, hidden_size=D, depth=depth, num_heads=heads, num_frames=frames,
                        num_classes=10, learn_sigma=learn_sigma, extras=extras)
    sd = O.make_weights(cfg, seed)
    if zero_gates:       # gate_msa / gate_mlp rows of every block's adaLN: each block is the identity on x
        for i in range(depth):
            for c in (2, 5):
                sd[f"blocks.{i}.adaLN_modulation.1.weight"][c * D:(c + 1) * D] = 0
                sd[f"blocks.{i}.adaLN_modulation.1.bias"][c * D:(c + 1) * D] = 0
    net = Latte(input_size=input_size, hidden_size=D, depth=depth, num_heads=heads, num_frames=frames, num_classes=10,
                learn_sigma=learn_sigma, extras=extras)
    net.load_state_dict(sd, strict=True)
    net = net.to(dev).eval()
    net.compute_dtype = dt
    return cfg, {k: v.to(dev) for k, v in sd.items()}, net


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("D,heads", [(384, 6), (1152, 16)])
@pytest.mark.parametrize("extras", [1, 2])
def test_conditioning(dev, dt, D, heads, extras):
    """precompute_conditioning: every adaLN row (2 blocks x 6D + the final layer's 2D) for 3 steps x 4 samples = 12 rows
    (the gemv runs them as 8 + 4), t in {0, 1, 500, 998, 999}, labels including the null class, against the oracle's
    t_embedder / y_embedder and the adaLN Linear in fp64 on the module's 16-bit weights."""
    from oracle import latte_oracle as O
    chk = _chk(dt)
    cfg, sd, net = _latte(dev, dt, D, heads, extras, True, seed=D + extras)
    ts = torch.tensor([[0, 1, 500, 999], [998, 999, 0, 1], [500, 998, 999, 0]], device=dev)
    y = torch.tensor([3, 10, 7, 0], device=dev) if extras == 2 else None     # 10 = num_classes: the null class
    got = net.precompute_conditioning(ts, y).reshape(12, -1)
    _, _, T, _ = net._pack()
    w16, ab = T["ada_w16"].double(), T["ada_b"].double()
    net.clear_conditioning()
    t = ts.reshape(-1)
    yy = y.repeat(3) if y is not None else None
    sd64 = {k: v.double() for k, v in sd.items()}
    c = O.t_embedder(sd64, t, torch.float64)
    if extras == 2:
        c = c + O.y_embedder(sd64, yy, torch.float64)
    ref = Fn.linear(Fn.silu(c), w16, ab)
    # magnitudes and first-order errors along the chain
    freqs = torch.exp(-math.log(10000) * torch.arange(0, 128, dtype=torch.float32) / 128).to(dev)   # oracle.timestep_embedding
    arg = (t[:, None].float() * freqs[None]).double()
    tf = torch.cat([torch.cos(arg), torch.sin(arg)], 1)
    e = U32 * (torch.cat([arg, arg], 1).abs() + 1)
    W0, b0, W2, b2 = (sd64[k] for k in ("t_embedder.mlp.0.weight", "t_embedder.mlp.0.bias", "t_embedder.mlp.2.weight",
                                        "t_embedder.mlp.2.bias"))
    h1 = tf @ W0.t() + b0
    e = e @ W0.abs().t() + U32 * math.sqrt(256) * (tf.abs() @ W0.abs().t() + b0.abs())
    s1 = Fn.silu(h1)
    e = silu_err(h1, e)
    lab = O.y_embedder(sd64, yy, torch.float64).abs() if extras == 2 else 0
    e = e @ W2.abs().t() + U32 * math.sqrt(D) * (s1.abs() @ W2.abs().t() + b2.abs() + lab)
    sc = Fn.silu(c)
    e = silu_err(c, e)
    e = e @ w16.abs().t() + U32 * math.sqrt(D) * (sc.abs() @ w16.abs().t() + ab.abs())
    bnd = A * U32 * ref.abs() + B * e
    chk.add("conditioning adaLN rows", f"D={D} extras={extras}", got, ref, bnd,
            lambda i: f"row {i[0]} (step {i[0] // 4}, sample {i[0] % 4}), adaLN column {i[1]}")
    chk.done()
    if extras == 2:     # rows 8..11 (the second gemv chunk) with the labels of the first chunk's rows 0..3 shifted by one
        yw = yy.clone()
        yw[8:] = yy[8:].roll(1)
        cw = O.t_embedder(sd64, t, torch.float64) + O.y_embedder(sd64, yw, torch.float64)
        _rejects(dt, "conditioning: another sample's label", got.double() + Fn.linear(Fn.silu(cw), w16, ab) - ref, ref, bnd)


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("D,heads", [(384, 6), (1152, 16), (1536, 24)])
@pytest.mark.parametrize("learn_sigma", [True, False], ids=["n_out32-tensor-core-head", "n_out16-final_layer_kernel"])
@pytest.mark.parametrize("extras", [1, 2])
def test_embedding_and_head(dev, dt, D, heads, learn_sigma, extras):
    """A depth-2 Latte whose gate_msa / gate_mlp adaLN rows are zero: both blocks add exactly 0 to the fp32 residual stream,
    so the output is patch_embed + pos_embed -> + temp_embed (block 0's fc2 epilogue) -> final LayerNorm + modulate ->
    head -> unpatchify, compared with the oracle's patch_embed / final_layer / unpatchify in fp64 on the shift / scale rows
    the kernels read (precompute_conditioning, bit-identical to the forward's) and the head weights they read (16-bit for
    the n_out = 32 tensor-core head, fp32 for final_layer_kernel)."""
    from oracle import latte_oracle as O
    chk = _chk(dt)
    cfg, sd, net = _latte(dev, dt, D, heads, extras, learn_sigma, seed=D + 2 * extras + learn_sigma, zero_gates=True)
    Bb, Fr, C, S, p = 2, cfg.num_frames, cfg.in_channels, cfg.input_size, cfg.patch_size
    g = torch.Generator(device=dev).manual_seed(D + extras)
    x = torch.randn(Bb, Fr, C, S, S, device=dev, generator=g)
    t = torch.tensor([999, 0], device=dev)
    y = torch.tensor([10, 4], device=dev) if extras == 2 else None
    with torch.no_grad():
        got = net(x, t, y=y)
    mod = net.precompute_conditioning(t[None], y)[0].double()
    _, _, T, _ = net._pack()
    net.clear_conditioning()
    N, K = cfg.num_patches, C * p * p
    mf = mod[:, 2 * 6 * D:]
    shift, scale = mf[:, :D].repeat_interleave(Fr, 0)[:, None], mf[:, D:].repeat_interleave(Fr, 0)[:, None]
    tc = sd["temp_embed"].double()[0].repeat(Bb, 1)[:, None]                     # [(b f), 1, D]
    sd64 = {k: v.double() for k, v in sd.items()}
    x64 = x.double()
    h = O.patch_embed(sd64, cfg, x64, torch.float64) + tc
    xp = x64.reshape(Bb * Fr, C, S // p, p, S // p, p).permute(0, 2, 4, 1, 3, 5).reshape(Bb * Fr, N, K)
    wp = sd64["x_embedder.proj.weight"].reshape(D, K)
    e_x = U32 * math.sqrt(K + 2) * (xp.abs() @ wp.abs().t() + sd64["x_embedder.proj.bias"].abs() + sd64["pos_embed"].abs() + tc.abs())
    mean = h.mean(-1, keepdim=True)
    rstd = (((h - mean) ** 2).mean(-1, keepdim=True) + 1e-6).rsqrt()
    xh = (h - mean) * rstd
    e_xh = rstd * (e_x + e_x.mean(-1, keepdim=True) + xh.abs() * (xh.abs() * e_x).mean(-1, keepdim=True)) + \
        U32 * (math.sqrt(D) * (rstd * h.abs().mean(-1, keepdim=True) + xh.abs()) + 3 * xh.abs())
    yv = xh * (1 + scale) + shift
    c1 = (1 + scale).abs()
    e_y = c1 * e_xh + U32 * (2 * xh.abs() * c1 + shift.abs())
    tensor_core = learn_sigma
    wf = (T["final_w16"] if tensor_core else T["final_w"]).double()
    bf = sd64["final_layer.linear.bias"]
    out = yv @ wf.t() + bf
    if tensor_core:
        e_y = e_y + U16[dt] * yv.abs()
    e_o = e_y @ wf.abs().t() + U32 * math.sqrt(D) * (yv.abs() @ wf.abs().t() + bf.abs())
    bnd = A * U32 * out.abs() + B * e_o
    if tensor_core and SUB[dt]:
        bnd = bnd + sqfloor(yv, wf.t(), SUB[dt])
    unp = lambda z: O.unpatchify(cfg, z).reshape(Bb, Fr, cfg.out_channels, S, S)     # noqa: E731
    ref, bnd = unp(out), unp(bnd)
    chk.add("embedding + head " + ("n_out=32 tensor-core" if tensor_core else "n_out=16 final_layer_kernel"),
            f"D={D} extras={extras}", got, ref, bnd,
            lambda i: f"sample {i[0]}, frame {i[1]}, channel {i[2]}, pixel ({i[3]}, {i[4]})")
    chk.done()
    wrong = got.reshape(Bb, Fr, cfg.out_channels, S // p, p, S // p, p).transpose(4, 6).reshape(got.shape)
    _rejects(dt, "unpatchify with the patch transposed", wrong, ref, bnd)


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("learn_sigma", [True, False])
def test_cfg_combine(dev, dt, learn_sigma):
    """forward_with_cfg on (x_half, x_half) == u + s (c - u) in fp32 on the halves of a plain forward of the same batch (so
    the same GEMM schedule), bit for bit on the guided eps channels; the other channels pass through unchanged."""
    _, _, net = _latte(dev, dt, 384, 6, 2, learn_sigma, seed=11)
    g = torch.Generator(device=dev).manual_seed(12)
    x = torch.randn(4, 4, 4, 16, 16, device=dev, generator=g)
    t = torch.tensor([999, 500, 999, 500], device=dev)
    y = torch.tensor([3, 7, 10, 10], device=dev)
    net.use_cuda_graphs = False
    s = 4.5
    with torch.no_grad():
        plain = net(torch.cat([x[:2], x[:2]]), t, y=y)
        guided = net.forward_with_cfg(x, t, y=y, cfg_scale=s)
    c, u = plain[:2, :, :4], plain[2:, :, :4]
    want = u + s * (c - u)
    assert torch.equal(guided[:2, :, :4], want), \
        f"max |diff| {float((guided[:2, :, :4] - want).abs().max()):.3g}, {int((guided[:2, :, :4] != want).sum())} elements differ"
    assert torch.equal(guided[2:, :, :4], want)
    assert torch.equal(guided[:, :, 4:], plain[:, :, 4:])
    fused = (u.double() + s * (c - u).double()).float()     # an fma: s * (c - u) not rounded before the add
    assert not torch.equal(fused, want), "this input does not tell an fma from the rounded product"
