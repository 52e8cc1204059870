"""The training GEMMs and the multi-tensor passes against fp64, element by element: `b200_wgrad` (both operands read
untransposed, fp32 reduce-add into dW scaled per column), `b200_dgrad` (W read in its [out, in] layout), fc1's
`b200_linear_gelu_both` (u and gelu(u) from one epilogue), the `NativeOps` routes around their shape rules, and
`b200_multi_cast` / `b200_multi_tensor` (operand casts, gradient norm, clipping, EMA).  Every GPU test is marked `gpu`; two
CPU tests check, through the host-only schedule dump, that each case of the tables below hits the schedule class it names
on a 132-SM H100, and each GPU test asserts the same at the device's own SM count before it computes anything.

The reference of each op is its expression in fp64 on the GPU, evaluated on the same 16-bit and fp32 tensors the kernel
reads, so the operands need no rounding term.  The kernels are called through the C ABI (`_lib`), except in the `NativeOps`
route tests.  Every output element must satisfy (tests/fp64_bounds.py, A = 2, B = 4, F = 3)

    |got - ref| <= A * u_out * |ref| + B * u_op * mag + floor

  * u_out: unit roundoff of the output (fp16 2^-11, bf16 2^-8, fp32 2^-24).  floor: one fp16 subnormal spacing (2^-24) for a
    16-bit fp16 output (at the training gradient scale 2^-20 every fp16 dgrad output is subnormal), 0 otherwise.
  * GEMM accumulation: u_op = ACC * sqrt(K) * 2^-24 on mag = |a| |w|^T (+ |bias|), ACC = 1 as in
    test_gpu_forward_ops_fp64.py, where it was measured for K-major operands up to K = 4608.  The transposed-operand modes
    run at K up to 64512 (the T2V caption K/V dgrad) and 20480 (wgrad at the XL/2 training shape), so
    `test_gemm_accumulation_transposed` measures the same ratio for mode 2 (dgrad) and mode 3 (wgrad) at K = 256, 4608,
    20480 and 65536 and holds it to B * ACC * sqrt(K).  On an H100 80GB HBM3 at a 700 W power limit, worst err / (2^-24 mag):

        K                        256     4608    20480   65536
        mode 2 fp16              6.82    12.3    16.8    27.7     / sqrt(K): 0.43  0.18  0.12  0.11
        mode 2 bf16              5.56    11.6    17.8    27.6     / sqrt(K): 0.35  0.17  0.12  0.11
        mode 3 fp16              12.3    31.8    59.6    108      / sqrt(K): 0.77  0.47  0.42  0.42
        mode 3 bf16              9.55    30.1    60.1    104      / sqrt(K): 0.60  0.44  0.42  0.41

    The ratio to sqrt(K) does not grow with K in either mode: it falls in mode 2, and in mode 3 it falls to 0.42 by
    K = 20480 and stays there up to 65536.  So the sqrt(K) form and ACC = 1 stand for the long-K training GEMMs too, with the
    worst case at a fifth of B * sqrt(K).  Mode 3 is measured as the forward file measures the K-major GEMM: dW = 0 +
    1 * (dY^T X), data-parallel, fp32 output.  Mode 2 has only a 16-bit output, whose rounding (2^-11 |ref|) would hide the
    accumulation error, so its input cancels exactly: the second half of the contraction repeats the first with W negated,
    ref = 0, and the output is the accumulation error itself, rounded with a relative error of 2^-11.
  * fp16-subnormal operands: at the training gradient scale 2^-20 every fp16 dY element is subnormal, and short-K GEMMs then
    leave the sqrt(K) model.  `test_wgrad_subnormal_operands` runs wgrad on such a dY and on the same 16-bit dY times 2^10,
    an exact rescale into the normal range (worst err / (2^-24 mag), and that / sqrt(K), same H100):

        K                        64      128     256     1024    4608    20480
        subnormal dY             90.3    47.5    31.1    25.9    58.5    168      / sqrt(K): 11.3  4.19  1.95  0.81  0.86  1.18
        same dY x 2^10           5.2     9.74    13.0    25.9    59.2    119      / sqrt(K): 0.65  0.86  0.81  0.81  0.87  0.83

    A wider run (three seeds; n_out x n_in = 512 x 384, 1152 x 256, 1152 x 1152) gave at most 112 (14.0 sqrt(K)) at K = 64,
    67 (5.9 sqrt(K)) at K = 128 and 3.4 sqrt(K) from K = 256 up for the subnormal dY, and 0.65 to 1.1 sqrt(K) for the
    rescaled one.

    The normal-range run follows the sqrt(K) model at every K, and in bf16 the two runs give the same bits, scaled.  So the
    excess comes from the tensor core's handling of fp16-subnormal operands, not from the kernel, whose arithmetic is the
    same in both runs.  It is largest at short K and falls below B sqrt(K) from K = 256 on.  The bound adds a constant,
    not a K-dependent term, for the products that have an fp16-subnormal operand (mag_sub = mag - |a_normal| |b_normal|):
    u_op mag gains SUB_ACC * 2^-24 * mag_sub with SUB_ACC = 32, which puts the worst short-K case at about 0.7 of the
    bound.  At K = 20480 the term adds 32 to sqrt(K) = 143.  At the training scale the bound still rejects dY's subnormals
    flushed to zero (all, or those below 2^-20) and a dropped quarter of K, for the 20480-row wgrads and the K = 64512
    caption K/V dgrad (asserted).
  * wgrad: dW = dW0 + c[col] * (dY^T X), fp32.  Per K-segment s of a tile the epilogue rounds c * partial once and
    reduce-adds it into dW once, so a tile cut into s segments (read per element from the schedule) carries
    ACC sqrt(K) |c| mag for the accumulation (the segments' sqrt(K_i) mag_i sum to at most sqrt(K) mag), |c| mag for the
    products and s adds of values below |dW0| + |c| mag:
    B u_op mag = B 2^-24 (ACC sqrt(K) |c| mag + SUB_ACC |c| mag_sub + s (|dW0| + |c| mag)).
  * dgrad: dX = dY W, 16-bit: the bias epilogue's bound without a bias, K = n_out.
  * gelu_both: u16 with the bias epilogue's bound.  a16 = gelu_tanh(u16) is checked against gelu_tanh in fp64 of the
    kernel's own u16 (the reference's autocast applies GELU to the rounded u), so only the epilogue's own error is left:
    tanh.approx.f32 (relative error 2^-11 of t = tanh(v)) times 0.5 |u|, and the four fp32 roundings of v = k0 (u + k1 u^3)
    times 0.5 |u| (1 - t^2) |v|, plus the output rounding and the fp16 floor.
  * multi_cast: bit for bit with `tensor.to(dtype)` (NaN equal to NaN).
  * multi_tensor SUMSQ: *accum += sum of src^2.  Each thread sums the squares of its float4s (or scalars) of
    ceil(total_chunks / blocks) chunks in fp32 -- at most 16 adds per chunk (the scalar path of an unaligned tensor) --
    then a 32-lane butterfly (5 fp32 adds) and an fp32 -> double block sum and atomic.  For a sum of positive terms each
    term passes through at most m = 1 (square) + 2 (float4 pairs) + L (the thread's adds) + 5 (warp) roundings, so
    |err| <= 1.01 m 2^-24 sum + 2^-53 per double add: a rigorous, linear bound.
  * multi_tensor SCALE: dst * coef in fp32, bit for bit.  AXPBY: a32 d + b32 f within three fp32 roundings of
    |a32 d| + |b32 f| (a32, b32 the fp32 values the kernel receives).

Every GEMM case runs in fp16 and bf16, with the gradient operand at the three scales of test_gpu_train_ops_fp64.py (1, 2^-20
and 2^-4).  Each op's bound is shown to reject a plausible wrong result built from the kernel's own output: a dropped
K-segment of a cut wgrad tile, col_scale applied per row, the last real row of a zero-padded wgrad left out, W read as W^T
in dgrad, GELU applied before the bias, and SUMSQ missing one entry or an unaligned tail.  One plausible wrong result is
not asserted: a16 computed from the unrounded accumulator instead of u16.  It moves gelu by at most |gelu'(u)| times
half a 16-bit spacing of u, that is |u gelu'(u)| u_out.  For u >= 0, |u gelu'(u)| <= 1.3 |gelu(u)|, inside
A u_out |gelu(u)|.  For -0.75 <= u < 0 the factor is at most 1.  Below -0.75, gelu(u) falls off faster than u gelu'(u) (the
factor is 9.6 at u = -3), but there |gelu'(u)| <= 0.13 and |t| >= 0.55, so the shift, at most 0.13 u_out |u|, stays below
the tanh.approx term B 0.5 |u| 2^-11 |t| >= 1.1 * 2^-11 |u| in fp16 and bf16.  So the bound cannot tell the two apart in
either dtype.  The worst err / bound of each op and dtype and the accumulation table are
printed at the end of the module (pytest -s)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from fp64_bounds import A, B, DTS, SUB, TANH_U, U16, U32, Checker, dtn, report_worst  # noqa: E402

ACC = 1.0                     # fp32 tensor-core accumulation: u_op = ACC * sqrt(K) * 2^-24 (measured, see the docstring)
SUB_ACC = 32.0                # extra u_op / 2^-24 of products with an fp16-subnormal operand (measured, see the docstring)
GELU_K0, GELU_K1 = 0.7978845608028654, 0.044715
SCALES = {"unit": 1.0, "train": 2.0 ** -20, "fp16-loss-scaled": 2.0 ** -20 * 2.0 ** 16}
EPI_BIAS, EPI_GATE_RESIDUAL = 0, 2
H100_SMS = 132

_WORST = {}
_ACC_TABLE = {}
_SUB_TABLE = {}


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    if _ACC_TABLE:
        print("\nfp32 accumulation with transposed operands: worst err / (2^-24 mag), and that / sqrt(K):")
        for (mode, dt, K), r in sorted(_ACC_TABLE.items()):
            print(f"  mode {mode} {dt:<9} K = {K:5d}   {r:8.3g}   {r / math.sqrt(K):8.3g}")
    if _SUB_TABLE:
        print("\nfp16 wgrad, dY at 2^-20 (all subnormal) and the same dY times 2^10 (normal): worst err / (2^-24 mag), / sqrt(K):")
        for K, (rs, rn) in sorted(_SUB_TABLE.items()):
            print(f"  K = {K:5d}   subnormal {rs:8.3g} {rs / math.sqrt(K):6.2f}   normal {rn:8.3g} {rn / math.sqrt(K):6.2f}")
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


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------ schedules
def _schedule(M, N, K, sms, wgrad):
    """(block_n, segments [n, 4] of (pair, tile, kb0, kb1)) of the GEMM dW[M=n_out, N=n_in] over K = rows (wgrad) or of a
    residual-epilogue b200_linear [M, N, K] (the transpose fallback of NativeOps.wgrad)."""
    from latte_b200 import _lib
    lib = _lib.load()
    bn = C.c_int()
    if wgrad:
        n = lib.b200_wgrad_schedule(K, M, N, sms, C.byref(bn), None, None, None, 0)
    else:
        n = lib.b200_gemm_schedule(M, N, K, EPI_GATE_RESIDUAL, 0, sms, C.byref(bn), None, None, None, 0)
    assert n > 0, _lib.last_error()
    seg = (C.c_int32 * (4 * n))()
    if wgrad:
        assert lib.b200_wgrad_schedule(K, M, N, sms, None, None, None, seg, n) == n
    else:
        assert lib.b200_gemm_schedule(M, N, K, EPI_GATE_RESIDUAL, 0, sms, None, None, None, seg, n) == n
    return bn.value, np.frombuffer(seg, dtype=np.int32).reshape(n, 4).copy()


def _tile_box(t, bn, M, N):
    """Rows and columns of the output covered by pair-tile t (two 128-row tiles of one bn-wide column block)."""
    num_n = (N + bn - 1) // bn
    r0, c0 = (t // num_n) * 256, (t % num_n) * bn
    return r0, min(M, r0 + 256), c0, min(N, c0 + bn)


def _segments_per_tile(seg):
    return np.bincount(seg[:, 1])


def _wgrad_class(rows, n_out, n_in, sms):
    """The schedule class of b200_wgrad with stream-K flags: data-parallel (no tile cut), two-segment stream-K, or a chain of
    more segments (with its length); and whether n_out is below one 128-row M tile (then every tile spans all of it)."""
    bn, seg = _schedule(n_out, n_in, rows, sms, True)
    s = int(_segments_per_tile(seg).max())
    cls = "data-parallel" if s == 1 else "stream-K 2" if s == 2 else f"chain {s}"
    if n_out < 128:
        assert len(_segments_per_tile(seg)) == (n_in + bn - 1) // bn
        cls += ", n_out < M tile"
    return cls


def _seg_map(M, N, K, sms, wgrad, dev):
    """Per output element: the number of K-segments its tile is cut into."""
    bn, seg = _schedule(M, N, K, sms, wgrad)
    s = torch.ones(M, N, dtype=torch.float64, device=dev)
    for t, n in enumerate(_segments_per_tile(seg)):
        if n > 1:
            r0, r1, c0, c1 = _tile_box(t, bn, M, N)
            s[r0:r1, c0:c1] = float(n)
    return s, bn, seg


# (name, rows, n_out, n_in, schedule class with stream-K flags on 132 SMs).  Every wgrad the engines send straight to
# b200_wgrad: S/2 and XL/2 at 20480 rows (5 samples x 16 frames x 256 tokens), tiny72's fc2, the output heads of
# patch 2, 4, 8 (n_out = p*p*8 or p*p*4, padded to 64), the p = 8 patch embed, LatteT2V's caption K/V and first caption
# projection, and the ABI's edges (n_out % 8 only; n_in = 1152: a half-wide last 256 tile).
WGRAD_CASES = [
    ("S/2 qkv", 20480, 1152, 384, "chain 8"), ("S/2 proj", 20480, 384, 384, "data-parallel"),
    ("S/2 fc1", 20480, 1536, 384, "chain 6"), ("S/2 fc2", 20480, 384, 1536, "chain 6"),
    ("XL/2 qkv", 20480, 3456, 1152, "stream-K 2"), ("XL/2 proj", 20480, 1152, 1152, "chain 4"),
    ("XL/2 fc1", 20480, 4608, 1152, "stream-K 2"), ("XL/2 fc2", 20480, 1152, 4608, "stream-K 2"),
    ("tiny72 fc2", 4096, 576, 2304, "data-parallel"),
    ("head 16", 20480, 16, 1152, "data-parallel, n_out < M tile"), ("head 32", 20480, 32, 1152, "data-parallel, n_out < M tile"),
    ("head 64", 20480, 64, 1152, "data-parallel, n_out < M tile"), ("head 128", 20480, 128, 1152, "data-parallel"),
    ("head 256", 20480, 256, 1152, "data-parallel"), ("head 512", 20480, 512, 1152, "chain 8"),
    ("patch p=8", 1280, 1152, 256, "data-parallel"),
    ("T2V kv", 256, 64512, 1152, "data-parallel"), ("T2V cap1", 256, 1152, 4096, "data-parallel"),
    ("edge n_out 8", 4096, 8, 1152, "data-parallel, n_out < M tile"), ("edge n_out 24", 4096, 24, 1152, "data-parallel, n_out < M tile"),
    ("edge n_out 40", 4096, 40, 1152, "data-parallel, n_out < M tile"),
]

# (name, rows, n_out, n_in): every dgrad of training.py / training_t2v.py (dX[rows, n_in] = dY[rows, n_out] W[n_out, n_in]),
# at ragged row counts; n_in = 384 and 1152 leave the last 256-wide tile half full.  b200_dgrad never streams along K.
DGRAD_CASES = [
    ("S/2 fc2", 20480, 384, 1536), ("S/2 fc1", 20480 + 37, 1536, 384), ("S/2 proj", 1001, 384, 384), ("S/2 qkv", 200, 1152, 384),
    ("XL/2 fc2", 20480, 1152, 4608), ("XL/2 fc1", 20480 + 37, 4608, 1152), ("XL/2 proj", 77, 1152, 1152),
    ("XL/2 qkv", 1001, 3456, 1152), ("head S/2", 20480, 64, 384), ("head XL/2", 20480 + 37, 64, 1152),
    ("T2V q2", 20480, 1152, 1152), ("T2V o2", 200, 1152, 1152), ("T2V cap2", 256, 1152, 1152), ("T2V cap2 64 rows", 64, 1152, 1152),
    ("T2V kv", 256, 64512, 1152), ("T2V kv 64 rows", 64, 64512, 1152),
]

# (name, M, N, K, zero rows at the end of A): training fc1 and the T2V caption projection (K = 4096, 256 rows of which the
# last 16 are padding); N = 1120 and 96 are 32 mod 64, so the last 64-column chunk of both outputs is half inside N.
GELU_CASES = [
    ("S/2 fc1", 20480, 1536, 384, 0), ("tiny72 fc1", 4096, 2304, 576, 0), ("XL/2 fc1", 20480, 4608, 1152, 0),
    ("T2V cap1", 256, 1152, 4096, 16), ("ragged XL/2 fc1", 1001, 4608, 1152, 0), ("N=1120", 77, 1120, 1152, 0),
    ("N=96", 200, 96, 384, 0),
]


@pytest.mark.parametrize("case", WGRAD_CASES, ids=lambda c: c[0])
def test_wgrad_schedule_classes(case):
    """CPU: each wgrad case hits the schedule class the table names on a 132-SM H100."""
    name, rows, n_out, n_in, want = case
    assert _wgrad_class(rows, n_out, n_in, H100_SMS) == want


def test_dgrad_and_gelu_schedules_are_data_parallel():
    """CPU: the dgrad and gelu_both cases are data-parallel (16-bit epilogues never stream along K)."""
    from latte_b200 import _lib
    lib = _lib.load()
    sk = C.c_int()
    for _, M, K, N in DGRAD_CASES:
        assert lib.b200_gemm_schedule(M, N, K, EPI_BIAS, 0, H100_SMS, None, None, C.byref(sk), None, 0) > 0 and sk.value == 0
    for _, M, N, K, _ in GELU_CASES:
        assert lib.b200_gemm_schedule(M, N, K, EPI_BIAS, 0, H100_SMS, None, None, C.byref(sk), None, 0) > 0 and sk.value == 0


# ------------------------------------------------------------------------------------------------ inputs
def _outliers(x, g, per_row=3, value=60.0):
    M, K = x.shape
    cols = torch.randint(0, K, (M, per_row), device=x.device, generator=g)
    sign = torch.randint(0, 2, (M, per_row), device=x.device, generator=g).to(x.dtype) * 2 - 1
    x.scatter_(1, cols, value * sign)
    return x


def _xavier(g, dev, n_out, n_in):
    """Xavier-uniform [n_out, n_in] with a block of 32 output rows at the adaLN-Zero scale (1e-4)."""
    lim = math.sqrt(6.0 / (n_out + n_in))
    w = (torch.rand(n_out, n_in, device=dev, generator=g) * 2 - 1) * lim
    w[n_out // 2:n_out // 2 + 32] *= 1e-4 / lim
    return w


def _grad(g, dev, rows, n, s, dt):
    """An upstream gradient at scale s: randn rows spread over two decades, and a block of columns 1000x smaller."""
    d = torch.randn(rows, n, device=dev, generator=g) * torch.logspace(-1, 1, rows, device=dev)[torch.rand(rows, device=dev, generator=g).argsort()][:, None]
    d[:, n // 3:n // 3 + 8] *= 1e-3
    return (d * s).to(dt)


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ------------------------------------------------------------------------------------------------ wgrad
def _wgrad_into(dW, dy, x, cs, sk):
    from latte_b200 import _lib, ops
    rows, n_out = dy.shape
    rc = _lib.load().b200_wgrad(dy.data_ptr(), x.data_ptr(), cs.data_ptr(), dW.data_ptr(), rows, n_out, x.shape[1], ops._dt(dy),
                                ops._sk_flags(dy.device).data_ptr() if sk else None, _stream())
    _lib.check(rc, "b200_wgrad")


def _sub_mag(a64, b64, mag, dt, lhs_t=False):
    """The part of mag = |a| |b| made of products with an fp16-subnormal operand (0 in bf16)."""
    if dt != torch.float16:
        return 0.0
    an, bn = a64.abs() * (a64.abs() >= 2.0 ** -14), b64.abs() * (b64.abs() >= 2.0 ** -14)
    return mag - ((an.t() if lhs_t else an) @ bn)


def _wgrad_bound(ref, dW0, cs, mag, K, segs, mag_sub=0.0):
    return A * U32 * ref.abs() + B * U32 * (ACC * math.sqrt(K) * cs.abs() * mag + SUB_ACC * cs.abs() * mag_sub
                                            + segs * (dW0.abs() + cs.abs() * mag))


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("case", WGRAD_CASES, ids=lambda c: c[0])
def test_wgrad(dev, dt, case):
    """dW (fp32, 16 guard rows behind it) = dW0 + c[col] * (dY^T X) through the C ABI, with stream-K flags and without
    (data-parallel), c all ones, a power-of-two loss scale, and random per-column values with zeros; the flagged run repeats
    bit for bit.  At 20480 rows and the training scale 2^-20 the bound must reject dY's fp16 subnormals flushed to zero (all
    of them, or those below 2^-20) and a dropped quarter of the K range."""
    name, rows, n_out, n_in, want = case
    sms = _sms()
    if sms == H100_SMS:     # the table's classes are those of a 132-SM H100; elsewhere the bounds follow the device's own schedule
        assert _wgrad_class(rows, n_out, n_in, sms) == want
    chk = _chk(dt)
    segs, bn, seg = _seg_map(n_out, n_in, rows, sms, True, dev)
    g = torch.Generator(device=dev).manual_seed(rows + 7 * n_out + 13 * n_in)
    x = _outliers(torch.randn(rows, n_in, device=dev, generator=g), g).to(dt)
    x64 = x.double()
    crand = torch.rand(n_in, device=dev, generator=g) * 2
    crand[::7] = 0
    col_scales = {"ones": torch.ones(n_in, device=dev), "2^-16": torch.full((n_in,), 2.0 ** -16, device=dev), "random": crand}
    for sname, s in SCALES.items():
        dy = _grad(g, dev, rows, n_out, s, dt)
        dy64 = dy.double()
        P = dy64.t() @ x64
        mag = dy64.abs().t() @ x64.abs()
        msub = _sub_mag(dy64, x64, mag, dt, True)
        buf0 = torch.randn(n_out + 16, n_in, device=dev, generator=g) * s
        dW0 = buf0[:n_out].double()
        for cname, cs in col_scales.items():
            c64 = cs.double()
            ref = dW0 + c64 * P
            for sk in (True, False):
                buf = buf0.clone()
                _wgrad_into(buf[:n_out], dy, x, cs, sk)
                torch.cuda.synchronize()
                assert torch.equal(buf[n_out:], buf0[n_out:]), f"{name}: guard rows behind dW written"
                bnd = _wgrad_bound(ref, dW0, c64, mag, rows, segs if sk else 1.0, msub)
                chk.add("wgrad", f"{name} {sname} col_scale={cname} stream-K={sk}", buf[:n_out], ref, bnd, _rc)
                if sk and cname == "random":
                    again = buf0.clone()
                    _wgrad_into(again[:n_out], dy, x, cs, True)
                    assert torch.equal(again, buf), f"{name}: the stream-K result is not bit-reproducible"
                    got_rand, bnd_rand, ref_rand = buf[:n_out].double(), bnd, ref
                if sk and cname == "ones":
                    got_ones, bnd_ones, ref_ones = buf[:n_out].double(), bnd, ref
            del ref
        chk.done()

        if sname == "train" and rows >= 20480:
            _long_k_rejections(dt, "wgrad", got_ones, ref_ones, bnd_ones, dy64, lambda d, k: d[k].t() @ x64[k], rows)
        if sname != "unit":
            continue
        # a dropped K-segment: the last segment of the most-cut tile
        counts = _segments_per_tile(seg)
        if counts.max() > 1:
            t = int(np.argmax(counts))
            _, _, kb0, kb1 = max((tuple(r) for r in seg if r[1] == t), key=lambda r: r[2])
            r0, r1, c0, c1 = _tile_box(t, bn, n_out, n_in)
            k0, k1 = kb0 * 64, kb1 * 64
            wrong = got_ones.clone()
            wrong[r0:r1, c0:c1] -= dy64[k0:k1, r0:r1].t() @ x64[k0:k1, c0:c1]
            _rejects(dt, f"wgrad: K-segment [{kb0}, {kb1}) of tile {t} dropped", wrong, ref_ones, bnd_ones)
        # col_scale applied per output row instead of per column
        if n_out == n_in:
            c64 = crand.double()
            wrong = got_rand + (c64[:, None] - c64[None, :]) * P
            _rejects(dt, "wgrad: col_scale applied per row", wrong, ref_rand, bnd_rand)
        del got_ones, got_rand


def _long_k_rejections(dt, op, got, ref, bnd, dy64, prod, K):
    """At the training scale: the bound rejects dY's fp16 subnormals flushed to zero, all of them or those below 2^-20
    (fp16 only: bf16 has no subnormals there), and a dropped quarter of the K range.  prod(d, k) is the GEMM with d in
    place of dY over the contraction indices k; wrong results are rounded like the kernel's output."""
    out = got.dtype if got.dtype != torch.float32 else torch.float64
    every = slice(None)
    if dt == torch.float16:
        for below in (2.0 ** -14, 2.0 ** -20):
            part = dy64 * (dy64.abs() < below)       # the products a flushing kernel would lose
            _rejects(dt, f"{op}: dY subnormals below {below:g} flushed", (got.double() - prod(part, every)).to(out), ref, bnd)
    q = slice(K // 4, K // 2)
    _rejects(dt, f"{op}: contraction indices [{q.start}, {q.stop}) dropped", (got.double() - prod(dy64, q)).to(out), ref, bnd)


# ------------------------------------------------------------------------------------------------ dgrad
def _dgrad_into(dx, dy, w):
    from latte_b200 import _lib, ops
    rows, n_out = dy.shape
    rc = _lib.load().b200_dgrad(dy.data_ptr(), w.data_ptr(), dx.data_ptr(), rows, n_out, w.shape[1], ops._dt(dy), _stream())
    _lib.check(rc, "b200_dgrad")


def _gemm16_bound(ref, mag, K, dt, mag_sub=0.0):
    return A * U16[dt] * ref.abs() + B * U32 * (ACC * math.sqrt(K) * mag + SUB_ACC * mag_sub) + SUB[dt]


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("case", DGRAD_CASES, ids=lambda c: c[0])
def test_dgrad(dev, dt, case):
    """dX (16-bit, 16 guard rows behind it) = dY W with W in its [out, in] layout, at three gradient scales.  For the T2V
    caption K/V (K = 64512) at the training scale the bound must reject flushed fp16 subnormals and a dropped quarter of K."""
    from latte_b200 import _lib
    name, rows, n_out, n_in = case
    sk = C.c_int()
    assert _lib.load().b200_gemm_schedule(rows, n_in, n_out, EPI_BIAS, 0, _sms(), None, None, C.byref(sk), None, 0) > 0
    assert sk.value == 0
    chk = _chk(dt)
    g = torch.Generator(device=dev).manual_seed(rows + 3 * n_out + 11 * n_in)
    w = _xavier(g, dev, n_out, n_in).to(dt)
    w64 = w.double()
    for sname, s in SCALES.items():
        dy = _grad(g, dev, rows, n_out, s, dt)
        dy64 = dy.double()
        ref = dy64 @ w64
        mag = dy64.abs() @ w64.abs()
        bnd = _gemm16_bound(ref, mag, n_out, dt, _sub_mag(dy64, w64, mag, dt))
        del mag
        buf0 = torch.randn(rows + 16, n_in, device=dev, generator=g).to(dt)
        buf = buf0.clone()
        _dgrad_into(buf[:rows], dy, w)
        torch.cuda.synchronize()
        assert torch.equal(buf[rows:], buf0[rows:]), f"{name}: guard rows behind dX written"
        chk.add("dgrad", f"{name} {sname}", buf[:rows], ref, bnd, _rc)
        if n_out == n_in and sname == "unit":        # W read as W^T
            _rejects(dt, "dgrad: W read transposed", (buf[:rows].double() + dy64 @ w64.t() - ref).to(dt), ref, bnd)
        if n_out == 64512 and sname == "train":      # the T2V caption K/V: the longest K
            _long_k_rejections(dt, "dgrad", buf[:rows], ref, bnd, dy64, lambda d, k: d[:, k] @ w64[k], n_out)
        del ref, bnd, dy64
    chk.done()


# ------------------------------------------------------------------------------------------------ linear_gelu_both
def _gelu_both_into(u, act, a, w, bias):
    from latte_b200 import _lib, ops
    M, K = a.shape
    rc = _lib.load().b200_linear_gelu_both(a.data_ptr(), w.data_ptr(), bias.data_ptr() if bias is not None else None, M, w.shape[0],
                                           K, ops._dt(a), u.data_ptr(), act.data_ptr(), _stream())
    _lib.check(rc, "b200_linear_gelu_both")


def _gelu64(u):
    return 0.5 * u * (1 + torch.tanh(GELU_K0 * (u + GELU_K1 * u ** 3)))


def _gelu_bound(u, dt):
    """Bound of a16 against gelu_tanh(u) in fp64 of the kernel's u16 (see the module docstring)."""
    v = GELU_K0 * (u + GELU_K1 * u ** 3)
    t = torch.tanh(v)
    ref = 0.5 * u * (1 + t)
    return ref, A * U16[dt] * ref.abs() + B * 0.5 * u.abs() * (TANH_U * t.abs() + 4 * U32 * v.abs() * (1 - t * t)) + SUB[dt]


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("case", GELU_CASES, ids=lambda c: c[0])
def test_linear_gelu_both(dev, dt, case):
    """u16 = a w^T + bias and a16 = gelu_tanh(u16) from one epilogue, with a bias and with bias = NULL; 16 guard rows behind
    both outputs.  Activations carry three +-60 outliers per row; a block of 32 weight rows (and their biases) is 1e-4."""
    name, M, N, K, pad = case
    chk = _chk(dt)
    g = torch.Generator(device=dev).manual_seed(M + N + K)
    a = _outliers(torch.randn(M, K, device=dev, generator=g), g)
    if pad:
        a[M - pad:] = 0
    a = a.to(dt)
    w = _xavier(g, dev, N, K).to(dt)
    bias = torch.randn(N, device=dev, generator=g) * 0.5
    bias[N // 2:N // 2 + 32] *= 1e-4
    a64, w64 = a.double(), w.double()
    acc = a64 @ w64.t()
    amag = a64.abs() @ w64.abs().t()
    del a64, w64
    for with_bias in (True, False):
        b64 = bias.double() if with_bias else torch.zeros(N, dtype=torch.float64, device=dev)
        pre = acc + b64
        bnd_u = _gemm16_bound(pre, amag + b64.abs(), K, dt)
        u0 = torch.randn(M + 16, N, device=dev, generator=g).to(dt)
        act0 = torch.randn(M + 16, N, device=dev, generator=g).to(dt)
        u, act = u0.clone(), act0.clone()
        _gelu_both_into(u[:M], act[:M], a, w, bias if with_bias else None)
        torch.cuda.synchronize()
        assert torch.equal(u[M:], u0[M:]) and torch.equal(act[M:], act0[M:]), f"{name}: guard rows written"
        tag = f"{name} bias={with_bias}"
        chk.add("gelu_both u16", tag, u[:M], pre, bnd_u, _rc)
        ref_a, bnd_a = _gelu_bound(u[:M].double(), dt)
        chk.add("gelu_both a16", tag, act[:M], ref_a, bnd_a, _rc)
        if with_bias:       # GELU applied before the bias: gelu(u - b) + b
            u64 = u[:M].double()
            late = _gelu64(u64 - b64) + b64
            _rejects(dt, "gelu_both: GELU applied before the bias", (act[:M].double() + late - ref_a).to(dt), ref_a, bnd_a)
        del pre, bnd_u, ref_a, bnd_a
    chk.done()


# ------------------------------------------------------------------------------------------------ accumulation table
@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTS)
def test_gemm_accumulation_transposed(dev, dt):
    """The fp32 accumulation of the transposed-operand modes alone, at K = 256, 4608, 20480 and 65536 (see the docstring):
    mode 3, dW = 0 + 1 * (dY^T X) data-parallel, n_out = n_in = 1152, three +-60 outliers per row of X; mode 2, dX = dY W at
    4096 x 1152 whose second K half repeats the first with W negated (ref = 0).  Records worst err / (2^-24 mag) per mode, dtype
    and K and holds it to B * ACC * sqrt(K)."""
    chk = _chk(dt)
    for K in (256, 4608, 20480, 65536):
        g = torch.Generator(device=dev).manual_seed(K)
        # mode 3
        dy = torch.randn(K, 1152, device=dev, generator=g).to(dt)
        x = _outliers(torch.randn(K, 1152, device=dev, generator=g), g).to(dt)
        dW = torch.zeros(1152, 1152, device=dev)
        _wgrad_into(dW, dy, x, torch.ones(1152, device=dev), False)
        dy64, x64 = dy.double(), x.double()
        ref = dy64.t() @ x64
        mag = dy64.abs().t() @ x64.abs()
        del dy64, x64, dy, x
        _ACC_TABLE[(3, dtn(dt), K)] = float(((dW.double() - ref).abs() / (U32 * mag)).max())
        chk.add("wgrad fp32 accumulation", f"K={K}", dW, ref, A * U32 * ref.abs() + B * ACC * math.sqrt(K) * U32 * mag, _rc)
        del ref, mag, dW
        # mode 2
        h = K // 2
        dyh = _outliers(torch.randn(4096, h, device=dev, generator=g), g).to(dt)
        wh = _xavier(g, dev, h, 1152).to(dt)
        dy, w = torch.cat([dyh, dyh], 1), torch.cat([wh, -wh], 0)
        dx = torch.empty(4096, 1152, dtype=dt, device=dev)
        _dgrad_into(dx, dy, w)
        mag = 2 * (dyh.double().abs() @ wh.double().abs())
        del dy, w, dyh, wh
        ref = torch.zeros_like(mag)
        _ACC_TABLE[(2, dtn(dt), K)] = float((dx.double().abs() / (U32 * mag)).max())
        chk.add("dgrad fp32 accumulation", f"K={K}", dx, ref, B * ACC * math.sqrt(K) * U32 * mag + SUB[dt], _rc)
        del mag, ref, dx
    chk.done()


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTS)
def test_wgrad_subnormal_operands(dev, dt):
    """Where the fp16-subnormal term comes from: wgrad (n_out 1152, n_in 256, data-parallel) with dY at the training scale
    2^-20 (every fp16 element subnormal) and with the same 16-bit dY times 2^10, an exact rescale into the normal range, at
    K = 64 ... 20480.  In bf16 (no subnormals at 2^-20) the two results are the same bits, scaled: the kernel's arithmetic is
    scale-invariant.  In fp16 the normal-range run must stay within B * ACC * sqrt(K) and the subnormal run within
    B * (ACC * sqrt(K) + SUB_ACC); both ratios are recorded and printed."""
    chk = _chk(dt)
    n_out, n_in = 1152, 256
    for K in (64, 128, 256, 1024, 4608, 20480):
        g = torch.Generator(device=dev).manual_seed(K + 1)
        x = _outliers(torch.randn(K, n_in, device=dev, generator=g), g).to(dt)
        dys = _grad(g, dev, K, n_out, 2.0 ** -20, dt)
        dyn = dys * 2.0 ** 10
        assert torch.equal(dyn * 2.0 ** -10, dys)
        ones = torch.ones(n_in, device=dev)
        got_s, got_n = torch.zeros(n_out, n_in, device=dev), torch.zeros(n_out, n_in, device=dev)
        _wgrad_into(got_s, dys, x, ones, False)
        _wgrad_into(got_n, dyn, x, ones, False)
        if dt == torch.bfloat16:
            assert torch.equal(got_n * 2.0 ** -10, got_s), f"K={K}: bf16 wgrad is not invariant under an exact 2^10 rescale"
            continue
        x64 = x.double()
        ratios = []
        for dy, got, sub in ((dys, got_s, SUB_ACC), (dyn, got_n, 0.0)):
            dy64 = dy.double()
            ref, mag = dy64.t() @ x64, dy64.abs().t() @ x64.abs()
            ratios.append(float(((got.double() - ref).abs() / (U32 * mag).clamp_min(1e-300)).max()))
            chk.add("wgrad fp16 " + ("subnormal dY" if sub else "dY x 2^10"), f"K={K}", got, ref,
                    A * U32 * ref.abs() + B * U32 * (ACC * math.sqrt(K) + sub) * mag, _rc)
        _SUB_TABLE[K] = tuple(ratios)
    chk.done()


# ------------------------------------------------------------------------------------------------ NativeOps routes
# (name, rows, n_out, n_in): rows % 64 != 0 (tokens at patch 4 and 8: 16 and 4 per frame) are zero-padded; n_in % 128 != 0
# (the patch embed at p = 2 and 4, K = C p p padded to 64, and tiny72's n_in = 576 weights) goes through two transposes and
# linear_accum.
NATIVE_WGRAD = [("head p=4", 3 * 7 * 16, 128, 384), ("head p=8", 5 * 3 * 4, 512, 384), ("patch p=4", 3 * 7 * 16, 384, 64),
                ("patch p=8", 5 * 3 * 4, 1152, 256), ("patch p=2", 2048, 1152, 64), ("tiny72 fc1", 4096, 2304, 576),
                ("tiny72 proj", 4096, 576, 576)]


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("case", NATIVE_WGRAD, ids=lambda c: c[0])
def test_native_wgrad_routes(dev, dt, case):
    from latte_b200.train_ops import NativeOps
    name, rows, n_out, n_in = case
    nat, chk = NativeOps(dt), _chk(dt)
    kp = -(-rows // 64) * 64
    direct = n_in % 128 == 0
    segs, _, _ = _seg_map(n_out, n_in, kp, _sms(), direct, dev)
    g = torch.Generator(device=dev).manual_seed(rows + n_out + n_in)
    x = _outliers(torch.randn(rows, n_in, device=dev, generator=g), g).to(dt)
    x64 = x.double()
    ones = torch.ones(n_in, dtype=torch.float64, device=dev)
    for sname, s in SCALES.items():
        dy = _grad(g, dev, rows, n_out, s, dt)
        dy64 = dy.double()
        dW0 = torch.randn(n_out, n_in, device=dev, generator=g) * s
        ref = dW0.double() + dy64.t() @ x64
        mag = dy64.abs().t() @ x64.abs()
        bnd = _wgrad_bound(ref, dW0.double(), ones, mag, kp, segs, _sub_mag(dy64, x64, mag, dt, True))
        got = nat.wgrad(dW0.clone(), dy, x)
        chk.add("NativeOps.wgrad " + ("padded rows" if direct else "transposed"), f"{name} {sname}", got, ref, bnd, _rc)
        if rows % 64 and sname == "unit":       # the last real row left out
            wrong = got.double() - dy64[-1][:, None] * x64[-1][None, :]
            _rejects(dt, "NativeOps.wgrad: last real row dropped", wrong, ref, bnd)
    chk.done()


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("rows,n_out", [(4096, 2304), (1001, 1728), (200, 576)], ids=["tiny72 fc1", "tiny72 qkv", "tiny72 proj"])
def test_native_dgrad_transposed(dev, dt, rows, n_out):
    """dgrad with n_in = 576 (tiny72): W^T through b200_transpose16, then the forward GEMM."""
    from latte_b200.train_ops import NativeOps
    nat, chk = NativeOps(dt), _chk(dt)
    g = torch.Generator(device=dev).manual_seed(rows + n_out)
    w = _xavier(g, dev, n_out, 576).to(dt)
    w64 = w.double()
    for sname, s in SCALES.items():
        dy = _grad(g, dev, rows, n_out, s, dt)
        dy64 = dy.double()
        ref = dy64 @ w64
        mag = dy64.abs() @ w64.abs()
        chk.add("NativeOps.dgrad transposed", f"rows={rows} n_out={n_out} {sname}", nat.dgrad(dy, w), ref,
                _gemm16_bound(ref, mag, n_out, dt, _sub_mag(dy64, w64, mag, dt)), _rc)
    chk.done()


# ------------------------------------------------------------------------------------------------ multi_cast
def _multi_cast(table, n, total, like):
    from latte_b200 import _lib, ops
    _lib.check(_lib.load().b200_multi_cast(table.data_ptr(), n, total, ops._dt(like), _stream()), "b200_multi_cast")


def _specials(dev):
    f32 = np.float32
    vals = [0.0, -0.0, 2.0 ** -24, -2.0 ** -24, 2.0 ** -25, 3 * 2.0 ** -25, 5 * 2.0 ** -25, 2.0 ** -14 - 2.0 ** -24, 6.1e-5,
            2.0 ** -130, -3 * 2.0 ** -133, 2.0 ** -149, 1.17e-38,
            1 + 2.0 ** -11, 1 + 3 * 2.0 ** -11, 1 + 2.0 ** -8, 1 + 3 * 2.0 ** -8, -(1 + 3 * 2.0 ** -8), 1 + 2.0 ** -8 + 2.0 ** -20,
            65504.0, float(f32(65519.99)), 65520.0, -65520.0, 1e30, -1e30, 3.4028234e38, math.inf, -math.inf, math.nan]
    return torch.tensor(vals, dtype=torch.float32, device=dev)


def _bad_bits(a, b):
    """Elements of two 16-bit tensors whose bits differ, NaN equal to NaN."""
    return (a.view(torch.int16) != b.view(torch.int16)) & ~(torch.isnan(a) & torch.isnan(b))


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTS)
def test_multi_cast(dev, dt):
    """One launch over entries of n4 = 1, 1023, 1024, 1025 and 1100 * 1024 float4 (total chunks above the launcher's 1056
    blocks: the grid stride and the binary search cross entry boundaries), each starting with the special values (+-0,
    fp16 and bf16 subnormals, exact ties, 65504 / 65519.99 / 65520, 1e30, +-inf, NaN); dst ranges share one buffer with gaps
    of 12 sentinel elements, which must stay untouched."""
    g = torch.Generator(device=dev).manual_seed(5)
    sp = _specials(dev)
    srcs, rows, first, off = [], [], 0, 12
    dst = torch.full((12 + sum(4 * n + 12 for n in (1, 1023, 1024, 1025, 1100 * 1024)),), 0.0, dtype=dt, device=dev)
    dst.view(torch.int16).fill_(0x5a5a)
    sentinel = dst.clone()
    offs = []
    for n4 in (1, 1023, 1024, 1025, 1100 * 1024):
        src = torch.randn(4 * n4, device=dev, generator=g) * 3
        k = min(4 * n4, sp.numel())
        src[:k] = sp[:k]
        src[-k:] = sp[:k].flip(0)
        srcs.append(src)
        rows.append([src.data_ptr(), dst[off:].data_ptr(), n4, first])
        offs.append(off)
        first += (n4 + 1023) // 1024
        off += 4 * n4 + 12
    assert first > 1056
    table = torch.tensor(rows, dtype=torch.int64).to(dev)
    _multi_cast(table, len(rows), first, dst)
    torch.cuda.synchronize()
    mask = torch.ones_like(dst, dtype=torch.bool)
    for src, o in zip(srcs, offs):
        got = dst[o:o + src.numel()]
        want = src.to(dt)
        bad = _bad_bits(got, want)
        assert not bad.any(), f"multi_cast {dtn(dt)}: {int(bad.sum())} of {src.numel()} elements differ, e.g. " \
            f"{src[bad][:4].tolist()} -> {got[bad][:4].tolist()}, want {want[bad][:4].tolist()}"
        mask[o:o + src.numel()] = False
    assert torch.equal(dst.view(torch.int16)[mask], sentinel.view(torch.int16)[mask]), "multi_cast wrote into a gap between entries"


# ------------------------------------------------------------------------------------------------ multi_tensor
def _mt_table(dev, srcs, dsts):
    rows, first = [], 0
    for a, b in zip(srcs, dsts):
        t = a if a is not None else b
        rows.append([a.data_ptr() if a is not None else 0, b.data_ptr() if b is not None else 0, t.numel(), first])
        first += (t.numel() + 4095) // 4096
    return torch.tensor(rows, dtype=torch.int64).to(dev), len(rows), first


def _mt(op, table, n, total, a=0.0, b=0.0, scalar=None, accum=None):
    from latte_b200 import _lib
    rc = _lib.load().b200_multi_tensor(table.data_ptr(), n, total, op, a, b, scalar.data_ptr() if scalar is not None else None,
                                       accum.data_ptr() if accum is not None else None, _stream())
    _lib.check(rc, "b200_multi_tensor")


def _mt_tensors(dev, g):
    """Entries: aligned n = 4096 * 3 + 5 (a tail of 1), an unaligned view (n = 10001, scalar path), an empty entry between two
    others, n = 7 whose 3 tail elements are 1000, and one of 1100 chunks (more chunks than the launcher's 1056 blocks)."""
    base = torch.randn(10001 + 4, device=dev, generator=g)
    tail = torch.randn(7, device=dev, generator=g)
    tail[4:] = 1000.0
    ts = [torch.randn(4096 * 3 + 5, device=dev, generator=g), base[1:10002], torch.empty(0, device=dev), tail,
          torch.randn(1100 * 4096, device=dev, generator=g) * 0.5, torch.randn(3, device=dev, generator=g)]
    assert ts[1].data_ptr() % 16 == 4
    return ts, base


@pytest.mark.gpu
def test_multi_tensor(dev):
    """SUMSQ against the fp64 sum of squares added to a nonzero accumulator, with the kernel's own linear bound; SCALE bit for
    bit; AXPBY within three fp32 roundings.  The bound must reject SUMSQ without one entry, or without the tail of the entry
    whose last three elements are 1000."""
    chk = Checker(torch.float32, _WORST)
    g = torch.Generator(device=dev).manual_seed(9)
    ts, base = _mt_tensors(dev, g)
    table, n, total = _mt_table(dev, ts, [None] * len(ts))
    blocks = min(total, 132 * 8)
    m = math.ceil(total / blocks) * 16 + 8                      # roundings a term can pass through (see the docstring)
    acc0 = 12345.678
    accum = torch.full((1,), acc0, dtype=torch.float64, device=dev)
    _mt(1, table, n, total, accum=accum)
    parts = [float((t.double() ** 2).sum()) if t.numel() else 0.0 for t in ts]
    ref = acc0 + sum(parts)

    def bound(r):
        return torch.tensor([1.01 * m * U32 * (r - acc0) + 2 * (blocks + 8) * 2.0 ** -53 * r], dtype=torch.float64, device=dev)
    refs = torch.tensor([ref], dtype=torch.float64, device=dev)
    chk.add("multi_tensor SUMSQ", f"{total} chunks", accum, refs, bound(ref), lambda i: "accum")
    chk.done()
    _rejects(torch.float32, "SUMSQ missing an entry", accum - parts[0], refs, bound(ref))
    _rejects(torch.float32, "SUMSQ missing an unaligned tail", accum - 3e6, refs, bound(ref))

    # SCALE: dst *= coef, in place, on the same entries (the unaligned view sits inside `base`)
    coef = torch.tensor([0.3712345], device=dev)
    before = [t.clone() for t in ts]
    base0 = base.clone()
    table, n, total = _mt_table(dev, [None] * len(ts), ts)
    _mt(2, table, n, total, scalar=coef)
    for t, t0 in zip(ts, before):
        assert torch.equal(t, t0 * coef), "multi_tensor SCALE is not bit-exact"
    assert base[0] == base0[0] and torch.equal(base[10002:], base0[10002:]), "SCALE wrote outside the unaligned view"

    # AXPBY: dst = a dst + b src (EMA)
    a32, b32 = float(np.float32(0.9999)), float(np.float32(1 - 0.9999))
    srcs = [torch.randn(t.shape, device=dev, generator=g) for t in ts]
    before = [t.clone() for t in ts]
    table, n, total = _mt_table(dev, srcs, ts)
    _mt(3, table, n, total, a=a32, b=b32)
    for t, t0, f in zip(ts, before, srcs):
        if t.numel():
            r = a32 * t0.double() + b32 * f.double()
            chk.add("multi_tensor AXPBY", f"n={t.numel()}", t, r, 3 * U32 * ((a32 * t0.double()).abs() + (b32 * f.double()).abs()),
                    lambda i: f"element {i[0]}")
    chk.done()
