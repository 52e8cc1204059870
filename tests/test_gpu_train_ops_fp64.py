"""GPU: every backward kernel of csrc/train.cu against fp64 autograd, element by element.

The reference of each op is torch autograd, in fp64 on the GPU, of the op's FORWARD expression evaluated on the same 16-bit
(and fp32) tensors the kernel reads; none of the hand-derived backward formulas the kernels share is used.  Each output
element must satisfy

    |got - ref| <= A * u_out * |ref| + B * u_op * mag + floor

  * u_out: unit roundoff of the output (fp16 2^-11, bf16 2^-8, fp32 2^-24).
  * u_op * mag: the forward error of the computation.  `mag` is the same fp64 computation on absolute values (|P| |dP - delta|
    and its products for the softmax backward).  u_op is the roundoff of the operand that is rounded on the way: 2^-11 / 2^-8
    where a 16-bit intermediate is formed (P and dS before the tensor-core products, dmod before the adaLN GEMM), 2^-11 for
    tanh.approx in the GELU derivative, and sqrt(n) * 2^-24 for an fp32 reduction of n terms (the probabilistic bound of
    Higham & Mary: rounding errors of a long sum grow like sqrt(n), not n).  In the softmax, u_op of a row also carries
    2 * 2^-24 * log2(e) * max|score|: the fp32 log-sum-exp offset of a row with +-30 logits or a -10000 mask bias.
    LayerNorm multiplies its fp32 term by 1 + rstd * mean|x| (a row with a large mean and a small spread loses digits in the
    mean).
  * floor: 0 in bf16.  In fp16, 2^-24 (one subnormal spacing) for the 16-bit output, plus, for every 16-bit intermediate of a
    product, F * sqrt(sum over the n terms of (min(2^-24, |operand|) * |other factor|)^2): each subnormal operand is off by at
    most half a spacing and those errors are independent, so their sum grows like sqrt(n); F = 3 puts the floor at about
    10 standard deviations of that sum (uniform errors), so outputs of 2 * 10^8 elements stay below it.  A floor linear in n
    (the worst case) would be as large as the gradient itself at the training scale and would not notice a kernel whose
    rounding is several times coarser -- e.g. one that puts the softmax scale hd^-1/2 onto the fp16 dS (8x coarser
    subnormal steps).

A = 2, B = 4, F = 3.  Every op runs in fp16 and bf16 at three scales of its upstream gradient: unit, the training step's (2^-20,
about 1e-6: a mean loss over F*C*H*W per sample and over the batch) and that times 2^16 (fp16 loss scaling).  Attention
inputs include peaked rows (logits +-30), a row whose maximum is the last key, a constant row (q = 0) and upstream-gradient
rows spread over 2.6 decades.  Failures report the worst err / bound and where it sits; the worst ratio of each op and dtype
is printed at the end of the module (pytest -s)."""
import math

import pytest
import torch

from fp64_bounds import A, B, DTS, LOG2E, SUB, TANH_U, U16, U32, Checker, report_worst  # noqa: E402
from fp64_bounds import edge_rows as _edge_rows, sqfloor as _sqfloor, to_rows as _to_rows, to_seq as _to_seq  # noqa: E402

pytestmark = pytest.mark.gpu

SCALES = {"unit": 1.0, "train": 2.0 ** -20, "fp16-loss-scaled": 2.0 ** -20 * 2.0 ** 16}
GELU_K0, GELU_K1 = 0.7978845608028654, 0.044715

_WORST = {}


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    report_worst(_WORST)


def _nat(dt):
    from latte_b200.train_ops import NativeOps
    return NativeOps(dt)


def _Checker(dt):
    return Checker(dt, _WORST)


def _rc(idx):
    return f"row {idx[0]}, column {idx[1]}"


def _sc(idx):
    return f"sample {idx[0]}, column {idx[1]}"


def _col(idx):
    return f"column {idx[0]}"


# ------------------------------------------------------------------------------------------------ elementwise backward ops
LN_CASES = [(3, 256, 37), (1, 4096, 0), (2, 4096, 1000)]     # (samples, rows_per_batch, rows missing from the last sample)


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("D", [384, 576, 768, 1024, 1152, 1536])     # ln_modulate_bwd's NV = 3, 6, 6, 9, 9, 12 variants
def test_ln_modulate_bwd(dev, dt, D):
    """d/dx, d/dshift, d/dscale of LayerNorm(x) (1 + scale[b]) + shift[b] (eps 1e-6), accumulated into dx and into strided
    dshift / dscale views of a dmod-shaped buffer, as the engine passes them.  Every third row of x has mean 8 and spread 0.05."""
    nat, chk = _nat(dt), _Checker(dt)
    g = torch.Generator(device=dev).manual_seed(D)
    for Bb, rpb, short in LN_CASES:
        T = Bb * rpb - short
        x = torch.randn(T, D, device=dev, generator=g) * 3 + 1
        x[::3] = 8 + 0.05 * torch.randn(x[::3].shape, device=dev, generator=g)
        mod = torch.randn(Bb, 6 * D, device=dev, generator=g) * 0.5
        shift, scale = mod[:, 0:D], mod[:, D:2 * D]
        dh0 = torch.randn(T, D, device=dev, generator=g)
        dx00 = torch.randn(T, D, device=dev, generator=g)
        dmod00 = torch.randn(Bb, 6 * D, device=dev, generator=g)
        bidx = torch.arange(T, device=dev) // rpb
        for sname, s in SCALES.items():
            dh = (dh0 * s).to(dt)
            dx, dmod = dx00 * s, dmod00 * s
            dx0, dmod0 = dx.clone(), dmod.clone()
            nat.ln_modulate_bwd(dh, x, shift, scale, rpb, dx, dmod[:, 0:D], dmod[:, D:2 * D])
            assert torch.equal(dmod[:, 2 * D:], dmod0[:, 2 * D:]), "ln_modulate_bwd wrote outside dshift / dscale"
            xx = x.double().requires_grad_(True)
            sh = shift.double().requires_grad_(True)
            scl = scale.double().requires_grad_(True)
            mean = xx.mean(1, keepdim=True)
            var = ((xx - mean) ** 2).mean(1, keepdim=True)
            rstd = (var + 1e-6).rsqrt()
            xh = (xx - mean) * rstd
            h = xh * (1 + scl[bidx]) + sh[bidx]
            dh64 = dh.double()
            (h * dh64).sum().backward()
            with torch.no_grad():
                rstd, xh = rstd.detach(), xh.detach()
                kap = 1 + rstd * x.double().abs().mean(1, keepdim=True)
                ga = dh64.abs() * (1 + scale.double().abs())[bidx]
                xa1 = xh.abs() + 1
                mag_dx = kap * rstd * (ga + ga.mean(1, keepdim=True) + xa1 * (ga * xa1).mean(1, keepdim=True))
                ref_dx = dx0.double() + xx.grad
                bnd = A * U32 * ref_dx.abs() + B * U32 * math.sqrt(D) * mag_dx
                tag = f"{sname} B={Bb} rpb={rpb} T={T}"
                chk.add("ln_modulate_bwd dx", tag, dx, ref_dx, bnd, _rc)
                n = math.sqrt(rpb)
                z = torch.zeros(Bb, D, dtype=torch.float64, device=dev)
                ref_sh = dmod0[:, 0:D].double() + sh.grad
                mag_sh = dmod0[:, 0:D].double().abs() + z.index_add(0, bidx, dh64.abs())
                chk.add("ln_modulate_bwd dshift", tag, dmod[:, 0:D], ref_sh, A * U32 * ref_sh.abs() + B * U32 * n * mag_sh, _sc)
                ref_sc = dmod0[:, D:2 * D].double() + scl.grad
                mag_sc = n * (dmod0[:, D:2 * D].double().abs() + z.index_add(0, bidx, dh64.abs() * xh.abs())) + \
                    math.sqrt(D) * z.index_add(0, bidx, dh64.abs() * kap * xa1)
                chk.add("ln_modulate_bwd dscale", tag, dmod[:, D:2 * D], ref_sc, A * U32 * ref_sc.abs() + B * U32 * mag_sc, _sc)
            del xx, sh, scl, h
    chk.done()


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("D,Bb,rpb,short", [(384, 3, 256, 50), (1152, 5, 4096, 0), (4608, 2, 2048, 7)])
def test_gate_bwd(dev, dt, D, Bb, rpb, short):
    """dm = dx * gate[b] (16-bit), dgate[b] += sum_rows dx * m (a strided view of dmod), dbias += sum_rows dx * gate[b]."""
    nat, chk = _nat(dt), _Checker(dt)
    g = torch.Generator(device=dev).manual_seed(D + rpb)
    T = Bb * rpb - short
    dx0 = torch.randn(T, D, device=dev, generator=g)
    m = torch.randn(T, D, device=dev, generator=g).to(dt)
    mod = torch.randn(Bb, 6 * D, device=dev, generator=g) * 0.5
    gate = mod[:, 2 * D:3 * D]
    dmod00 = torch.randn(Bb, 6 * D, device=dev, generator=g)
    db00 = torch.randn(D, device=dev, generator=g)
    bidx = torch.arange(T, device=dev) // rpb
    for sname, s in SCALES.items():
        dx = dx0 * s
        dmod, dbias = dmod00 * s, db00 * s
        dmod0, dbias0 = dmod.clone(), dbias.clone()
        dm = nat.gate_bwd(dx, m, gate, rpb, dmod[:, 2 * D:3 * D], dbias)
        assert torch.equal(dmod[:, :2 * D], dmod0[:, :2 * D]) and torch.equal(dmod[:, 3 * D:], dmod0[:, 3 * D:])
        xx = dx.double()
        mm = m.double().requires_grad_(True)
        gg = gate.double().requires_grad_(True)
        bias = torch.zeros(D, dtype=torch.float64, device=dev, requires_grad=True)
        y = gg[bidx] * (mm + bias)          # x_out = x + gate[b] * (m + bias): d/dm, d/dgate, d/dbias of <x_out, dx>
        (y * xx).sum().backward()
        with torch.no_grad():
            tag = f"{sname} T={T}"
            ref_dm = mm.grad
            chk.add("gate_bwd dm", tag, dm, ref_dm, A * (U16[dt] + U32) * ref_dm.abs() + SUB[dt], _rc)
            z = torch.zeros(Bb, D, dtype=torch.float64, device=dev)
            ref_g = dmod0[:, 2 * D:3 * D].double() + gg.grad
            mag_g = dmod0[:, 2 * D:3 * D].double().abs() + z.index_add(0, bidx, xx.abs() * m.double().abs())
            chk.add("gate_bwd dgate", tag, dmod[:, 2 * D:3 * D], ref_g, A * U32 * ref_g.abs() + B * U32 * math.sqrt(rpb) * mag_g, _sc)
            ref_b = dbias0.double() + bias.grad
            mag_b = dbias0.double().abs() + (xx.abs() * gate.double().abs()[bidx]).sum(0)
            chk.add("gate_bwd dbias", tag, dbias, ref_b, A * U32 * ref_b.abs() + B * U32 * math.sqrt(T) * mag_b, _col)
        del mm, gg, bias, y
    chk.done()


def _gelu64(u):
    return 0.5 * u * (1 + torch.tanh(GELU_K0 * (u + GELU_K1 * u ** 3)))


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("D,T", [(384, 1000), (1152, 4096), (4608, 16 * 256 * 5)])
def test_gelu_bwd(dev, dt, D, T):
    """du = da * gelu_tanh'(u) (16-bit) and dbias += sum_rows du, at D = 4608 (the last 1024-column block is half full); u
    near 0 in columns 0..63 and |u| in [4, 8] in columns 64..127; da has a mean, so dbias is far from a random walk."""
    nat, chk = _nat(dt), _Checker(dt)
    g = torch.Generator(device=dev).manual_seed(D + T)
    u = torch.randn(T, D, device=dev, generator=g) * 2
    u[:, :64] = torch.randn(T, 64, device=dev, generator=g) * 1e-3
    u[:, 64:128] = (4 + 4 * torch.rand(T, 64, device=dev, generator=g)) * torch.randn(T, 64, device=dev, generator=g).sign()
    u = u.to(dt)
    da0 = torch.randn(T, D, device=dev, generator=g) + 1
    db00 = torch.randn(D, device=dev, generator=g)
    u64 = u.double()
    with torch.no_grad():
        th = torch.tanh(GELU_K0 * (u64 + GELU_K1 * u64 ** 3))
        tw = th.abs() * (0.5 + u64.abs() * th.abs() * GELU_K0 * (1 + 3 * GELU_K1 * u64 ** 2))      # d gelu' / d tanh, times |tanh|
        gabs = 0.5 * (1 + th).abs() + 0.5 * u64.abs() * (1 - th * th) * GELU_K0 * (1 + 3 * GELU_K1 * u64 ** 2)
        del th
    for sname, s in SCALES.items():
        da = (da0 * s).to(dt)
        dbias = db00 * s
        dbias0 = dbias.clone()
        du = nat.gelu_bwd(da, u, dbias)
        uu = u64.clone().requires_grad_(True)
        da64 = da.double()
        (_gelu64(uu) * da64).sum().backward()
        with torch.no_grad():
            tag = f"{sname} T={T}"
            ref = uu.grad
            e_t = TANH_U * da64.abs() * tw
            e_a = da64.abs() * gabs
            chk.add("gelu_bwd du", tag, du, ref, A * U16[dt] * ref.abs() + B * (e_t + U32 * e_a) + SUB[dt], _rc)
            ref_b = dbias0.double() + ref.sum(0)
            mag_b = B * (e_t.sum(0) + U32 * math.sqrt(T) * (dbias0.double().abs() + e_a.sum(0)))
            chk.add("gelu_bwd dbias", tag, dbias, ref_b, A * U32 * ref_b.abs() + mag_b, _col)
            del e_t, e_a, ref
        del uu, da64
    chk.done()


@pytest.mark.parametrize("dt", DTS)
def test_colsum(dev, dt):
    """Column sums accumulated into fp32 (bias gradients): 16-bit inputs at 384, 1152 and 4608 columns, and fp32 input."""
    nat, chk = _nat(dt), _Checker(dt)
    g = torch.Generator(device=dev).manual_seed(5)
    for R, Dc, kind in [(1000, 384, dt), (20480, 1152, dt), (20480, 4608, dt), (4100, 1152, torch.float32)]:
        a0 = torch.randn(R, Dc, device=dev, generator=g)
        b00 = torch.randn(Dc, device=dev, generator=g)
        for sname, s in SCALES.items():
            a = (a0 * s).to(kind)
            base = b00 * s
            out = nat.colsum(a, base.clone())
            aa = a.double()
            bias = torch.zeros(Dc, dtype=torch.float64, device=dev, requires_grad=True)
            (bias * aa).sum().backward()            # d/dbias of <y + bias, a> with a the upstream gradient: its column sums
            ref = base.double() + bias.grad
            mag = base.double().abs() + aa.abs().sum(0)
            chk.add(f"colsum {'fp32' if kind == torch.float32 else '16-bit'}", f"{sname} {R}x{Dc}", out, ref,
                    A * U32 * ref.abs() + B * U32 * math.sqrt(R) * mag, _col)
    chk.done()


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("rows", [1, 2, 5, 8, 96])
def test_ada_gradients(dev, dt, rows):
    """dW = dmod^T silu(c) and dsc = dmod W of the stacked adaLN Linear at Latte-XL/2's NA = 28*6*1152 + 2*1152 = 195840 and
    D = 1152: one pass each up to 8 rows; 96 rows (LatteIMG's per-frame rows) go through the weight-gradient GEMM with dmod
    rounded to 16 bits.  dmod has the row stride of a wider buffer."""
    nat, chk = _nat(dt), _Checker(dt)
    D, NA = 1152, 28 * 6 * 1152 + 2 * 1152
    g = torch.Generator(device=dev).manual_seed(rows)
    dbuf0 = torch.randn(rows, NA + 64, device=dev, generator=g)
    sc = torch.randn(rows, D, device=dev, generator=g).to(dt)
    w = (torch.randn(NA, D, device=dev, generator=g) / 34).to(dt)
    gemm = rows > 8
    for sname, s in SCALES.items():
        dmod = (dbuf0 * s)[:, :NA]
        dW = nat.ada_outer(dmod, sc)
        dsc = nat.ada_dsc(dmod, w)
        s64 = sc.double().requires_grad_(True)
        w64 = w.double().requires_grad_(True)
        d64 = dmod.double()
        ((s64 @ w64.t()) * d64).sum().backward()
        ref_w, ref_s = w64.grad, s64.grad
        del w64, s64
        with torch.no_grad():
            tag = f"{sname} rows={rows}"
            u_op = U16[dt] if gemm else 0.0
            mag = d64.abs().t() @ sc.double().abs()
            bnd = A * U32 * ref_w.abs() + B * (u_op + U32 * math.sqrt(rows)) * mag
            del mag
            if gemm and SUB[dt]:
                bnd += _sqfloor(d64, sc.double(), SUB[dt], lhs_t=True)
            chk.add("ada_outer", tag, dW, ref_w, bnd, lambda i: f"row {i[0]} of the stacked weight, column {i[1]}")
            del bnd, ref_w, dW
            mag = d64.abs() @ w.double().abs()
            bnd = A * U32 * ref_s.abs() + B * (u_op + U32 * math.sqrt(NA)) * mag
            if gemm and SUB[dt]:
                bnd += _sqfloor(d64, w.double(), SUB[dt])
            chk.add("ada_dsc", tag, dsc, ref_s, bnd, _sc)
    chk.done()


# ------------------------------------------------------------------------------------------------ attention backward
def _softmax_bwd_terms(q, k, v, do, bias, dt):
    """fp64 autograd of o = softmax(q k^T hd^-1/2 + bias) v with upstream do (q [.., Sq, hd], k / v [.., Sk, hd]), and the
    error-bound terms of the kernels' dq / dk / dv: B * u_op * mag + floor (see the module docstring)."""
    sc = q.shape[-1] ** -0.5
    qq, kk, vv = (t.clone().requires_grad_(True) for t in (q, k, v))
    s = qq @ kk.transpose(-1, -2) * sc
    if bias is not None:
        s = s + bias
    p = torch.softmax(s, -1)
    ((p @ vv) * do).sum().backward()
    out = {"dq": qq.grad, "dk": kk.grad, "dv": vv.grad}
    with torch.no_grad():
        P = p.detach()
        u_row = U16[dt] + 2 * U32 * LOG2E * s.detach().abs().amax(-1, keepdim=True)
        del s, p, qq, kk, vv
        dP = do @ v.transpose(-1, -2)
        delta = (P * dP).sum(-1, keepdim=True)
        dabs = (P * (do.abs() @ v.abs().transpose(-1, -2))).sum(-1, keepdim=True)     # |delta| as computed from |dO| |O|
        mdS = P * ((dP - delta).abs() + dabs)
        del dP
        wdS, wP = u_row * mdS, u_row * P
        terms = {"dq": B * sc * (wdS @ k.abs()), "dk": B * sc * (wdS.transpose(-1, -2) @ q.abs()),
                 "dv": B * (wP.transpose(-1, -2) @ do.abs())}
        del wdS, wP
        if SUB[dt]:
            terms["dq"] += sc * _sqfloor(mdS, k, SUB[dt]) + SUB[dt]
            terms["dk"] += sc * _sqfloor(mdS, q, SUB[dt], lhs_t=True) + SUB[dt]
            terms["dv"] += _sqfloor(P, do, SUB[dt], lhs_t=True) + SUB[dt]
    return out, terms


def _attention_case(dev, dt, Bb, Fr, N, H, hd, temporal):
    nat, chk = _nat(dt), _Checker(dt)
    kind = "temporal" if temporal else "spatial"
    S, nseq = (Fr, Bb * N) if temporal else (N, Bb * Fr)
    T, D = Bb * Fr * N, H * hd
    g = torch.Generator(device=dev).manual_seed(Bb * 100003 + Fr * 1009 + N * 7 + hd)
    x = torch.randn(nseq, 3, H, S, hd, device=dev, generator=g)
    _edge_rows(x)
    qkv = _to_rows(x, Bb, Fr, N, H, hd, temporal).to(dt).contiguous()
    del x
    o = nat.attention(qkv, Bb, Fr, N, H, temporal)
    do0 = torch.randn(T, D, device=dev, generator=g) * torch.exp(torch.empty(T, 1, device=dev).uniform_(-3, 3, generator=g))
    qs = _to_seq(qkv, Bb, Fr, N, 3, H, hd, temporal).double()
    step = max(1, (1 << 24) // (H * S * S))           # sequences per fp64 reference chunk: <= 2^24 scores per tensor

    def where(c0):
        def f(i):
            sq, h, pos, d = c0 + i[0], i[1], i[2], i[3]
            row = ((sq // N) * Fr + pos) * N + sq % N if temporal else sq * N + pos
            return f"{kind} sequence {sq}, head {h}, position {pos} (row {row}), dim {d}"
        return f

    for sname, s in SCALES.items():
        do = (do0 * s).to(dt)
        got = _to_seq(nat.attention_bwd(qkv, o, do, Bb, Fr, N, H, temporal), Bb, Fr, N, 3, H, hd, temporal)
        dos = _to_seq(do, Bb, Fr, N, 1, H, hd, temporal)
        for c0 in range(0, nseq, step):
            c1 = min(nseq, c0 + step)
            ref, terms = _softmax_bwd_terms(qs[c0:c1, 0], qs[c0:c1, 1], qs[c0:c1, 2], dos[c0:c1, 0].double(), None, dt)
            for i, name in enumerate(("dq", "dk", "dv")):
                bnd = A * U16[dt] * ref[name].abs() + terms[name]
                chk.add(f"attention_bwd {kind} {name}", f"{sname} B={Bb} F={Fr} N={N} H={H} hd={hd}", got[c0:c1, i],
                        ref[name], bnd, where(c0))
            del ref, terms
    chk.done()


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("H,hd", [(16, 72), (6, 64)])
@pytest.mark.parametrize("N,Bf", [(64, (2, 4)), (128, (1, 4)), (256, (2, 2)), (1024, (1, 2))])
def test_attention_bwd_spatial(dev, dt, H, hd, N, Bf):
    _attention_case(dev, dt, Bf[0], Bf[1], N, H, hd, False)


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("H,hd", [(16, 72), (6, 64)])
@pytest.mark.parametrize("Fr", [1, 2, 15, 16, 17, 33, 64, 100, 128])
def test_attention_bwd_temporal(dev, dt, H, hd, Fr):
    """F <= 16: the one-warp-per-sequence kernel; F > 16: the two-kernel backward over strided rows (partial last block unless
    F is a multiple of 64).  Five tokens per frame."""
    _attention_case(dev, dt, 2, Fr, 5, H, hd, True)


# ------------------------------------------------------------------------------------------------ cross-attention backward
XCASES = [  # (videos, query rows per sample, caption length, heads, hd, mask, images per video)
    (2, 128, 1, 16, 72, None, 0), (1, 4096, 20, 16, 72, "partial", 0), (2, 4096, 77, 16, 72, "all", 0),
    (1, 16384, 120, 16, 72, "partial", 0), (1, 16384, 128, 16, 72, None, 0), (3, 128, 128, 6, 64, "all", 0),
    (2, 1024, 120, 16, 72, "partial", 3),
]


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("case", XCASES, ids=lambda c: "-".join(str(v) for v in c))
def test_cross_attention_bwd(dev, dt, case):
    """softmax(q k^T hd^-1/2 + key_bias) v backward with q / kv / dkv laid out as training_t2v.py passes them: q rows of a
    buffer holding the video rows and then the image rows (images: one more call with B * images samples of 256 rows), k | v
    a column window of the stacked caption K/V of all layers, dK | dV written into the same window of a NaN-filled buffer,
    key_bias rows sliced per call.  Masks: none, keys L/2+1.. of sample 0, and a fully masked last sample."""
    Bv, rows, L, H, hd, mask, images = case
    D = H * hd
    nat, chk = _nat(dt), _Checker(dt)
    g = torch.Generator(device=dev).manual_seed(rows + L + hd + images)
    img_rows = 256
    calls = [(0, Bv, rows, 0)]                                       # (first q row, samples, q rows per sample, first sample)
    if images:
        calls.append((Bv * rows, Bv * images, img_rows, Bv))
    nsamp = Bv + Bv * images
    qall = torch.randn(Bv * rows + Bv * images * img_rows, D, device=dev, generator=g).to(dt)
    col0 = 2 * D                                                     # layer 1 of a 3-layer stacked K/V
    kvall = torch.randn(nsamp * L, 3 * 2 * D, device=dev, generator=g).to(dt)
    bias = None
    if mask is not None:
        bias = torch.zeros(nsamp, 128, device=dev)
        bias[0, L // 2 + 1:L] = -10000.0
        if mask == "all":
            bias[nsamp - 1, :L] = -10000.0
        if images:
            bias[Bv + 1, :L // 3] = -10000.0
    do0 = torch.randn(qall.shape, device=dev, generator=g) * torch.exp(torch.empty(qall.shape[0], 1, device=dev).uniform_(-3, 3, generator=g))
    kv = kvall[:, col0:col0 + 2 * D]
    o = torch.cat([nat.cross_attention(qall[r0:r0 + nb * rq], kv[s0 * L:(s0 + nb) * L], nb, rq, L, H,
                                       bias[s0:s0 + nb] if bias is not None else None) for r0, nb, rq, s0 in calls])
    for sname, s in SCALES.items():
        do = (do0 * s).to(dt)
        dkv = torch.full((nsamp * L, 3 * 2 * D), float("nan"), device=dev, dtype=dt)
        dq = torch.cat([nat.cross_attention_bwd(qall[r0:r0 + nb * rq], kv[s0 * L:(s0 + nb) * L], o[r0:r0 + nb * rq],
                                                do[r0:r0 + nb * rq], nb, rq, L, H, bias[s0:s0 + nb] if bias is not None else None,
                                                dkv[s0 * L:(s0 + nb) * L], col0) for r0, nb, rq, s0 in calls])
        assert torch.isnan(dkv[:, :col0]).all() and torch.isnan(dkv[:, col0 + 2 * D:]).all(), "dkv written outside its window"
        for r0, nb, rq, s0 in calls:
            q4 = qall[r0:r0 + nb * rq].double().reshape(nb, rq, H, hd).transpose(1, 2)
            kv5 = kv[s0 * L:(s0 + nb) * L].double().reshape(nb, L, 2, H, hd)
            k4, v4 = kv5[:, :, 0].transpose(1, 2), kv5[:, :, 1].transpose(1, 2)
            do4 = do[r0:r0 + nb * rq].double().reshape(nb, rq, H, hd).transpose(1, 2)
            dq4 = dq[r0:r0 + nb * rq].reshape(nb, rq, H, hd).transpose(1, 2)
            dkv5 = dkv[s0 * L:(s0 + nb) * L, col0:col0 + 2 * D].reshape(nb, L, 2, H, hd)
            got = {"dq": dq4, "dk": dkv5[:, :, 0].transpose(1, 2), "dv": dkv5[:, :, 1].transpose(1, 2)}
            b4 = bias[s0:s0 + nb, None, None, :L].double() if bias is not None else None
            for n0 in range(nb):                                     # one sample at a time: <= 16 x 16384 x 128 scores
                ref, terms = _softmax_bwd_terms(q4[n0:n0 + 1], k4[n0:n0 + 1], v4[n0:n0 + 1], do4[n0:n0 + 1],
                                                b4[n0:n0 + 1] if b4 is not None else None, dt)
                for name in ("dq", "dk", "dv"):
                    what = "query" if name == "dq" else "key"

                    def where(i, what=what, n0=n0, s0=s0):
                        return f"sample {s0 + n0}, head {i[1]}, {what} {i[2]}, dim {i[3]}"
                    chk.add(f"cross_attention_bwd {name}", f"{sname} {case}", got[name][n0:n0 + 1], ref[name],
                            A * U16[dt] * ref[name].abs() + terms[name], where)
                del ref, terms
    chk.done()
