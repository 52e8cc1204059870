"""Element-by-element error bounds against fp64 references, shared by the fp64 kernel tests (test_gpu_train_ops_fp64.py,
test_gpu_forward_ops_fp64.py, test_gpu_t5_fp64.py, test_gpu_t2v_glue_fp64.py).  Each output element must satisfy

    |got - ref| <= A * u_out * |ref| + B * u_op * mag + floor

with the unit roundoffs below; each test module derives its u_op * mag and floor terms in its docstring.  `Checker` keeps the
worst err / bound per op and dtype in a dict owned by the test module, which prints it at the end (`report_worst`)."""
import math

import torch

DTS = [torch.float16, torch.bfloat16]
U16 = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
U32 = 2.0 ** -24
SUB = {torch.float16: 2.0 ** -24, torch.bfloat16: 0.0}     # subnormal spacing of the 16-bit type (bf16: none that matters)
TANH_U = 2.0 ** -11                                          # tanh.approx.f32 relative error
EX2_U = 2.0 ** -22                                           # ex2.approx.f32 relative error
LOG2E = 1.4426950408889634
GELU_K0, GELU_K1 = 0.7978845608028654, 0.044715
A, B, F = 2.0, 4.0, 3.0
ACC = 1.0        # forward fp32 tensor-core accumulation: u_op = ACC * sqrt(K) * 2^-24 (measured in test_gpu_forward_ops_fp64.py)


def dtn(dt):
    return str(dt).replace("torch.", "")


class Checker:
    """Compares every output of one test, keeps the worst err / bound per op and dtype in `worst`, and fails at the end
    listing every output above 1 with its location.  `worst=None` records nothing (used to show that a wrong result is
    rejected)."""

    def __init__(self, dt, worst=None):
        self.dt, self.worst, self.bad = dt, worst, []

    def add(self, op, what, got, ref, bound, where):
        got = got.double()
        err = (got - ref).abs()
        ratio = torch.where(bound > 0, err / bound.clamp_min(1e-300),
                            torch.where(err > 0, torch.full_like(err, math.inf), torch.zeros_like(err)))
        ratio = torch.where(torch.isfinite(got), ratio, torch.full_like(ratio, math.inf))
        i = int(torch.argmax(ratio).item())
        r = float(ratio.reshape(-1)[i].item())
        idx = [int(v) for v in torch.unravel_index(torch.tensor(i), ratio.shape)]
        loc = (f"{what} at {where(idx)}: got {got.reshape(-1)[i].item():.6g}, ref {ref.reshape(-1)[i].item():.6g}, "
               f"bound {bound.reshape(-1)[i].item():.3g}")
        key = (op, dtn(self.dt))
        if self.worst is not None and (key not in self.worst or r > self.worst[key][0]):
            self.worst[key] = (r, loc)
        if r > 1.0:
            self.bad.append(f"{op} {loc}: err/bound {r:.3g}")
        return r

    def done(self):
        assert not self.bad, "\n".join(self.bad[:12])


def report_worst(worst):
    if worst:
        print("\nworst err / bound per op and dtype:")
        for (op, dt), (r, where) in sorted(worst.items()):
            print(f"  {op:<34} {dt:<9} {r:8.3g}   {where}")


def sqfloor(x, y, s, lhs_t=False):
    """F * sqrt(sum_k (min(s, |x|) * |y|)^2) as a matrix product: x [.., m, k] (or [.., k, m] with lhs_t), y [.., k, n]."""
    xm = x.abs().clamp_max(s) ** 2
    if lhs_t:
        xm = xm.transpose(-1, -2)
    return F * (xm @ (y * y)).sqrt()


def gelu_fwd_terms(pre, uacc, mag):
    """fp64 gelu_tanh(pre) of a GEMM pre-activation and its bound term B * (...) without the output rounding: |gelu'(pre)|
    uacc mag for the accumulation, tanh.approx.f32 (relative 2^-11 of t = tanh(u)) times 0.5 |pre|, and four fp32
    roundings of u = k0 (x + k1 x^3) times 0.5 |pre| (1 - t^2) |u|."""
    u = GELU_K0 * (pre + GELU_K1 * pre ** 3)
    t = torch.tanh(u)
    ref = 0.5 * pre * (1 + t)
    dg = (0.5 * (1 + t) + 0.5 * pre * (1 - t * t) * GELU_K0 * (1 + 3 * GELU_K1 * pre ** 2)).abs()
    return ref, B * (dg * uacc * mag + 0.5 * pre.abs() * (TANH_U * t.abs() + 4 * U32 * u.abs() * (1 - t * t)))


def silu_err(x, e_in):
    """First-order error of silu(x) = x / (1 + __expf(-x)) given an input error e_in: |silu'(x)| e_in, the __expf error
    (2 + 1.173 |x| ulp of fp32) and the rounding of 1 + e and of the division."""
    sg = torch.sigmoid(x)
    d = (sg * (1 + x * (1 - sg))).abs()
    return d * e_in + U32 * (2 * (2 + 1.173 * x.abs()) + 2) * (x * sg).abs()


def softmax_fwd_terms(q, k, v, bias, dt, scale=None):
    """fp64 softmax(q k^T scale + bias) v (q [.., Sq, hd], k / v [.., Sk, hd]; scale None = hd^-1/2; bias None or an additive
    fp32 score bias broadcast to [.., Sq, Sk]) and its bound terms B * u_op * mag + floor, with u_op per query row =
    2^-11 / 2^-8 (P rounded to 16 bits before the PV product) + 2 * 2^-24 * log2(e) * max|s| (the fp32 exp2 argument) +
    2^-22 (ex2.approx.f32) + ACC * sqrt(hd) * 2^-24 * max_j |q| |k_j| * scale (the fp32 QK^T) + sqrt(Sk) * 2^-24 (the fp32
    PV and l sums), and mag = sum_j p_j |v_j|.  max|s| is taken over the keys with p_j > 0 only: an error in the exp2 argument
    of key j moves p_j by a relative 2^-24 |s_j| ln 2, nothing for a key whose probability is 0 in fp64 and in fp32 (a -1e30
    padding key: ex2 of about -1.4e30; a -10000 key beside an unmasked one: ex2 of about -14000).  Such keys inside max|s|
    would make the bound ~1e23 for the -1e30 padding and accept anything.  fp16 floor: 2^-24 plus
    F * p_max * sqrt(sum_j (min(2^-24, P_j) |v_j|)^2), P_j = p_j / p_max the unnormalised probability the kernel rounds.
    Returns (out, term, p)."""
    hd, S = q.shape[-1], k.shape[-2]
    sc = hd ** -0.5 if scale is None else scale
    s = q @ k.transpose(-1, -2) * sc
    if bias is not None:
        s = s + bias
    p = torch.softmax(s, -1)
    out = p @ v
    qk = (q.abs() @ k.abs().transpose(-1, -2)) * sc
    smax = torch.where(p > 0, s.abs(), torch.zeros_like(s)).amax(-1, keepdim=True)
    u_row = (U16[dt] + EX2_U + 2 * U32 * LOG2E * smax + ACC * math.sqrt(hd) * U32 * qk.amax(-1, keepdim=True)
             + math.sqrt(S) * U32)
    del s, qk
    term = B * u_row * (p @ v.abs())
    if SUB[dt]:
        pmax = p.amax(-1, keepdim=True)
        term += sqfloor(p / pmax, v, SUB[dt]) * pmax + SUB[dt]
    return out, term, p


# ------------------------------------------------------------------------------------------------ attention layouts
def to_seq(t, Bb, Fr, N, parts, H, hd, temporal):
    """[B*F*N, parts*H*hd] rows (b, f, n) -> [sequences, parts, H, S, hd]: spatial sequences (b, f) over n, temporal (b, n)
    over f."""
    x = t.reshape(Bb, Fr, N, parts, H, hd)
    if temporal:
        return x.permute(0, 2, 3, 4, 1, 5).reshape(Bb * N, parts, H, Fr, hd)
    return x.permute(0, 1, 3, 4, 2, 5).reshape(Bb * Fr, parts, H, N, hd)


def to_rows(x, Bb, Fr, N, H, hd, temporal):
    parts = x.shape[1]
    if temporal:
        return x.reshape(Bb, N, parts, H, Fr, hd).permute(0, 4, 1, 2, 3, 5).reshape(Bb * Fr * N, parts * H * hd)
    return x.reshape(Bb, Fr, parts, H, N, hd).permute(0, 1, 4, 2, 3, 5).reshape(Bb * Fr * N, parts * H * hd)


def edge_rows(x):
    """x [sequences, 3, H, S, hd] (q | k | v): query 0 peaks at the LAST key (logit 30), query 1 is constant (q = 0), query 2
    has logits +30 at the middle key and -30 at key 0, query 3 shares its maximum between keys 1 and S - 2."""
    S, hd = x.shape[3], x.shape[4]
    k = x[:, 1]

    def toward(j, logit):
        kj = k[:, :, j]
        return kj * (logit * math.sqrt(hd) / (kj * kj).sum(-1, keepdim=True))
    x[:, 0, :, 0] = toward(S - 1, 30.0)
    if S > 1:
        x[:, 0, :, 1] = 0
    if S > 2:
        x[:, 0, :, 2] = toward(S // 2, 30.0) + toward(0, -30.0)
    if S > 3:
        x[:, 0, :, 3] = toward(1, 12.0) + toward(S - 2, 12.0)
