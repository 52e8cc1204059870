"""The training objective (`b200_training_loss`, reached through `SpacedDiffusion.training_losses`) in fp64 with a
per-element error bound for the kernel's fp32 arithmetic, shared by tests/test_loss_bounds.py (CPU: the bound accepts the
oracle's own fp32 evaluation and rejects plausible wrong results) and tests/test_gpu_diffusion_loss_fp64.py (the kernel).

Reference.  The objective's expressions in fp64 on the fp32 inputs the kernel reads (x0, x_t, noise, the model output) and
on the schedule tables it reads (`SpacedDiffusion._state`: the float64 tables rounded to fp32).  Two choices follow torch's
fp32 evaluation rather than the fp64 one: the t = 0 branch is picked by comparing fp32 x0 with fp32(+-0.999) (0.999 itself
rounds up to 0.99900001, so x0 = fp32(0.999) takes the middle branch in fp32 and the edge branch in fp64, and the gradients
differ by a factor of 4 there), and the clamp is fp32(1e-12), with a zero gradient at or below it.  The tanh-CDF tails,
the KL near the optimum (-1 + x + exp(-x) with x = lv - mn tiny) and ca - cb are evaluated in forms that keep their digits
in fp64 (sigmoid, expm1, tanh a - tanh b = sinh(a - b) / (cosh a cosh b)).  Per sample n = F C H W elements:

    mse = sum (noise - eps)^2 / n,  vb = sum term / (n ln 2),  d mse / d eps = -2 (noise - eps) / n,
    d vb / d v = dterm/dlv 0.5 (max_log - min_log) / (n ln 2),  term = KL (t > 0) or -log max(arg, 1e-12) (t = 0).

Bound.  A first-order error is carried through the kernel's operation chain, one fp32 rounding (2^-24 relative) per
operation, FMA contraction allowed: frac, lv, pred, mean, tm, dm; e1 = __expf(mn - lv) and e2 = dm^2 __expf(-lv) with the
__expf error 2 + 1.173 |x| ulp (CUDA C Programming Guide); for e2, 2 |dm| e_dm E + e_dm^2 E + e2 (...), E = exp(-lv), so
the bound holds as dm -> 0.  The error of lv enters the KL through its derivative 0.5 (1 - e1 - e2): near the optimum
that cancels, and a bound that added the three parts would accept a wrong variance interpolation.  At t = 0: inv_std =
__expf(-0.5 lv), z_a, z_b, the cubic, tanhf (2 ulp; exactly +-1 when |y| >= 10, where 1 - tanh(y) = 4e-9 is under a
fifteenth of the fp32 spacing below 1, so a saturated CDF is exactly 0 or 1), the CDF and its derivative, and arg = ca - cb,
ca or 1 - cb.  Then -__logf(max(arg, 1e-12)) is bounded over the interval arg +- B e_arg, clamped as the kernel clamps,
plus the __logf error (2^-21.41 absolute on [0.5, 2], 3 ulp elsewhere): in the saturated case 1 - cb is exactly 0 in fp32,
where e_arg / arg would be infinite.  Where the interval straddles the clamp either the clamped value with gradient 0 or
the live value is accepted; where it lies below, the gradient must be exactly 0.  The gradient -darg / arg is bounded over
the same intervals.  Per element:

    |got - ref| <= A * 2^-24 * |ref| + B * e        (tests/fp64_bounds.py: A = 2, B = 4)

with the interval terms already scaled by B.  The per-sample sums add the per-element bounds plus
B * 2^-24 * (iters + 13 + bx) * sum |term| (bx = min(64, ceil(n / 256)) blocks of 256 threads, iters = ceil(n / (bx 256))
grid-stride iterations per thread, then 5 warp-shuffle levels, the 8-warp block sum, slack, and bx atomicAdds in any
order); the means add three fp32 roundings (torch divides by a Python scalar as a multiply by the fp32 reciprocal of the
fp32-rounded scalar).  The gradients add the kernel's fp32 factors: 3 roundings for -2 d inv_n, 6 for
dterm_dlv 0.5 (mx - mn) inv_n / ln 2 (the subtraction, inv_n, the constant 1/ln 2 and three products)."""
import math

import numpy as np
import torch

from fp64_bounds import A, B, GELU_K0, GELU_K1, U32, Checker

ULP = 2 * U32                              # one ulp of an fp32 value is at most 2^-23 of its magnitude
BIN = 1.0 / 255.0
CLAMP = float(np.float32(1e-12))
THR = float(np.float32(0.999))
LN2 = math.log(2.0)
TANH_SAT = 10.0
LOGF_ABS = 2.0 ** -21.41
SUM_SLACK = 13


def t_values(T):
    """Chain indices every regime draws its t from: the decoder NLL (0), the first steps, the middle and the last two
    (on the 1000-step chain 0, 1, 2, 10, 500, 998, 999)."""
    return (0, 1, 2, 10, T // 2, T - 2, T - 1)


def planted_x0():
    """+-fp32(0.999) and their fp32 neighbours, +-1 and +-3: the values where the t = 0 branches switch or sit far off."""
    f = np.float32(0.999)
    v = [f, np.nextafter(f, np.float32(2)), np.nextafter(f, np.float32(0)), 1.0, 3.0]
    return [float(s * x) for x in v for s in (1.0, -1.0)]


def geometry(n):
    """(bx, iters) of launch_training_loss for n elements per sample."""
    bx = min(64, (n + 255) // 256)
    return bx, (n + bx * 256 - 1) // (bx * 256)


def tables(diff, device):
    """[6, T] fp32: sqrt_recip_alphas_cumprod, sqrt_recipm1_alphas_cumprod, posterior_mean_coef1, posterior_mean_coef2,
    posterior_log_variance_clipped, log_betas -- the rows `b200_training_loss` reads."""
    return diff._state(device, 1)[1][:6]


def make_case(diff, shape, ts, sigma, seed, device):
    """Inputs of one training-loss call.  x0 ~ N(0, 1) clipped to +-4 (latents), noise ~ N(0, 1), eps = noise + sigma N(0, 1),
    var_values ~ U[-1, 1]; x_t from the module's q_sample.  Per sample: frame 0 channel 0 starts with `planted_x0()`;
    channel 1 of every frame cycles v through -1 (lv == min_log exactly), 1, -1.5, 1.5; channel 3 of the last frame has
    eps = noise +- U[4, 10] (at t = 0 the decoder bin is 4 to 11 standard deviations away: the CDFs saturate and the
    clamp at 1e-12 is reached)."""
    Bb, Fr, Cc, H, W = shape
    g = torch.Generator(device=device).manual_seed(seed)
    x0 = torch.randn(shape, device=device, generator=g).clamp_(-4, 4)
    pl = torch.tensor(planted_x0(), device=device)
    x0.view(Bb, Fr, Cc, H * W)[:, 0, 0, :pl.numel()] = pl
    noise = torch.randn(shape, device=device, generator=g)
    eps = noise + sigma * torch.randn(shape, device=device, generator=g)
    far = 4 + 6 * torch.rand(Bb, H, W, device=device, generator=g)
    sign = torch.randint(0, 2, (Bb, H, W), device=device, generator=g).float() * 2 - 1
    eps[:, -1, 3] = noise[:, -1, 3] + sign * far
    v = torch.rand(shape, device=device, generator=g) * 2 - 1
    vv = v.view(Bb, Fr, Cc, H * W)
    for j, val in enumerate((-1.0, 1.0, -1.5, 1.5)):
        vv[:, :, 1, j::4] = val
    t = torch.tensor(ts, device=device, dtype=torch.int64)
    xt = diff.q_sample(x0, t, noise)
    mo = torch.cat([eps, v], dim=2).contiguous()
    return {"x0": x0, "xt": xt, "noise": noise, "mo": mo, "t": t}


def _logcosh(y):
    a = y.abs()
    return a + torch.log1p(torch.exp(-2 * a)) - LN2


def _cdf_side(p, isd, e_p, e_isd):
    """One side of the discretised likelihood: z = inv_std * p, y = k0 (z + k1 z^3), the CDF 0.5 (1 + tanh y) and its
    derivative 0.5 (1 - tanh^2 y) k0 (1 + 3 k1 z^2), each with its first-order fp32 error."""
    z = isd * p
    e_z = p.abs() * e_isd + isd * e_p + U32 * z.abs()
    q = GELU_K1 * z ** 3
    w = z + q
    e_w = (1 + 3 * GELU_K1 * z * z) * e_z + 4 * U32 * q.abs() + U32 * w.abs()
    y = GELU_K0 * w
    e_y = GELU_K0 * e_w + 2 * U32 * y.abs()
    th = torch.tanh(y)
    se = 4 * torch.sigmoid(2 * y) * torch.sigmoid(-2 * y)        # 1 - tanh^2, with its digits in the tails
    sat = y.abs() - B * e_y >= TANH_SAT
    e_th = torch.where(sat, 2 * torch.sigmoid(-2 * y.abs()), se * e_y + 2 * ULP * th.abs())
    cdf = torch.sigmoid(2 * y)
    e_cdf = 0.5 * (e_th + torch.where(sat, torch.zeros_like(th), U32 * (1 + th).abs()))
    P = 1 + 3 * GELU_K1 * z * z
    e_P = 6 * GELU_K1 * z.abs() * e_z + U32 * (4 * (P - 1) + P)
    e_S = torch.where(sat, se, 2 * th.abs() * e_th + U32 * (th * th + se))
    D = 0.5 * GELU_K0 * se * P
    e_D = 0.5 * GELU_K0 * (P * e_S + se * e_P) + 3 * U32 * D
    return z, e_z, y, cdf, e_cdf, D, e_D


def evaluate(case, tab, variant=None):
    """fp64 reference of one call (and, with variant None, its bounds).  Per-sample "mse", "vb" (means, vb in bits),
    "mse_sum", "vb_sum" (the kernel's raw sums, vb in nats); per element "g_eps" = d mse / d eps, "g_var" = d vb / d v,
    "g_vb_eps" = d vb / d eps (what an unfrozen mean would add), all [B, F, C, HW]; "bnd_*" their bounds.

    `variant` builds a plausible wrong result: "clip_pred_x0" (pred_x0 clipped to [-1, 1], the sampling default),
    "swap_min_max_log" (min_log and max_log swapped in the variance interpolation), "kl_at_t0" (a t = 0 sample scored with the
    KL), "swap_hi_branch" (x0 > 0.999 scored with log cdf_plus), "no_inv_ln2" (the variance gradient in nats),
    "flip_dz_dlv" (the t = 0 gradient with dz/dlv = +z/2), "unfrozen_mean" (d vb / d eps added to the eps channels),
    "neighbour_t" (the previous sample's t in the VB part), "mse_over_2c" (the MSE averaged over 2C channels),
    "grad_through_clamp" (-darg / max(arg, 1e-12) where arg is clamped)."""
    mo = case["mo"].double()
    Bb, Fr, C2 = mo.shape[:3]
    Cc = C2 // 2
    sh = (Bb, Fr, Cc, -1)
    x0f = case["x0"].reshape(sh)
    x0, xt, nz = x0f.double(), case["xt"].reshape(sh).double(), case["noise"].reshape(sh).double()
    mo = mo.reshape(Bb, Fr, C2, -1)
    eps, v = mo[:, :, :Cc], mo[:, :, Cc:]
    n = Fr * Cc * x0.shape[-1]
    t = case["t"]
    tv = t.roll(1) if variant == "neighbour_t" else t
    co = tab.double()[:, tv].view(6, Bb, 1, 1, 1)
    Ac, Bc, c1, c2, mn, mx = co
    t0 = (tv == 0).view(Bb, 1, 1, 1)

    d = nz - eps
    sq = d * d
    frac = (v + 1) / 2
    fa = 1 - frac if variant == "swap_min_max_log" else frac
    x = fa * (mx - mn)                                                 # lv - mn, without the cancellation
    lv = mn + x
    pred = Ac * xt - Bc * eps
    if variant == "clip_pred_x0":
        pred = pred.clamp(-1, 1)
    mean = c1 * pred + c2 * xt
    # KL to the true posterior (t > 0)
    tm = c1 * x0 + c2 * xt
    dm = tm - mean
    E1, E = torch.exp(-x), torch.exp(-lv)
    e2 = dm * dm * E
    kl = 0.5 * (x + torch.expm1(-x) + e2)
    gk = 0.5 * (-torch.expm1(-x) - e2)
    # discretised decoder NLL (t = 0)
    cen = x0 - mean
    isd = torch.exp(-0.5 * lv)
    e_lv = (mx.abs() * U32 * frac.abs() + mn.abs() * (U32 * frac.abs() + U32 * (1 - frac).abs())
            + U32 * ((frac * mx).abs() + ((1 - frac) * mn).abs() + lv.abs()))
    e_pred = U32 * ((Ac * xt).abs() + (Bc * eps).abs() + pred.abs())
    e_mean = c1.abs() * e_pred + U32 * ((c1 * pred).abs() + (c2 * xt).abs() + mean.abs())
    e_cen = e_mean + U32 * cen.abs()
    e_isd = isd * (0.5 * e_lv + ULP * (2 + 1.173 * (0.5 * lv).abs()))
    pa, pb = cen + BIN, cen - BIN
    za, e_za, ya, ca, e_ca, da, e_da = _cdf_side(pa, isd, e_cen + U32 * (BIN + pa.abs()), e_isd)
    zb, e_zb, yb, cb, e_cb, db, e_db = _cdf_side(pb, isd, e_cen + U32 * (BIN + pb.abs()), e_isd)
    lo, hi = x0f < -THR, x0f > THR
    dy = ya - yb                                                       # > 0: the CDF is increasing
    mid = 0.5 * torch.exp(dy + torch.log(-torch.expm1(-2 * dy)) - LN2 - _logcosh(ya) - _logcosh(yb))
    ga, gb = da * (-0.5 * za), db * (-0.5 * zb)                        # d ca / dlv, d cb / dlv (dz/dlv = -z/2)
    hi_arg, hi_darg = (ca, ga) if variant == "swap_hi_branch" else (torch.sigmoid(-2 * yb), -gb)
    arg = torch.where(lo, ca, torch.where(hi, hi_arg, mid))
    darg = torch.where(lo, ga, torch.where(hi, hi_darg, ga - gb))
    if variant == "flip_dz_dlv":
        darg = -darg
    live = arg > CLAMP
    argc = arg.clamp_min(CLAMP)
    nll = -torch.log(argc)
    gn = -darg / argc if variant == "grad_through_clamp" else torch.where(live, -darg / argc, torch.zeros_like(arg))

    t0b = t0 if variant != "kl_at_t0" else torch.zeros_like(t0)
    term = torch.where(t0b, nll, kl)
    gterm = torch.where(t0b, gn, gk)
    dmean = -c1 * Bc                                                   # d mean / d eps
    dmdm = torch.where(lo, -da * isd, torch.where(hi, db * isd, -(da - db) * isd))   # d arg / d mean
    dterm_deps = torch.where(t0, torch.where(live, -dmdm / argc, torch.zeros_like(arg)), -dm * E) * dmean
    n_mse = 2 * n if variant == "mse_over_2c" else n
    half_range = 0.5 * ((mn - mx) if variant == "swap_min_max_log" else (mx - mn))
    vb_scale = 1.0 if variant == "no_inv_ln2" else 1.0 / LN2
    out = {"mse_sum": sq.sum((1, 2, 3)) * n / n_mse, "vb_sum": term.sum((1, 2, 3)),
           "g_eps": -2 * d / n, "g_var": gterm * half_range / n * vb_scale, "g_vb_eps": dterm_deps / (n * LN2)}
    if variant == "unfrozen_mean":
        out["g_eps"] = out["g_eps"] + out["g_vb_eps"]
    out["mse"] = out["mse_sum"] / n
    out["vb"] = out["vb_sum"] / n * vb_scale
    if variant is not None:
        return out

    # ---- bounds: KL
    ml = -x
    r1 = E1 * (U32 * (mn - lv).abs() + ULP * (2 + 1.173 * ml.abs()))
    e_tm = U32 * ((c1 * x0).abs() + (c2 * xt).abs() + tm.abs())
    e_dm = e_tm + e_mean + U32 * dm.abs()
    r2 = 2 * dm.abs() * e_dm * E + e_dm * e_dm * E + e2 * (ULP * (2 + 1.173 * lv.abs()) + 2 * U32)
    s1 = lv - 1
    s2 = s1 - mn
    s3 = s2 + E1
    e_kl = 0.5 * ((1 - E1 - e2).abs() * e_lv + r1 + r2 + U32 * (s1.abs() + s2.abs() + s3.abs() + (s3 + e2).abs()))
    e_gk = 0.5 * ((E1 + e2) * e_lv + r1 + r2 + U32 * ((1 - E1).abs() + (1 - E1 - e2).abs()))
    # ---- bounds: NLL, over the interval arg +- B e_arg
    e_ga = 0.5 * (za.abs() * e_da + da * e_za) + U32 * ga.abs()
    e_gb = 0.5 * (zb.abs() * e_db + db * e_zb) + U32 * gb.abs()
    e_arg = torch.where(lo, e_ca, torch.where(hi, e_cb, e_ca + e_cb) + U32 * arg.abs())
    e_darg = torch.where(lo, e_ga, torch.where(hi, e_gb, e_ga + e_gb + U32 * darg.abs()))
    a_lo, a_hi = arg - B * e_arg, arg + B * e_arg
    T_lo, T_hi = -torch.log(a_hi.clamp_min(CLAMP)), -torch.log(a_lo.clamp_min(CLAMP))
    b_nll = (torch.maximum(T_hi - nll, nll - T_lo)
             + B * (LOGF_ABS + 3 * ULP * torch.maximum(T_lo.abs(), T_hi.abs())))
    den_lo = a_lo.clamp_min(CLAMP)
    corners = torch.stack([-(darg + s * B * e_darg) / dd for s in (-1, 1) for dd in (den_lo, a_hi)])
    r_lo, r_hi = corners.amin(0), corners.amax(0)
    b_live = torch.maximum((r_hi - gn).abs(), (r_lo - gn).abs()) + B * U32 * torch.maximum(r_lo.abs(), r_hi.abs())
    zero = torch.zeros_like(arg)
    b_gn = torch.maximum(torch.where(a_hi > CLAMP, b_live, zero), torch.where(a_lo <= CLAMP, gn.abs(), zero))
    b_term = torch.where(t0, b_nll, B * e_kl)
    b_gterm = torch.where(t0, b_gn, B * e_gk)
    bx, iters = geometry(n)
    acc = B * U32 * (iters + SUM_SLACK + bx)
    out["bnd_mse_sum"] = B * 3 * U32 * sq.sum((1, 2, 3)) + acc * sq.sum((1, 2, 3)) + A * U32 * out["mse_sum"]
    out["bnd_vb_sum"] = b_term.sum((1, 2, 3)) + acc * term.abs().sum((1, 2, 3)) + A * U32 * out["vb_sum"].abs()
    out["bnd_mse"] = out["bnd_mse_sum"] / n + B * 3 * U32 * out["mse"]
    out["bnd_vb"] = out["bnd_vb_sum"] / (n * LN2) + B * 3 * U32 * out["vb"].abs()
    out["bnd_g_eps"] = (A + B * 3) * U32 * out["g_eps"].abs()
    out["bnd_g_var"] = (half_range.abs() / (n * LN2)) * b_gterm + (A + B * 6) * U32 * out["g_var"].abs()
    # torch autograd forms d lv / d v as 0.5 g mx - 0.5 g mn: two products at the tables' magnitude before a subtraction
    # that cancels at the last steps (mx - mn ~ 1e-6 at t = 998).  The kernel subtracts the tables first (exactly, by
    # Sterbenz), so this term belongs to the bound of the oracle's fp32 autograd only (check(..., autograd=True)).
    out["autograd_g_var"] = B * U32 * 0.5 * (mx.abs() + mn.abs()) * gterm.abs() / (n * LN2)
    out["b_term"], out["term"], out["arg"], out["t0"] = b_term, term, arg, t0
    return out


# ------------------------------------------------------------------------------------------------ rejections
REJECT_TS = (0, 1, 10, 500)      # the batch every rejection runs on (sigma = 1: eps far enough that every term is live)
REJECTIONS = {                   # variant: (quantity, t of the samples it is checked on; None = all)
    "clip_pred_x0": ("vb", 500),
    "swap_min_max_log": ("g_var", 10),
    "kl_at_t0": ("vb", 0),
    "swap_hi_branch": ("g_var", 0),
    "no_inv_ln2": ("g_var", 500),
    "flip_dz_dlv": ("g_var", 0),
    "unfrozen_mean": ("g_eps", 1),
    "neighbour_t": ("vb", None),
    "mse_over_2c": ("mse", None),
    "grad_through_clamp": ("g_var", 0),
}


def _where(t):
    ts = t.tolist()
    return {1: lambda i: f"sample {i[0]} (t = {ts[i[0]]})",
            4: lambda i: f"sample {i[0]} (t = {ts[i[0]]}), frame {i[1]}, channel {i[2]}, pixel {i[3]}"}


def check(chk, got, ref, t, what, keys=("mse", "vb", "g_eps", "g_var"), scale=None, autograd=False):
    """Adds every quantity of `got` (per-sample mse / vb, per-element g_eps / g_var; or "mse_sum" / "vb_sum") to the
    Checker against `ref` and its bounds.  `scale` ({"mse": [B], "vb": [B]} fp64 per-sample backward weights) turns the
    gradient references into mo.grad of a weighted backward: one more fp32 product per element.  `autograd`: `got` is
    torch's fp32 autograd of the oracle, whose d lv / d v ordering adds ref["autograd_g_var"]."""
    wh = _where(t)
    for k in keys:
        r, bnd = ref[k], ref["bnd_" + k]
        if autograd and k == "g_var":
            bnd = bnd + ref["autograd_g_var"]
        if scale is not None and k.startswith("g_"):
            w = scale["mse" if k == "g_eps" else "vb"].view(-1, 1, 1, 1)
            r, bnd = r * w, bnd * w.abs() + B * U32 * (r * w).abs()
        g = got[k].reshape(r.shape)
        chk.add(k, what, g, r, bnd, wh[g.dim()])
    return chk


def assert_rejections(got, case, tab, ref):
    """Each wrong variant, as the kernel's (or the oracle's) own result plus (wrong reference - reference) on the samples
    REJECTIONS places it on, must be rejected by the bound."""
    wh = _where(case["t"])
    for variant, (k, t_sel) in REJECTIONS.items():
        wrong = evaluate(case, tab, variant)
        rows = torch.ones_like(case["t"], dtype=torch.bool) if t_sel is None else case["t"] == t_sel
        assert bool(rows.any()), variant
        g = got[k].reshape(ref[k].shape).double()
        rows = rows.view(-1, *([1] * (g.dim() - 1)))
        bnd = torch.where(rows, ref["bnd_" + k], torch.full_like(g, math.inf))     # other samples: anything passes
        m = Checker("wrong")
        m.add(k, variant, g + (wrong[k] - ref[k]), ref[k], bnd, wh[g.dim()])
        assert m.bad, f"{variant}: the bound accepts a wrong {k}"
