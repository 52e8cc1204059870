"""CPU, no GPU: the training objective's fp64 reference and error bound (tests/loss_fp64.py) before they are applied to
`b200_training_loss`.  (1) The closed-form values and gradients equal torch.autograd of oracle/sampler_oracle.training_losses
run in fp64 (its `_extract` rounds the tables to fp32 and promotes them, as the kernel reads them).  (2) The bound accepts
the oracle's own fp32 evaluation -- values, and gradients from autograd -- in every regime the GPU test runs: t in
{0, 1, 2, 10, 500, 998, 999}, eps at 1e-3, 0.1 and 1 from the noise, the planted x0 and var_values and the saturated
t = 0 slice, on the full and the respaced "250" schedule; so the bound is not tighter than fp32 itself.  (3) The bound
rejects every wrong variant the GPU test rejects, built from the oracle's fp32 result.  The worst err / bound per
quantity and regime is printed at the end of the module (pytest -s)."""
import math

import numpy as np
import pytest
import torch

import loss_fp64 as L
from fp64_bounds import Checker, report_worst

_WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    report_worst(_WORST)


def _diff(respacing):
    from latte_b200.diffusion import create_diffusion
    from oracle import sampler_oracle as O
    return create_diffusion(respacing), O.make_schedule(respacing)


def _oracle(sched, case, dtype):
    """oracle training_losses in `dtype` with autograd: per-sample mse / vb, and d loss.sum() / d model output split into
    the eps channels (d mse / d eps: the VB term sees a detached eps) and the variance channels (d vb / d v)."""
    from oracle import sampler_oracle as O
    old = torch.get_default_dtype()
    torch.set_default_dtype(dtype)
    try:
        mo = case["mo"].to(dtype).clone().requires_grad_(True)
        out = O.training_losses(sched, lambda x, t, **kw: mo, case["x0"].to(dtype), case["t"], case["noise"].to(dtype))
        out["loss"].sum().backward()
    finally:
        torch.set_default_dtype(old)
    Bb, Fr, C2 = mo.shape[:3]
    g = mo.grad.reshape(Bb, Fr, C2, -1)
    return {"mse": out["mse"].detach(), "vb": out["vb"].detach(), "g_eps": g[:, :, :C2 // 2], "g_var": g[:, :, C2 // 2:]}


@pytest.mark.parametrize("respacing", ["", "250"])
def test_closed_form_matches_oracle_autograd_fp64(respacing):
    """Away from the branch thresholds and the clamp, the fp64 closed form (values, d mse / d eps, d vb / d v, and the
    d vb / d eps an unfrozen mean would add) equals the oracle's fp64 autograd to ~1e-12."""
    from oracle import sampler_oracle as O
    diff, sched = _diff(respacing)
    ts = list(L.t_values(diff.num_timesteps))
    g = torch.Generator().manual_seed(5)
    shape = (len(ts), 2, 4, 4, 6)
    x0 = torch.randn(shape, generator=g) * 0.8
    x0 = torch.where(((x0.abs() - L.THR).abs() < 1e-2), torch.full_like(x0, 0.5), x0)
    noise = torch.randn(shape, generator=g)
    eps = noise + 0.1 * torch.randn(shape, generator=g)
    v = torch.rand(shape, generator=g) * 3 - 1.5
    mo = torch.cat([eps, v], 2)
    t = torch.tensor(ts)
    torch.set_default_dtype(torch.float64)
    try:
        xt64 = O.q_sample(sched, x0.double(), t, noise.double())
        mo2 = mo.double().requires_grad_(True)
        O.vb_terms_bpd(sched, mo2, x0.double(), xt64, t).sum().backward()
    finally:
        torch.set_default_dtype(torch.float32)
    got = _oracle(sched, {"mo": mo, "x0": x0, "t": t, "noise": noise}, torch.float64)
    ref = L.evaluate({"x0": x0, "xt": xt64, "noise": noise, "mo": mo, "t": t}, L.tables(diff, torch.device("cpu")))
    assert bool((ref["arg"][ref["t0"].expand_as(ref["arg"])] > 1e-6).all())
    got["g_vb_eps"] = mo2.grad.reshape(len(ts), 2, 8, -1)[:, :, :4]
    # d vb / d v = 0.5 (1 - exp(mn - lv) - e2) (...): at the last steps lv - mn ~ 1e-7 and the oracle's own fp64 autograd of
    # the plain expression keeps only ~1e-16 of the 0.5 (mx - mn) / (n ln 2) it cancels from; that is its scale
    tab = L.tables(diff, torch.device("cpu")).double()[:, t]
    cancel = 0.5 * (tab[5] - tab[4]).abs() / (math.prod(shape[1:]) * L.LN2)
    for k in ("mse", "vb", "g_eps", "g_var", "g_vb_eps"):
        a, b = got[k].reshape(len(ts), -1), ref[k].reshape(len(ts), -1)
        scale = b.abs().amax(1)
        if k == "g_var":
            scale = torch.maximum(scale, cancel)
        rel = ((a - b).abs().amax(1) / scale).max().item()
        assert rel < 1e-12, (k, rel)


CASES = [((3, 1, 4, 4, 4), ""), ((4, 3, 4, 8, 8), ""), ((7, 2, 4, 6, 10), ""), ((7, 1, 4, 8, 8), "250")]


@pytest.mark.parametrize("sigma", [1e-3, 0.1, 1.0])
@pytest.mark.parametrize("shape,respacing", CASES)
def test_bound_accepts_oracle_fp32(shape, respacing, sigma):
    diff, sched = _diff(respacing)
    vals = L.t_values(diff.num_timesteps)
    ts = [0] + [vals[(i + shape[0]) % len(vals)] for i in range(1, shape[0])]
    case = L.make_case(diff, shape, ts, sigma, seed=sum(shape) + int(sigma * 1000), device=torch.device("cpu"))
    from oracle import sampler_oracle as O
    assert torch.equal(case["xt"], O.q_sample(sched, case["x0"], case["t"], case["noise"]))
    got = _oracle(sched, case, torch.float32)
    ref = L.evaluate(case, L.tables(diff, torch.device("cpu")))
    L.check(Checker(f"s{sigma:g}", _WORST), got, ref, case["t"], f"oracle fp32 {shape} '{respacing}'", autograd=True).done()


def test_bound_rejects_wrong_variants():
    diff, sched = _diff("")
    case = L.make_case(diff, (len(L.REJECT_TS), 2, 4, 8, 8), L.REJECT_TS, 1.0, seed=3, device=torch.device("cpu"))
    got = _oracle(sched, case, torch.float32)
    tab = L.tables(diff, torch.device("cpu"))
    ref = L.evaluate(case, tab)
    L.check(Checker("reject-batch", _WORST), got, ref, case["t"], "oracle fp32", autograd=True).done()
    L.assert_rejections(got, case, tab, ref)


def test_planted_values_straddle_the_thresholds():
    """The planted x0 sit on both sides of fp32(+-0.999) and pick different branches, as torch's fp32 comparison does."""
    p = torch.tensor(L.planted_x0())
    assert float(np.float32(0.999)) == L.THR
    assert int((p > L.THR).sum()) == 3 and int((p < -L.THR).sum()) == 3
    assert int(((p.abs() <= L.THR) & (p.abs() > 0.99)).sum()) == 4
