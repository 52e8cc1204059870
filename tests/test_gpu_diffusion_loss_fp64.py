"""GPU: the training objective `b200_training_loss` (csrc/sampler.cu) against fp64, element by element: each sample's sum of
squared errors and of variational-bound terms, and dmo, the gradient of the loss with respect to the model output that
seeds every backward kernel.  The reference and the bound are tests/loss_fp64.py (rehearsed on the CPU against the oracle's
own fp32 evaluation by tests/test_loss_bounds.py): the objective in fp64 on the fp32 inputs and tables the kernel reads,
and a first-order error carried through the kernel's fp32 operations, so the check holds where the KL cancels near the
optimum and where the decoder CDFs saturate.

Shapes (B, F, C, H, W) cover part of one block (64 elements per sample), one iteration per thread (768), a partial last
block (10,800), the Latte training latent (65,536: 64 blocks x 4 grid-stride iterations), an image batch of 8 (4,096),
LatteIMG's 16 frames + 8 images (98,304) and 128 frames of 64 x 64 (2,097,152: 128 iterations per thread).  Each sample
has its own t from {0, 1, 2, 10, 500, 998, 999}; eps is 1e-3, 0.1 or 1 from the noise; the t = 0 branches see x0 at
+-fp32(0.999), its fp32 neighbours, +-1 and +-3; var_values include exactly +-1 (and -1 gives lv == min_log) and +-1.5;
one slice puts eps 4 to 10 from the noise, where at t = 0 the CDFs saturate, arg is clamped at 1e-12 and the gradient
must be exactly 0.  One case runs on the respaced "250" schedule.

Each case is checked through the C ABI (sums prefilled with 1e30, dmo with NaN and followed by guard rows; then again
with dmo = NULL) and through `create_diffusion(...).training_losses` with the model output as the model, which adds
q_sample, `_FusedLoss` and its backward: a weighted backward on loss, mse and vb, and train.py's loss.mean().  Ten
wrong variants built from the kernel's own result are rejected where their term is well conditioned.  The worst
err / bound per quantity and regime is printed at the end of the module (pytest -s)."""
import ctypes as C

import pytest
import torch

import loss_fp64 as L
from fp64_bounds import A, U32, Checker, report_worst

pytestmark = pytest.mark.gpu

_WORST = {}
GUARD = 4096
SHAPES = [(3, 1, 4, 4, 4), (4, 3, 4, 8, 8), (3, 5, 4, 18, 30), (2, 16, 4, 32, 32), (8, 1, 4, 32, 32), (2, 24, 4, 32, 32),
          (2, 128, 4, 64, 64)]
SIGMAS = [1e-3, 0.1, 1.0]


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    report_worst(_WORST)


def _diff(respacing):
    from latte_b200.diffusion import create_diffusion
    return create_diffusion(respacing)


def _abi(diff, case, with_dmo=True):
    """b200_training_loss on `case`: sums [2, B] prefilled with 1e30; dmo in a NaN buffer followed by GUARD floats of 7."""
    from latte_b200 import _lib
    mo = case["mo"]
    Bb, Fr, C2 = mo.shape[:3]
    sums = torch.full((2, Bb), 1e30, device=mo.device)
    buf = torch.full((mo.numel() + GUARD,), float("nan"), device=mo.device)
    buf[mo.numel():] = 7.0
    rc = _lib.load().b200_training_loss(
        C.byref(diff._state(mo.device, Bb)[0]), case["t"].data_ptr(), case["x0"].data_ptr(), case["xt"].data_ptr(),
        case["noise"].data_ptr(), mo.data_ptr(), Bb, Fr, C2 // 2, mo[0, 0, 0].numel(), sums.data_ptr(),
        buf.data_ptr() if with_dmo else None, torch.cuda.current_stream(mo.device).cuda_stream)
    _lib.check(rc, "b200_training_loss")
    torch.cuda.synchronize()
    return sums, buf


def _through_module(diff, case, reduce):
    """diff.training_losses with the model output as the model; backward of `reduce(terms)`.  Returns the terms and
    {"mse", "vb", "g_eps", "g_var"} with the gradients split from mo.grad."""
    mo = case["mo"].clone().requires_grad_(True)
    terms = diff.training_losses(lambda x, t, **kw: mo, case["x0"], case["t"], noise=case["noise"])
    reduce(terms).backward()
    Bb, Fr, C2 = mo.shape[:3]
    g = mo.grad.reshape(Bb, Fr, C2, -1)
    return terms, {"mse": terms["mse"].detach(), "vb": terms["vb"].detach(), "g_eps": g[:, :, :C2 // 2],
                   "g_var": g[:, :, C2 // 2:]}


def _run_case(diff, case, regime, what):
    tab = L.tables(diff, case["mo"].device)
    ref = L.evaluate(case, tab)
    t = case["t"]
    Bb = t.numel()
    chk = Checker(regime, _WORST)
    # the C ABI: every dmo element written, nothing past it, sums independent of their prefill
    sums, buf = _abi(diff, case)
    n_mo = case["mo"].numel()
    assert bool((buf[n_mo:] == 7.0).all()), "b200_training_loss wrote past dmo"
    dmo = buf[:n_mo].view(case["mo"].shape).reshape(Bb, case["mo"].shape[1], case["mo"].shape[2], -1)
    C2 = dmo.shape[2]
    got = {"mse_sum": sums[0], "vb_sum": sums[1], "g_eps": dmo[:, :, :C2 // 2], "g_var": dmo[:, :, C2 // 2:]}
    L.check(chk, got, ref, t, f"{what} C ABI", keys=("mse_sum", "vb_sum", "g_eps", "g_var"))
    sums0, _ = _abi(diff, case, with_dmo=False)
    L.check(chk, {"mse_sum": sums0[0], "vb_sum": sums0[1]}, ref, t, f"{what} dmo = NULL", keys=("mse_sum", "vb_sum"))
    # the module: per-sample weights on loss, mse and vb, then train.py's loss.mean()
    w = torch.tensor([1.0, 0.5, 2.0, 1.5] * ((Bb + 3) // 4), device=t.device)[:Bb]
    terms, got = _through_module(diff, case, lambda d: (d["loss"] * w).sum() + 0.25 * d["mse"].sum() + 0.75 * (d["vb"] * w).sum())
    w64 = w.double()
    L.check(chk, got, ref, t, f"{what} training_losses weighted", scale={"mse": w64 + 0.25, "vb": 1.75 * w64})
    loss_ref = ref["mse"] + ref["vb"]
    chk.add("loss", f"{what} training_losses", terms["loss"].detach(), loss_ref,
            ref["bnd_mse"] + ref["bnd_vb"] + A * U32 * loss_ref.abs(), lambda i: f"sample {i[0]} (t = {t[i[0]].item()})")
    _, got = _through_module(diff, case, lambda d: d["loss"].mean())
    inv = torch.full((Bb,), 1.0 / Bb, dtype=torch.float64, device=t.device)
    L.check(chk, got, ref, t, f"{what} training_losses loss.mean()", scale={"mse": inv, "vb": inv})
    chk.done()


@pytest.mark.parametrize("sigma", SIGMAS)
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_training_loss_fp64(dev, shape, sigma):
    diff = _diff("")
    vals = L.t_values(diff.num_timesteps)
    k = SHAPES.index(shape) * 3 + SIGMAS.index(sigma)
    ts = [0] + [vals[1 + (i + k) % (len(vals) - 1)] for i in range(shape[0] - 1)]
    case = L.make_case(diff, shape, ts, sigma, seed=100 * k + 7, device=dev)
    _run_case(diff, case, f"s{sigma:g}", f"{shape} t={ts}")


def test_training_loss_fp64_respaced_250(dev):
    diff = _diff("250")
    ts = list(L.t_values(diff.num_timesteps))
    case = L.make_case(diff, (len(ts), 3, 4, 8, 8), ts, 0.1, seed=250, device=dev)
    _run_case(diff, case, "250 s0.1", f"'250' t={ts}")


def test_training_loss_rejects_wrong_variants(dev):
    """The bound rejects each wrong variant built from the kernel's own result (through training_losses and
    loss.sum().backward(), so the gradients are dmo itself) on the sample where that term is well conditioned."""
    diff = _diff("")
    case = L.make_case(diff, (len(L.REJECT_TS), 2, 4, 8, 8), L.REJECT_TS, 1.0, seed=3, device=dev)
    tab = L.tables(diff, dev)
    ref = L.evaluate(case, tab)
    _, got = _through_module(diff, case, lambda d: d["loss"].sum())
    L.check(Checker("reject-batch", _WORST), got, ref, case["t"], "kernel").done()
    L.assert_rejections(got, case, tab, ref)
