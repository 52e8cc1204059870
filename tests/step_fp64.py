"""Row-by-row gradient budget of a whole training step against fp64, shared by test_gpu_train_step_fp64.py (the native step
at the geometry and gradient scale the models train at) and test_train_step_bounds.py (the same machinery on the CPU).

For every trainable parameter and every row r (a dim-0 slice of a weight, a 64-element chunk of a vector; R rows):

    |g_nat[r] - g64[r]| <= K a[r] + A u |g64[r]| + (Z |g64|_F + Z0 m) / sqrt(R)
    a[r] = max(|g_ac[r] - g64[r]|, rho max(|g64[r]|, |g64|_F / sqrt(R))),  rho = |g_ac - g64|_F / |g64|_F

g64 is autograd of the functional oracle in fp64 on the same weights and inputs, g_ac the oracle under the reference's own
mixed-precision recipe (bf16 autocast on fp32 weights), u the unit roundoff of the gradient's type, m the median of the
parameters' fp64 gradient norms.

* a[r] is the recipe's own error on row r, or its relative error on the whole tensor times the row's norm if that is
  larger.  The gradients of the adaLN, timestep-embedder and label-embedder weights are outer products of B per-sample
  vectors (B = 2 in the GPU cases), so each of their rows carries the rounding of just B scalars, in the native step and
  in g_ac alike.  The per-row ratio of two such errors is a ratio of two scalars of the same size and is heavy-tailed:
  over thousands of rows, a few land where g_ac happens to be almost exact.  With a[r] = |g_ac[r] - g64[r]| alone, those
  rows needed K = 18.3 (latte_xl), although the native error of every such tensor is no larger than g_ac's.
* The Z0 term covers gradients that are rounding noise in exact arithmetic (LatteT2V's key biases: softmax is
  shift-invariant).  Their own norm is no scale for that noise, so this floor uses the median gradient norm m; the plain
  Z |g64|_F / sqrt(R) term alone would require them to be exactly zero.  test_gpu_train_checkpointing.py floors the same
  way.
* For fp16 parameters (`model.half()`) g_ac is the oracle on the same fp16 values under fp16 autocast: fp16 operands,
  as the native step has.  The oracle in fp16 throughout is no yardstick at d loss / d output of about 2^-17: it loses
  most of every weight gradient to underflow.

The wrong results the budget must reject are built from fp64 oracle variants as got + (g_wrong - g64), or by permuting got."""
import collections
import contextlib
import math

import torch

from oracle import latte_img_oracle as LI
from oracle import latte_oracle as O
from oracle import sampler_oracle as S
from oracle import t2v_img_oracle as TI
from oracle import t2v_oracle as T

U = {torch.float32: 2.0 ** -24, torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
# (K, A, Z, Z0) per recipe, set from a run of tests/test_gpu_train_step_fp64.py on an NVIDIA H100 80GB HBM3 at a 700 W power
# limit; the figures it printed are in that file's docstring
BUDGET = {"bf16_autocast": (4.0, 1.0, 2.0 ** -10, 2.0 ** -10), "fp16_params": (4.0, 1.0, 2.0 ** -10, 2.0 ** -5)}

Row = collections.namedtuple("Row", "ratio row need_k need_z e a r")


def rows(g):
    g = g.double()
    if g.dim() >= 2:
        return g.reshape(g.shape[0], -1)
    return torch.nn.functional.pad(g.reshape(-1), (0, (-g.numel()) % 64)).reshape(-1, 64)


def ratio(got, g64, gac, budget, m):
    """The worst row of one parameter: err / budget, its index, the K and the Z at which the parameter's worst rows would sit
    on their budgets (Z: the Z0 coefficient), and that row's error e, yardstick a and fp64 norm r."""
    k, A, z, z0 = budget
    e = rows(got.double() - g64).norm(dim=1)
    r = rows(g64).norm(dim=1)
    if gac is not None and k > 0:
        d = rows(gac.double() - g64)
        rho = d.norm() / g64.double().norm().clamp_min(1e-300)
        a = torch.maximum(d.norm(dim=1), rho * r.clamp_min(g64.double().norm().item() / math.sqrt(r.numel())))
    else:
        a = torch.zeros_like(r)
    n64 = g64.double().norm().item()
    floor = m / math.sqrt(r.numel())
    rest = A * U[got.dtype] * r + (z * n64 + z0 * m) / math.sqrt(r.numel())
    b = k * a + rest
    q = torch.where(b > 0, e / b.clamp_min(1e-300), torch.where(e > 0, math.inf, 0.0))
    q = torch.where(torch.isfinite(e), q, math.inf)
    i = int(torch.argmax(q))
    nk = torch.where(a > 0, (e - rest) / a.clamp_min(1e-300), torch.where(e > rest, math.inf, 0.0))
    nz = (e - k * a - A * U[got.dtype] * r - z * n64 / math.sqrt(r.numel())) / floor if floor > 0 else torch.zeros_like(e)
    fin = lambda v: torch.where(torch.isfinite(e), v, math.inf)   # noqa: E731
    return Row(float(q[i]), i, float(fin(nk).max()), float(fin(nz).max()), float(e[i]), float(a[i]), float(r[i]))


def check(got, g64, gac, budget, names=None):
    """{name: Row} over `names` (default: every parameter of g64); gac None for a budget with K = 0."""
    m = torch.tensor([g.double().norm().item() for g in g64.values()]).median().item()
    return {n: ratio(got[n], g64[n], None if gac is None else gac[n], budget, m) for n in (names if names is not None else g64)}


def worst(res):
    n = max(res, key=lambda k: res[k].ratio)
    return n, res[n]


# ------------------------------------------------------------------------------------------------------------ the oracle
def oracle_forward(kind, cfg, sd, dtype, inp, variant=None):
    """fn(x, t) -> model output in the (B, F, 2C, H, W) layout training_losses takes.  inp: y, y_image, images, text, mask.
    variant: None, "no_mask" (the caption mask ignored) or "other_labels" (each sample's images get the next sample's
    labels); "last_frame" is `last_frame_missing` around the call."""
    mask = None if variant == "no_mask" else inp.get("mask")
    if kind == "latte":
        return lambda x, t: O.latte_forward(sd, cfg, x, t, inp.get("y"), dtype)
    if kind == "img":
        yi = inp["y_image"].roll(1, 0) if variant == "other_labels" else inp["y_image"]
        return lambda x, t: LI.latte_img_forward(sd, cfg, x, t, inp["y"], yi, inp["images"], training=True, dtype=dtype)
    cf = lambda x: x.permute(0, 2, 1, 3, 4)                  # noqa: E731  (B, F, C, H, W) <-> (B, C, F, H, W)
    if kind == "t2v":
        return lambda x, t: cf(T.t2v_forward(sd, cfg, cf(x), t, inp["text"], dtype, True, mask))
    return lambda x, t: cf(TI.t2v_train_forward(sd, cfg, cf(x), t, inp["text"], inp["images"], mask, dtype))


@contextlib.contextmanager
def last_frame_missing():
    """The temporal blocks' parameters get no gradient from the last video frame: that frame's rows of each temporal block's
    output are recomputed with the parameters detached (same values, the rest of the graph intact)."""
    def cut(block, temporal):
        def run(sd, i, x, *a):
            out = block(sd, i, x, *a)
            if not temporal(i):
                return out
            frozen = block({k: v.detach() for k, v in sd.items()}, i, x, *a)
            return torch.cat((out[:, :-1], frozen[:, -1:]), 1)
        return run
    saved = [(O, "transformer_block"), (LI, "transformer_block"), (T, "temporal_block"), (TI, "temporal_block")]
    old = [getattr(mod, n) for mod, n in saved]
    O.transformer_block = LI.transformer_block = cut(old[0], lambda i: i % 2 == 1)
    T.temporal_block = TI.temporal_block = cut(old[2], lambda i: True)
    try:
        yield
    finally:
        for (mod, n), f in zip(saved, old):
            setattr(mod, n, f)


def oracle_step(fwd, sd, x0, t, noise, dev, autocast=None, sample0=None, hook=None):
    """sampler_oracle.training_losses(...)["loss"].mean() around fwd on `dev` (the objective on the CPU, in the model
    output's precision: fp64 for an fp64 model, fp32 otherwise, as the native step takes mo.float()); autograd gradients of
    every leaf of sd that requires grad.  sample0: names whose gradient of sample 0's share of the loss alone is returned as
    well.  hook: applied to the gradient of the model output."""
    s = S.make_schedule("")

    def model(x, tt, **kw):
        ctx = torch.autocast(dev.type, dtype=autocast) if autocast is not None else contextlib.nullcontext()
        with ctx:
            mo = fwd(x.to(dev), tt.to(dev))
        if hook is not None:
            mo.register_hook(hook)
        return mo.to("cpu", torch.float64 if mo.dtype == torch.float64 else torch.float32)
    terms = S.training_losses(s, model, x0.cpu(), t.cpu(), noise.cpu())
    leaves = {k: v for k, v in sd.items() if v.requires_grad}
    loss = terms["loss"].mean()
    g = dict(zip(leaves, torch.autograd.grad(loss, list(leaves.values()), retain_graph=sample0 is not None)))
    if sample0 is None:
        return g
    g0 = torch.autograd.grad(terms["loss"][0] / len(t), [leaves[k] for k in sample0])
    return g, dict(zip(sample0, g0))


def swap_heads(g, hd, start=0):
    """Rows of heads 0 and 1 from row `start` on exchanged (same norm)."""
    w = g.clone()
    a, b, c = start, start + hd, start + 2 * hd
    w[a:b], w[b:c] = g[b:c], g[a:b]
    return w


def flush(limit):
    return lambda g: torch.where(g.abs() < limit, torch.zeros_like(g), g)


def is_adaln(n):
    return any(s in n for s in ("adaLN_modulation", "scale_shift_table", "adaln_single.linear"))


def is_temporal(n):
    if n.startswith("temporal_transformer_blocks."):
        return True
    return n.startswith("blocks.") and int(n.split(".")[1]) % 2 == 1
