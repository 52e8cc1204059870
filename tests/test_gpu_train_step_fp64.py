"""GPU: the whole native training step pinned to fp64 tensor by tensor and row by row, at the geometry and gradient scale the
models train at.

The native side is `diffusion.training_losses(model, ...)["loss"].mean().backward()` through the modules, as train.py runs
it.  The reference is computed here, on the same weights (the module's parameters in fp64), x0, noise, t, labels, captions
and masks, by the functional oracles in fp64 with sampler_oracle.training_losses and autograd (tests/step_fp64.py; the
CPU suite pins those oracles to the unmodified reference).  Every trainable parameter's every row must satisfy the
budget of tests/step_fp64.py, whose yardstick g_ac is the oracle under the same recipe in torch on the GPU: bf16 autocast on
the fp32 weights (train.py's recipe), or fp16 autocast on the values of the fp16 parameters (`model.half()`).  The native
step must be no less accurate than the reference's own recipe, row for row, to within K = 4.

Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit (the whole file takes about 30 s there):

    case            recipe   worst / budget   largest K a row needs   native / autocast error of the worst tensor
    latte_xl        bf16     0.73             2.88                    0.0108 / 0.0114 of |g64|
    latte_xl        fp16     0.43             1.38
    latte_s_ckpt    bf16     0.60             2.33                    0.0083 / 0.0089
    latte_s_ckpt    fp16     0.27             0.82                    0.0075 / 0.0086
    img_xl          bf16     0.50             1.94                    0.0113 / 0.0120
    img_xl          fp16     0.35             1.14
    t2v_latte1      bf16     0.40             1.50                    0.0145 / 0.0149
    t2v_latte1      fp16     0.51             1.70 (Z0 0.0152)
    t2v_latte1_img  bf16     0.44             1.72                    0.0171 / 0.0179
    t2v_latte1_img  fp16     0.50             1.83 (Z0 0.0067)

With fp16 parameters, LatteT2V's key-bias gradients, which are zero in exact arithmetic, come out at up to 0.0036 of the
median gradient norm: the Z0 of 2^-5 for that recipe covers them with a margin of two.  The weakest rejection is the last
frame missing from LatteT2V's temporal blocks, at 1.36 to 2.0 times the budget.

Cases: n = F C H W = 65536 per sample (16 frames of 4 x 32 x 32 latents; with images, 12 video frames + 4 images), so
d loss / d model output is about 2^-17 as in a real step; t = 0 (decoder NLL) and t = 999 in each batch; depth 2 (one
spatial and one temporal block for Latte, two layer pairs for LatteT2V).  latte_s_ckpt runs with gradient checkpointing.

The budget rejects, in every case and recipe where they apply: two heads' value rows swapped in a qkv weight gradient
(norms equal, so the norm-only comparisons accept it; value rows, because at this scale the fp16 query / key gradients
are mostly subnormal in the native step and in torch alike, and a yardstick that coarse cannot tell their heads apart),
one sample's share missing from the adaLN / scale_shift_table gradients, the last frame missing from the temporal blocks'
gradients, the caption mask ignored in the cross-attention, the images given the other
sample's labels, and with fp16 parameters gradients of the model output below 2^-14 flushed to zero.

Also: a loss scaled by 2^16 (GradScaler, then unscale_) gives the same gradients as the unscaled step; an fp16-autocast step
whose scaled gradients overflow is skipped by the scaler; a second backward through the loss raises."""
import contextlib
import time

import pytest
import torch

import step_fp64 as SB
from test_gpu_train_checkpointing import _deterministic
from oracle import latte_oracle as O
from oracle import t2v_img_oracle as TI
from oracle import t2v_oracle as T

pytestmark = pytest.mark.gpu

PRECISIONS = ["bf16_autocast", "fp16_params"]
LATTE1_LAYER = dict(num_attention_heads=16, attention_head_dim=72, num_layers=2, sample_size=32, video_length=16, caption_channels=4096)
CASES = ["latte_xl", "latte_s_ckpt", "img_xl", "t2v_latte1", "t2v_latte1_img"]


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


class Case:
    """kind, cfg, module, oracle inputs `inp`, x0 / t / noise (CPU) and `native(m, x, t)` in the training_losses layout."""

    def __init__(self, name, dev):
        from latte_b200 import Latte, LatteIMG, LatteT2V
        g = torch.Generator().manual_seed(sum(map(ord, name)))
        self.t = torch.tensor([0, 999])
        if name.startswith(("latte", "img")):
            D, H = (384, 6) if name == "latte_s_ckpt" else (1152, 16)
            I = 4 if name == "img_xl" else 0
            Fr = 16 - I
            self.cfg = O.LatteConfig(input_size=32, hidden_size=D, depth=2, num_heads=H, num_frames=Fr, class_dropout_prob=0.0)
            kw = dict(input_size=32, hidden_size=D, depth=2, num_heads=H, num_frames=Fr, num_classes=101, class_dropout_prob=0.0,
                      extras=2)
            self.m = LatteIMG(**kw) if I else Latte(**kw)
            self.m.load_state_dict(O.make_weights(self.cfg, 21), strict=True)
            self.kind, self.hd = ("img" if I else "latte"), D // H
            self.qkv, self.v0 = "blocks.0.attn.qkv.weight", 2 * D
            self.inp = dict(y=torch.tensor([3, 57], device=dev))
            if I:
                self.inp.update(y_image=torch.tensor([[1, 2, 3, 4], [5, 6, 7, 8]], device=dev), images=I)
            self.x0 = torch.randn(2, 16, 4, 32, 32, generator=g)

            def native(m, x, tt):
                if I:
                    return m(x, tt, y=self.inp["y"], y_image=self.inp["y_image"], use_image_num=I)
                return m(x, tt, y=self.inp["y"])
        else:
            I = 4 if name.endswith("_img") else 0
            self.cfg = T.T2VConfig(**{**LATTE1_LAYER, "video_length": 16 - I})
            self.m = LatteT2V(**{**LATTE1_LAYER, "video_length": 16 - I})
            self.m.load_state_dict(T.make_weights(self.cfg, 17), strict=True)
            self.kind, self.hd = ("t2v_img" if I else "t2v"), 72
            self.qkv, self.v0 = "transformer_blocks.0.attn1.to_v.weight", 0
            if I:
                x, _, text = TI.make_img_inputs(self.cfg, 2, I, 120, 18)
                mask = torch.ones(2, 1 + I, 120)
                mask[1, 0, 12:] = 0                      # the video prompt of sample 1: 12 valid tokens
                mask[0, 2, 40:] = 0
                mask[1, 4, 1:] = 0
            else:
                x, _, text = T.make_inputs(self.cfg, 2, 120, 18)
                mask = torch.ones(2, 120)
                mask[1, 12:] = 0
            self.inp = dict(text=text.to(dev), mask=mask.to(dev), images=I)
            self.x0 = x.permute(0, 2, 1, 3, 4).contiguous()

            def native(m, x, tt):
                return m(x.permute(0, 2, 1, 3, 4), tt, encoder_hidden_states=self.inp["text"],
                         encoder_attention_mask=self.inp["mask"], use_image_num=I).sample.permute(0, 2, 1, 3, 4)
        self.noise = torch.randn(self.x0.shape, generator=g)
        self.native = native
        self.m = self.m.to(dev).train()
        if name.endswith("_ckpt"):
            self.m.enable_gradient_checkpointing()

    def step(self, dev, autocast=None, scaler=None):
        """One native step: zero_grad, training_losses under `autocast`, backward (of the scaled loss with `scaler`)."""
        from latte_b200.diffusion import create_diffusion
        self.m.zero_grad(set_to_none=True)
        d = create_diffusion(timestep_respacing="")
        ctx = torch.autocast("cuda", dtype=autocast) if autocast is not None else contextlib.nullcontext()
        with ctx:
            loss = d.training_losses(lambda x, tt, **kw: self.native(self.m, x, tt), self.x0.to(dev), self.t.to(dev),
                                     noise=self.noise.to(dev))["loss"].mean()
        (scaler.scale(loss) if scaler is not None else loss).backward()
        torch.cuda.synchronize()
        return loss

    def grads(self):
        return {k: p.grad.detach().clone() for k, p in self.m.named_parameters() if p.requires_grad}

    def sd(self, dev, dtype):
        train = {k for k, p in self.m.named_parameters() if p.requires_grad}
        return {k: v.detach().to(dev, dtype).requires_grad_(k in train) for k, v in self.m.state_dict().items()
                if v.is_floating_point()}

    def oracle(self, dev, dtype, variant=None, **kw):
        sd = self.sd(dev, dtype)
        fwd = SB.oracle_forward(self.kind, self.cfg, sd, dtype, self.inp, variant)
        return SB.oracle_step(fwd, sd, self.x0, self.t, self.noise, dev, **kw)


def _rejected(what, got, g64, gac, budget, wrong, names, missed):
    bad = {n: (got[n].double() + (wrong[n] - g64[n])).to(got[n].dtype) for n in names}
    n, w = SB.worst(SB.check(bad, g64, gac, budget, names))
    print(f"    rejects {what}: {n} row {w.row} at {w.ratio:.3g} x its budget")
    if w.ratio <= 1.0:
        missed.append((what, n, w))


def _rel(a, b):
    return ((a.double() - b).norm() / b.norm().clamp_min(1e-300)).item()


@pytest.mark.parametrize("recipe", PRECISIONS)
@pytest.mark.parametrize("case", CASES)
def test_step_within_fp64_budget(dev, case, recipe):
    t0 = time.perf_counter()
    c = Case(case, dev)
    if recipe == "fp16_params":
        c.m.half()
    c.step(dev, autocast=torch.bfloat16 if recipe == "bf16_autocast" else None)
    got = c.grads()
    adaln = [k for k in got if SB.is_adaln(k)]
    g64, g0 = c.oracle(dev, torch.float64, sample0=adaln)
    gac = c.oracle(dev, torch.float32, autocast=torch.bfloat16 if recipe == "bf16_autocast" else torch.float16)
    assert set(got) == set(g64)
    budget = SB.BUDGET[recipe]
    res = SB.check(got, g64, gac, budget)
    n, w = SB.worst(res)
    print(f"\n{case} {recipe}: {len(res)} parameters, worst {n} row {w.row} at {w.ratio:.3g} x its budget (K, A, Z, Z0 = "
          f"{budget[0]:g}, {budget[1]:g}, {budget[2]:.3g}, {budget[3]:.3g}); largest K a row needs {max(v.need_k for v in res.values()):.3g}, "
          f"largest Z0 {max(v.need_z for v in res.values()):.3g}")
    for k, v in sorted(res.items(), key=lambda kv: -kv[1].ratio)[:3]:
        print(f"    {k}: row {v.row}: |err| {v.e:.3g}, a {v.a:.3g}, |g64| {v.r:.3g}; tensor: native {_rel(got[k], g64[k]):.3g}"
              + (f", autocast {_rel(gac[k], g64[k]):.3g}" if gac is not None else "") + " of |g64|")
    over = sorted(((v.ratio, k, v.row) for k, v in res.items() if v.ratio > 1.0), reverse=True)[:8]
    missed = []

    # two heads' rows swapped: the same norm, so every norm comparison accepts it
    bad = dict(got)
    bad[c.qkv] = SB.swap_heads(got[c.qkv], c.hd, c.v0)
    assert abs(bad[c.qkv].double().norm().item() - got[c.qkv].double().norm().item()) <= 1e-6 * got[c.qkv].double().norm().item()
    _rejected(f"two swapped heads in {c.qkv}", got, g64, gac, budget, {c.qkv: g64[c.qkv] + (bad[c.qkv].double() - got[c.qkv])},
              [c.qkv], missed)
    _rejected("sample 1 missing from the adaLN gradients", got, g64, gac, budget, g0, adaln, missed)
    with SB.last_frame_missing():
        wrong = c.oracle(dev, torch.float64)
    _rejected("the last frame missing from the temporal blocks", got, g64, gac, budget, wrong,
              [n for n in got if SB.is_temporal(n)], missed)
    if c.kind.startswith("t2v"):
        wrong = c.oracle(dev, torch.float64, variant="no_mask")
        _rejected("the caption mask ignored", got, g64, gac, budget, wrong, [n for n in got if ".attn2." in n], missed)
    if c.kind == "img":
        wrong = c.oracle(dev, torch.float64, variant="other_labels")
        _rejected("the images given the other sample's labels", got, g64, gac, budget, wrong, list(got), missed)
    if recipe == "fp16_params":
        wrong = c.oracle(dev, torch.float64, hook=SB.flush(2.0 ** -14))
        _rejected("output gradients below 2^-14 flushed", got, g64, gac, budget, wrong, list(got), missed)
    print(f"    {time.perf_counter() - t0:.1f} s")
    assert not over, over
    assert not missed, missed


# ------------------------------------------------------------------------------------------------------------ loss scaling
@pytest.mark.parametrize("case", ["latte_xl", "t2v_latte1"])
def test_power_of_two_loss_scale_is_exact(dev, case):
    """bf16 autocast: the loss scaled by 2^16 and unscaled again gives the unscaled step's gradients -- bit for bit where no
    float atomic is involved, within two plain runs' spread (or 1e-5 of the norm) elsewhere.  Scaling by a power of two
    commutes with every rounding while nothing is subnormal or overflows."""
    c = Case(case, dev)
    c.step(dev, torch.bfloat16)
    g1 = c.grads()
    c.step(dev, torch.bfloat16)
    g2 = c.grads()
    scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 16)
    opt = torch.optim.SGD(c.m.parameters(), lr=0.0)
    c.step(dev, torch.bfloat16, scaler)
    scaler.unscale_(opt)
    gs = c.grads()
    det = [k for k in g1 if _deterministic(k)]
    same = [k for k in det if torch.equal(gs[k], g1[k])]
    med = torch.tensor([g.double().norm().item() for g in g1.values()]).median().item()
    worst = 0.0
    for k in g1.keys() - set(det):
        diff, spread = (gs[k].double() - g1[k].double()).norm().item(), (g2[k].double() - g1[k].double()).norm().item()
        floor = 1e-5 * max(g1[k].double().norm().item(), med)
        worst = max(worst, diff / floor)
        assert diff <= max(spread, floor), (k, diff, spread, floor)
    print(f"\n{case}: 2^16-scaled step: {len(same)} of {len(det)} GEMM weight gradients bit-identical, "
          f"{len(g1) - len(det)} others within {worst:.3g} of their floor")
    assert len(same) == len(det), sorted(set(det) - set(same))[:8]


def test_fp16_overflow_skips_the_step(dev):
    """fp32 parameters under torch.autocast(float16) (fp16 operands): a 2^40 loss scale makes d loss / d output about 2^23,
    past fp16's 65504.  The overflow must reach .grad as inf / NaN, so that scaler.step skips the update, the parameters stay
    as they were and the scale is halved."""
    c = Case("latte_s_ckpt", dev)
    c.m.disable_gradient_checkpointing()
    before = {k: p.detach().clone() for k, p in c.m.named_parameters()}
    opt = torch.optim.AdamW(c.m.parameters(), lr=1e-3)
    scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 40)
    c.step(dev, torch.float16, scaler)
    bad = [k for k, g in c.grads().items() if not torch.isfinite(g).all()]
    scaler.step(opt)
    scaler.update()
    print(f"\nfp16 autocast at scale 2^40: {len(bad)} gradients non-finite; step skipped, scale now 2^"
          f"{torch.log2(torch.tensor(scaler.get_scale())).item():.0f}")
    assert bad
    assert all(torch.equal(p, before[k]) for k, p in c.m.named_parameters())
    assert scaler.get_scale() == 2.0 ** 39


# ------------------------------------------------------------------------------------------------------------ second backward
class _Toy(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.a = torch.nn.Parameter(torch.tensor(0.7))
        self.b = torch.nn.Parameter(torch.tensor(-0.3))

    def forward(self, x, t):
        return torch.cat((torch.tanh(self.a * x), torch.sin(self.b * x)), dim=2)


def test_second_backward_through_the_loss(dev):
    """A second backward through the fused loss node behaves as one through torch's own loss expressions: through a freed
    graph it raises autograd's error; through a retained graph it adds the gradient again.  The native modules refuse a
    second backward of their step either way."""
    from latte_b200 import Latte
    from latte_b200.diffusion import create_diffusion
    d = create_diffusion(timestep_respacing="")
    g = torch.Generator().manual_seed(2)
    x0, noise = torch.randn(2, 4, 4, 16, 16, generator=g).to(dev), torch.randn(2, 4, 4, 16, 16, generator=g).to(dev)
    t = torch.tensor([0, 500], device=dev)

    toy = _Toy().to(dev)
    for retain in (False, True):
        toy.zero_grad(set_to_none=True)
        loss = d.training_losses(toy, x0, t, noise=noise)["loss"].mean()
        loss.backward(retain_graph=retain)
        first = [p.grad.clone() for p in toy.parameters()]
        if not retain:
            with pytest.raises(RuntimeError, match="backward through the graph a second time"):
                loss.backward()
            continue
        loss.backward()
        assert all(torch.equal(p.grad, 2 * f) for p, f in zip(toy.parameters(), first))

    cfg = O.make_config("Latte-tiny64/2", input_size=16, num_frames=4, class_dropout_prob=0.0)
    m = Latte(input_size=16, hidden_size=128, depth=2, num_heads=2, num_frames=4, num_classes=101, extras=2, class_dropout_prob=0.0)
    m.load_state_dict(O.make_weights(cfg, 21), strict=True)
    m = m.to(dev).train()
    y = torch.tensor([3, 57], device=dev)
    for retain in (False, True):
        m.zero_grad(set_to_none=True)
        loss = d.training_losses(m, x0, t, dict(y=y), noise=noise)["loss"].mean()
        loss.backward(retain_graph=retain)
        with pytest.raises(RuntimeError, match="backward called twice" if retain else "backward through the graph a second time"):
            loss.backward()
