"""CPU: the machinery of test_gpu_train_step_fp64.py rehearsed at the train_tiny64 shape.

* The fp64 oracle step (oracle forward + sampler_oracle.training_losses + autograd, tests/step_fp64.py) reproduces the
  gradients the unmodified reference produced in fp32 (tests/golden/train_tiny64.npz): its full `grad::` tensors and the norm
  of every parameter's gradient.  This pins the fp64 reference the GPU test measures the native step against.
* Every wrong result that test rejects exceeds the budget at the chosen K and Z here too, with a CPU bf16-autocast run of the
  oracle as g_ac and as the result the wrong gradient is added to: two heads' rows swapped in a qkv weight gradient (which a
  norm comparison accepts), one sample missing from the adaLN gradients, the last frame missing from the temporal blocks,
  the caption mask ignored in the cross-attention, the images given the other sample's labels, and gradients of the model
  output below 2^-14 flushed to zero."""
import os

import numpy as np
import pytest
import torch

import step_fp64 as SB
from oracle import latte_oracle as O
from oracle import t2v_img_oracle as TI
from oracle import t2v_oracle as T

CPU = torch.device("cpu")
BF = SB.BUDGET["bf16_autocast"]


def _sd(weights, dtype, frozen=("pos_embed", "temp_embed")):
    return {k: v.to(dtype).requires_grad_(k not in frozen) for k, v in weights.items()}


def _steps(kind, cfg, weights, x0, t, noise, inp, sample0=None):
    """(g64, g_ac[, sample 0's g64]) of one oracle step."""
    s64 = _sd(weights, torch.float64)
    out = SB.oracle_step(SB.oracle_forward(kind, cfg, s64, torch.float64, inp), s64, x0, t, noise, CPU, sample0=sample0)
    s32 = _sd(weights, torch.float32)
    gac = SB.oracle_step(SB.oracle_forward(kind, cfg, s32, torch.float32, inp), s32, x0, t, noise, CPU, autocast=torch.bfloat16)
    return (out[0], gac, out[1]) if sample0 else (out, gac)


def _variant(kind, cfg, weights, x0, t, noise, inp, variant=None, hook=None):
    s64 = _sd(weights, torch.float64)
    return SB.oracle_step(SB.oracle_forward(kind, cfg, s64, torch.float64, inp, variant), s64, x0, t, noise, CPU, hook=hook)


def _rejects(got, g64, gac, wrong, names):
    bad = {n: (got[n].double() + (wrong[n] - g64[n])).to(got[n].dtype) for n in names}
    n, w = SB.worst(SB.check(bad, g64, gac, BF, names))
    assert w.ratio > 1.0, (n, w)


@pytest.fixture(scope="module")
def tiny64(golden_dir):
    g = np.load(os.path.join(golden_dir, "train_tiny64.npz"))
    cfg = O.make_config("Latte-tiny64/2", input_size=16, num_frames=8)
    w = O.make_weights(cfg, 21)
    x0, noise, t, y = (torch.from_numpy(g[k]) for k in ("x0", "noise", "t", "y"))
    adaln = [k for k in w if SB.is_adaln(k)]
    g64, gac, g0 = _steps("latte", cfg, w, x0, t, noise, dict(y=y), sample0=adaln)
    return g, cfg, w, (x0, t, noise, dict(y=y)), g64, gac, g0


def test_fp64_oracle_step_matches_reference_gradients(tiny64):
    """The fp64 model under the reference's fp32 objective reproduces the golden to 1e-5; under the fp64 objective the budget
    uses it differs from the golden by up to 1.5 % (element max): at t = 0 the decoder NLL takes logs of differences of
    nearly equal CDFs, which fp32 resolves poorly (the fp64 objective itself is pinned in test_loss_bounds.py)."""
    g, cfg, w, (x0, t, noise, inp), _, _, _ = tiny64
    s64 = _sd(w, torch.float64)
    fwd = SB.oracle_forward("latte", cfg, s64, torch.float64, inp)
    g64 = SB.oracle_step(lambda x, tt: fwd(x, tt).float(), s64, x0, t, noise, CPU)
    names = [str(n) for n in g["grad_names"]]
    assert sorted(names) == sorted(g64)
    for k, want in zip(names, g["grad_norms"]):
        got = g64[k].norm().item()
        assert abs(got - want) <= 1e-5 * want + 1e-9, (k, got, want)
    full = [key for key in g.files if key.startswith("grad::")]
    assert full
    for key in full:
        ref = torch.from_numpy(g[key]).double()
        err = (g64[key[6:]] - ref).abs().max().item()
        assert err <= 1e-5 * ref.abs().max().item() + 1e-9, (key, err)


def test_scaled_gradient_is_rejected(tiny64):
    """Every parameter's gradient 10 % too large exceeds the budget (bf16 autocast is within about 1 % of fp64 here)."""
    _, _, _, _, g64, gac, _ = tiny64
    res = SB.check({k: (v * 1.1).float() for k, v in g64.items()}, g64, gac, BF)
    assert all(w.ratio > 1.0 for w in res.values()), sorted((w.ratio, k) for k, w in res.items())[:4]


def test_budget_rejects_swapped_heads(tiny64):
    _, cfg, _, _, g64, gac, _ = tiny64
    n = "blocks.0.attn.qkv.weight"
    bad = dict(gac)
    bad[n] = SB.swap_heads(gac[n], cfg.head_dim)
    # a comparison of norms cannot see it
    assert abs(bad[n].double().norm().item() - gac[n].double().norm().item()) <= 1e-12 * gac[n].double().norm().item()
    assert SB.check(bad, g64, gac, BF, [n])[n].ratio > 1.0


def test_budget_rejects_missing_sample_in_adaln(tiny64):
    _, _, _, _, g64, gac, g0 = tiny64
    _rejects(gac, g64, gac, g0, list(g0))


def test_budget_rejects_missing_last_frame_in_temporal_blocks(tiny64):
    _, cfg, w, (x0, t, noise, inp), g64, gac, _ = tiny64
    with SB.last_frame_missing():
        wrong = _variant("latte", cfg, w, x0, t, noise, inp)
    _rejects(gac, g64, gac, wrong, [k for k in g64 if SB.is_temporal(k)])


def test_budget_rejects_flushed_output_gradient(tiny64):
    _, cfg, w, (x0, t, noise, inp), g64, gac, _ = tiny64
    wrong = _variant("latte", cfg, w, x0, t, noise, inp, hook=SB.flush(2.0 ** -14))
    _rejects(gac, g64, gac, wrong, list(g64))


def test_budget_rejects_ignored_caption_mask():
    cfg = T.T2VConfig(num_attention_heads=2, attention_head_dim=64, num_layers=1, sample_size=16, video_length=8,
                      caption_channels=256)
    w = T.make_weights(cfg, 9)
    x, t, text = T.make_inputs(cfg, 2, 20, 10)
    mask = torch.ones(2, 20)
    mask[1, 12:] = 0
    gen = torch.Generator().manual_seed(3)
    x0, noise = x.permute(0, 2, 1, 3, 4).contiguous(), torch.randn(2, 8, 4, 16, 16, generator=gen)
    t = torch.tensor([0, 999])
    inp = dict(text=text, mask=mask)
    g64, gac = _steps("t2v", cfg, w, x0, t, noise, inp)
    wrong = _variant("t2v", cfg, w, x0, t, noise, inp, variant="no_mask")
    _rejects(gac, g64, gac, wrong, [k for k in g64 if ".attn2." in k])


def test_budget_rejects_other_samples_image_labels():
    cfg = O.make_config("Latte-tiny64/2", input_size=16, num_frames=4, class_dropout_prob=0.0)
    w = O.make_weights(cfg, 21)
    gen = torch.Generator().manual_seed(4)
    x0, noise = torch.randn(2, 6, 4, 16, 16, generator=gen), torch.randn(2, 6, 4, 16, 16, generator=gen)
    t = torch.tensor([0, 999])
    inp = dict(y=torch.tensor([3, 57]), y_image=torch.tensor([[1, 2], [3, 4]]), images=2)
    g64, gac = _steps("img", cfg, w, x0, t, noise, inp)
    wrong = _variant("img", cfg, w, x0, t, noise, inp, variant="other_labels")
    _rejects(gac, g64, gac, wrong, list(g64))


def test_budget_rejects_ignored_3d_caption_mask():
    """The T2V video + image forward with 3-D caption masks, which the GPU test uses as its fp64 reference: ignoring the
    masks is rejected there too."""
    cfg = T.T2VConfig(num_attention_heads=2, attention_head_dim=64, num_layers=1, sample_size=16, video_length=4,
                      caption_channels=256)
    w = T.make_weights(cfg, 9)
    x, t, text = TI.make_img_inputs(cfg, 2, 2, 20)
    mask = torch.ones(2, 3, 20)
    mask[0, 1, 5:] = 0
    mask[1, 0, 12:] = 0
    x0 = x.permute(0, 2, 1, 3, 4).contiguous()
    noise = torch.randn(x0.shape, generator=torch.Generator().manual_seed(5))
    t = torch.tensor([0, 999])
    inp = dict(text=text, mask=mask, images=2)
    g64, gac = _steps("t2v_img", cfg, w, x0, t, noise, inp)
    wrong = _variant("t2v_img", cfg, w, x0, t, noise, inp, variant="no_mask")
    _rejects(gac, g64, gac, wrong, [k for k in g64 if ".attn2." in k])
