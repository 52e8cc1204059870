"""GPU: video + image joint training (LatteIMG) on the native path, and the adaLN gradients above 8 conditioning rows.

The step is checked against the UNMODIFIED reference's gradients (tests/golden/train_img_tiny64_e{1,2}.npz) with
tests/test_gpu_train.py's tolerances (each gradient norm within 1 % in fp16, 8 % in bf16).  Tolerance of the adaLN gradients
above 8 rows: dmod is rounded to the operand type (what the reference computes under bf16 autocast); against fp64 on those
rounded values the only error left is fp32 accumulation, held to 1e-4 of the largest magnitude."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DTS = [torch.float16, torch.bfloat16]
EPS = {torch.float16: 1e-3, torch.bfloat16: 8e-3}
F, I, B = 4, 3, 2


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


def _rel(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


def _golden_model(golden_dir, dev, extras, cls=None):
    from latte_b200 import LatteIMG
    from oracle import latte_oracle as O
    g = np.load(os.path.join(golden_dir, f"train_img_tiny64_e{extras}.npz"))
    cfg = O.make_config("Latte-tiny64/2", input_size=16, num_frames=F, extras=extras, class_dropout_prob=0.0)
    m = (cls or LatteIMG)(input_size=16, hidden_size=128, depth=2, num_heads=2, num_frames=F, num_classes=101, extras=extras,
                          class_dropout_prob=0.0)
    m.load_state_dict(O.make_weights(cfg, 21), strict=True)
    return g, cfg, m.to(dev)


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("extras", [2, 1])
def test_training_step_matches_reference_gradients(dev, golden_dir, dt, extras):
    """model.train() + diffusion.training_losses(model, x, t, dict(y, y_image, use_image_num)) + loss.backward()
    (train_with_img.py:214-241), y_image as the script builds it: a list of B CPU label tensors."""
    from latte_b200.diffusion import create_diffusion
    g, cfg, m = _golden_model(golden_dir, dev, extras)
    m.train()
    m.train_dtype = dt
    d = create_diffusion(timestep_respacing="")
    x0, noise = torch.from_numpy(g["x0"]).to(dev), torch.from_numpy(g["noise"]).to(dev)
    t = torch.from_numpy(g["t"]).to(dev)
    kw = dict(use_image_num=I)
    if extras == 2:
        kw.update(y=torch.from_numpy(g["y"]).to(dev), y_image=list(torch.from_numpy(g["y_image"])))
    terms = d.training_losses(m, x0, t, kw, noise=noise)
    loss = terms["loss"].mean()
    assert abs(loss.item() - float(g["loss"])) < 3 * EPS[dt] * abs(float(g["loss"]))
    loss.backward()
    named = dict(m.named_parameters())
    names = [str(n) for n in g["grad_names"]]
    assert set(names) == {k for k, p in named.items() if p.grad is not None}
    for k, want in zip(names, g["grad_norms"]):
        got = named[k].grad.double().norm().item()
        assert abs(got - want) <= 10 * EPS[dt] * want, (k, got, want)
    for key in g.files:
        if key.startswith("grad::"):
            e = _rel(named[key[6:]].grad, torch.from_numpy(g[key]).to(dev))
            assert e < 10 * EPS[dt], (key, e)


def test_eval_forward_with_images_extras1(dev, golden_dir):
    """Eval mode with images (extras = 1): the engine's forward without saved activations, against the reference's output."""
    g, cfg, m = _golden_model(golden_dir, dev, 1)
    m.eval()
    m.train_dtype = torch.float16
    x0, t = torch.from_numpy(g["x0"]).to(dev), torch.from_numpy(g["t"]).to(dev)
    with torch.no_grad():
        out = m(x0, t, use_image_num=I)
    ref = torch.from_numpy(g["eval_out"]).to(dev)
    assert out.shape == ref.shape
    assert (out - ref).abs().max().item() < 2e-2 * ref.abs().max().item()


@pytest.mark.parametrize("dt", DTS)
def test_no_images_is_latte(dev, golden_dir, dt):
    """use_image_num = 0: training forward, eval forward (eager and CUDA-graph replay) and forward_with_cfg bit-identical to
    Latte on the same weights; gradients equal up to the order of the backward's atomic reductions."""
    from latte_b200 import Latte
    g, cfg, mi = _golden_model(golden_dir, dev, 2)
    _, _, ml = _golden_model(golden_dir, dev, 2, cls=Latte)
    x0 = torch.from_numpy(g["x0"]).to(dev)[:, :F].contiguous()
    t, y = torch.from_numpy(g["t"]).to(dev), torch.from_numpy(g["y"]).to(dev)
    dout = torch.randn(x0.shape[0], F, 8, 16, 16, generator=torch.Generator().manual_seed(3)).to(dev)
    res = []
    for m in (mi, ml):
        m.train()
        m.train_dtype = dt
        m.zero_grad(set_to_none=True)
        out = m(x0, t, y=y)
        out.backward(dout)
        grads = {k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None}
        m.eval()
        with torch.no_grad():
            ev = [m(x0, t, y=y) for _ in range(3)]                         # eager, then CUDA-graph capture and replay
            cfgo = m.forward_with_cfg(x0, t, y=y, cfg_scale=4.0)
        res.append((out.detach(), grads, ev, cfgo))
    (oa, ga, ea, ca), (ob, gb, eb, cb) = res
    assert torch.equal(oa, ob) and torch.equal(ca, cb)
    assert all(torch.equal(a, b) for a, b in zip(ea, eb))
    # the backward's column and per-sample reductions add with float atomics, so two runs of Latte itself agree to summation
    # order only: the same bound for LatteIMG against Latte
    assert set(ga) == set(gb)
    for k in ga:
        assert _rel(ga[k], gb[k]) < 1e-3, (k, _rel(ga[k], gb[k]))


@pytest.mark.parametrize("dt", DTS)
def test_video_outputs_ignore_image_frames(dev, golden_dir, dt):
    """Image frames pass the temporal blocks by: the video frames' outputs are bit-identical whatever the image frames hold
    (other contents, other labels, NaN)."""
    g, cfg, m = _golden_model(golden_dir, dev, 2)
    m.train()
    m.train_dtype = dt
    x0 = torch.from_numpy(g["x0"]).to(dev)
    t, y, yi = (torch.from_numpy(g[k]).to(dev) for k in ("t", "y", "y_image"))
    x1 = x0.clone()
    x1[:, F:] = torch.randn(B, I, 4, 16, 16, generator=torch.Generator().manual_seed(8)).to(dev)
    xn = x0.clone()
    xn[:, F:] = float("nan")
    yi2 = (yi + 7) % 101
    for grad in (False, True):
        with torch.set_grad_enabled(grad):
            base = m(x0, t, y=y, y_image=yi, use_image_num=I).detach()
            assert torch.isfinite(base).all()
            for x, labels in ((x1, yi), (x0, yi2), (xn, yi)):
                out = m(x, t, y=y, y_image=labels, use_image_num=I).detach()
                assert torch.equal(out[:, :F], base[:, :F])
            assert not torch.equal(m(x1, t, y=y, y_image=yi, use_image_num=I)[:, F:], base[:, F:])


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("R", [9, 14, 36, 96, 256])
def test_adaln_gradients_above_eight_rows(dev, dt, R):
    from latte_b200.train_ops import NativeOps
    nat = NativeOps(dt)
    g = torch.Generator().manual_seed(R)
    D = 1152
    NA = 4 * 6 * D + 2 * D
    dmod = torch.randn(R, NA, generator=g).to(dev)
    sc = torch.randn(R, D, generator=g).to(dev).to(dt)
    w = (torch.randn(NA, D, generator=g) / 20).to(dev).to(dt)
    d64 = dmod.to(dt).double()
    want_dw = d64.t() @ sc.double()
    want_dsc = d64 @ w.double()
    got_dw, got_dsc = nat.ada_outer(dmod, sc), nat.ada_dsc(dmod, w)
    assert got_dw.shape == (NA, D) and got_dsc.shape == (R, D)
    for got, want, name in ((got_dw, want_dw, "dW"), (got_dsc, want_dsc, "dsc")):
        err = (got.double() - want).abs().max().item()
        assert err <= 1e-4 * want.abs().max().item(), (name, err)
    # and against the unrounded fp64 product: within the operand rounding
    assert _rel(got_dw, dmod.double().t() @ sc.double()) < EPS[dt]


def test_latte_training_step_at_batch_12(dev):
    """A local batch above 8 (plain Latte): the adaLN gradients take the GEMM path; native bf16 vs the engine through TorchOps."""
    from latte_b200 import Latte, training
    from latte_b200.train_ops import NativeOps
    from oracle import latte_oracle as O
    from oracle.train_ops_oracle import TorchOps
    cfg = O.make_config("Latte-tiny64/2", input_size=16, num_frames=8)
    m = Latte(input_size=16, hidden_size=128, depth=2, num_heads=2, num_frames=8, num_classes=101, extras=2)
    m.load_state_dict(O.make_weights(cfg, 21), strict=True)
    m = m.to(dev)
    gen = torch.Generator().manual_seed(12)
    x = torch.randn(12, 8, 4, 16, 16, generator=gen).to(dev)
    t = torch.randint(0, 1000, (12,), generator=gen).to(dev)
    y = torch.randint(0, 101, (12,), generator=gen).to(dev)
    dout = torch.randn(12, 8, 8, 16, 16, generator=gen).to(dev)
    grads = []
    for ops, od in ((NativeOps(torch.bfloat16), torch.bfloat16), (TorchOps(torch.float32), torch.float32)):
        m.zero_grad(set_to_none=True)
        out = training.train_forward(m, ops, od, x, training.conditioning(m, t, y))
        out.backward(dout)
        grads.append(({k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None}, out.detach()))
    (gn, on), (gr, orf) = grads
    assert _rel(on, orf) < 3 * EPS[torch.bfloat16]
    assert set(gn) == set(gr)
    for k in gr:
        assert _rel(gn[k], gr[k]) < 8 * EPS[torch.bfloat16], k


def test_label_dropout_one_maps_every_label_to_null(dev):
    """class_dropout_prob = 1.0 in training mode: video and image labels all become the null class (token_drop)."""
    from latte_b200 import LatteIMG
    from oracle import latte_oracle as O
    from oracle.latte_img_oracle import latte_img_forward
    cfg = O.make_config("Latte-tiny64/2", input_size=16, num_frames=F, class_dropout_prob=1.0)
    sd = O.make_weights(cfg, 4)
    m = LatteIMG(input_size=16, hidden_size=128, depth=2, num_heads=2, num_frames=F, num_classes=101, class_dropout_prob=1.0)
    m.load_state_dict(sd, strict=True)
    m = m.to(dev).train()
    m.train_dtype = torch.float16
    gen = torch.Generator().manual_seed(5)
    x = torch.randn(B, F + I, 4, 16, 16, generator=gen)
    t, y, yi = torch.tensor([10, 800]), torch.tensor([3, 4]), torch.tensor([[1, 2, 3], [4, 5, 6]])
    out = m(x.to(dev), t.to(dev), y=y.to(dev), y_image=yi.to(dev), use_image_num=I)
    null = torch.full_like(y, 101)
    ref = latte_img_forward(sd, cfg, x, t, null, torch.full_like(yi, 101), I)
    assert (out.detach().cpu() - ref).abs().max().item() < 2e-2 * ref.abs().max().item()


def test_autocast_step_at_xl_head_geometry(dev):
    """bf16 autocast at the XL/2 attention geometry (head_dim 72, 256 tokens) with the ucf101_img shape B = 4, F = 16, I = 8:
    96 conditioning rows, finite loss and gradients."""
    from latte_b200 import LatteIMG
    from latte_b200.diffusion import create_diffusion
    from oracle import latte_oracle as O
    cfg = O.make_config("Latte-tiny72/2", input_size=32, num_frames=16)
    m = LatteIMG(input_size=32, hidden_size=576, depth=4, num_heads=8, num_frames=16, num_classes=101)
    m.load_state_dict(O.make_weights(cfg, 6), strict=True)
    m = m.to(dev).train()
    gen = torch.Generator().manual_seed(6)
    x = torch.randn(4, 24, 4, 32, 32, generator=gen).to(dev)
    t = torch.tensor([0, 250, 500, 999], device=dev)
    y = torch.tensor([1, 2, 3, 4], device=dev)
    yi = [torch.randint(0, 101, (8,), generator=gen) for _ in range(4)]
    d = create_diffusion(timestep_respacing="")
    with torch.autocast("cuda", dtype=torch.bfloat16):
        loss = d.training_losses(m, x, t, dict(y=y, y_image=yi, use_image_num=8))["loss"].mean()
    loss.backward()
    assert torch.isfinite(loss)
    for k, p in m.named_parameters():
        if p.requires_grad:
            assert p.grad is not None and torch.isfinite(p.grad).all(), k
