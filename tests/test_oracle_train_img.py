"""CPU: video + image joint training (LatteIMG, reference models/latte_img.py + train_with_img.py:214-241).

The goldens (tests/golden/train_img_tiny64_e{1,2}.npz, oracle/make_golden_train_img.py) hold one training step of the UNMODIFIED
reference module: Latte-tiny64/2, N = 64 tokens, F = 4 video frames + I = 3 images, B = 2, class_dropout_prob = 0.  Checked
here: the oracle's restatement of the LatteIMG forward under autograd, and the product training engine driven through
oracle/train_ops_oracle.TorchOps in fp32 under the product's `diffusion.training_losses` -- which pins the row layout (video rows
first, image rows after), the per-frame conditioning and the temporal blocks' video-only prefix.  Plus the public surface:
the factory, the parameters that receive gradients and the input checks."""
import inspect
import os
import weakref
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from latte_b200 import Latte, LatteIMG, LatteIMG_models, training
from latte_b200.diffusion import create_diffusion
from latte_b200.models import get_models
from oracle import latte_oracle as O
from oracle.latte_img_oracle import latte_img_forward
from oracle.train_ops_oracle import TorchOps

F, I, B = 4, 3, 2
EXTRAS = [2, 1]


def _setup(golden_dir, extras):
    g = np.load(os.path.join(golden_dir, f"train_img_tiny64_e{extras}.npz"))
    cfg = O.make_config("Latte-tiny64/2", input_size=16, num_frames=F, extras=extras, class_dropout_prob=0.0)
    sd = O.make_weights(cfg, 21)
    m = LatteIMG(input_size=16, hidden_size=128, depth=2, num_heads=2, num_frames=F, num_classes=101, extras=extras,
                 class_dropout_prob=0.0)
    m.load_state_dict(sd, strict=True)
    return g, cfg, sd, m


def _inputs(g):
    return (torch.from_numpy(g["x0"]), torch.from_numpy(g["noise"]), torch.from_numpy(g["t"]), torch.from_numpy(g["y"]),
            torch.from_numpy(g["y_image"]))


def _check_grads(g, named, tol):
    names = [str(k) for k in g["grad_names"]]
    assert set(names) == {k for k, p in named.items() if p.grad is not None}
    for k, want in zip(names, g["grad_norms"]):
        got = named[k].grad.double().norm().item()
        assert abs(got - want) <= tol * want + 1e-9, (k, got, want)
    for key in g.files:
        if key.startswith("grad::"):
            ref = torch.from_numpy(g[key])
            err = (named[key[6:]].grad - ref).abs().max().item()
            assert err <= tol * ref.abs().max().item() + 1e-8, (key, err)


@pytest.mark.parametrize("extras", EXTRAS)
def test_oracle_autograd_matches_reference(golden_dir, extras):
    g, cfg, sd, _ = _setup(golden_dir, extras)
    x0, noise, t, y, yi = _inputs(g)
    sdg = {k: v.clone().requires_grad_(k not in ("pos_embed", "temp_embed")) for k, v in sd.items()}
    d = create_diffusion(timestep_respacing="")
    terms = d.training_losses(lambda x, tt, **kw: latte_img_forward(sdg, cfg, x, tt, y if extras == 2 else None,
                                                                       yi if extras == 2 else None, I), x0, t, None, noise=noise)
    got = np.stack([terms[k].detach().numpy() for k in ("loss", "mse", "vb")])
    np.testing.assert_allclose(got, g["loss_terms"], rtol=1e-4, atol=1e-6)
    terms["loss"].mean().backward()
    _check_grads(g, {k: v for k, v in sdg.items() if v.requires_grad}, 1e-4)
    if extras == 1:
        with torch.no_grad():
            out = latte_img_forward(sd, cfg, x0, t, use_image_num=I, training=False)
        np.testing.assert_allclose(out.numpy(), g["eval_out"], rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("extras", EXTRAS)
def test_engine_gradients_equal_reference(golden_dir, extras):
    """The product engine (row layout, per-frame conditioning, temporal prefix, the autograd node) in fp32 through TorchOps."""
    g, cfg, sd, m = _setup(golden_dir, extras)
    m.train()
    x0, noise, t, y, yi = _inputs(g)
    d = create_diffusion(timestep_respacing="")
    ops = TorchOps(torch.float32)

    def model_fn(x, tt, y=None, y_image=None, use_image_num=0):
        c = training.frame_conditioning(m, tt, y, torch.stack(list(y_image)) if y_image is not None else None, use_image_num)
        return training.train_forward(m, ops, torch.float32, x, c, images=use_image_num)

    kw = dict(y=y, y_image=list(yi), use_image_num=I) if extras == 2 else dict(y=None, use_image_num=I)
    terms = d.training_losses(model_fn, x0, t, kw, noise=noise)
    loss = terms["loss"].mean()                      # train_with_img.py:236
    assert abs(loss.item() - float(g["loss"])) < 1e-4 * abs(float(g["loss"]))
    loss.backward()
    _check_grads(g, dict(m.named_parameters()), 1e-4)


def test_engine_forward_only_equals_training_forward(golden_dir):
    """The no-grad forward (no activations kept) computes what the training forward computes."""
    g, cfg, sd, m = _setup(golden_dir, 2)
    x0, _, t, y, yi = _inputs(g)
    ops = TorchOps(torch.float32)
    c = training.frame_conditioning(m, t, y, yi, I)
    a = training.image_forward(m, ops, torch.float32, x0, c, I)
    b = training.train_forward(m, ops, torch.float32, x0, c.detach(), images=I).detach()
    assert torch.equal(a, b)
    want = latte_img_forward(sd, cfg, x0, t, y, yi, I)
    assert (a - want).abs().max().item() <= 1e-4 * want.abs().max().item()


def test_engine_forward_only_frees_each_block_before_the_next(golden_dir):
    """The no-grad forward keeps no activations: when a block (or the output head) starts, the activations of the blocks
    before it are already freed -- the peak stays at one block's, not the whole model's training activations."""
    g, cfg, sd, m = _setup(golden_dir, 2)
    x0, _, t, y, yi = _inputs(g)
    ops = TorchOps(torch.float32)
    made, alive = [], []
    gelu_both, ln_modulate = ops.linear_gelu_both, ops.ln_modulate

    def tracked_gelu_both(*a):
        u, act = gelu_both(*a)
        made.extend((weakref.ref(u), weakref.ref(act)))
        return u, act

    def tracked_ln_modulate(*a):
        alive.append(sum(r() is not None for r in made))
        return ln_modulate(*a)
    ops.linear_gelu_both, ops.ln_modulate = tracked_gelu_both, tracked_ln_modulate
    with torch.no_grad():
        training.image_forward(m, ops, torch.float32, x0, training.frame_conditioning(m, t, y, yi, I), I)
    assert len(made) == 2 * m.depth and len(alive) == 2 * m.depth + 1
    assert alive == [0] * len(alive)


def test_frame_conditioning_matches_reference_per_frame_rows():
    m = LatteIMG(input_size=16, hidden_size=128, depth=2, num_heads=2, num_frames=F, num_classes=11, class_dropout_prob=0.1)
    t, y, yi = torch.tensor([5, 900]), torch.tensor([1, 11]), torch.tensor([[2, 3, 11], [4, 5, 6]])
    with torch.no_grad():
        c = training.frame_conditioning(m, t, y, yi, I)
        cb = training.conditioning(m, t, y)
        tab = m.y_embedder.embedding_table.weight
        temb = cb - tab[y]
    assert c.shape == (B * (F + I), 128)
    for b in range(B):
        for f in range(F):
            assert torch.equal(c[b * F + f], cb[b])                                   # video rows: the per-sample c
        for i in range(I):
            assert torch.allclose(c[B * F + b * I + i], temb[b] + tab[yi[b, i]], atol=1e-6)


def test_factory_builds_latte_img_for_all_twelve_names(golden_dir):
    names = {f"LatteIMG-{s}/{p}" for s in ("XL", "L", "B", "S") for p in (2, 4, 8)}
    assert set(LatteIMG_models) == names
    shapes = {"XL": (28, 1152, 16), "L": (24, 1024, 16), "B": (12, 768, 12), "S": (12, 384, 6)}
    for name in sorted(names):
        size, patch = name.split("-")[1].split("/")
        with torch.device("meta"):                     # shapes only: no storage for the 675M-parameter tables
            net = get_models(SimpleNamespace(model=name, latent_size=32, num_classes=101, num_frames=16, learn_sigma=True,
                                             extras=2))
        assert type(net) is LatteIMG and (net.depth, net.hidden_size, net.num_heads) == shapes[size]
        assert net.patch_size == int(patch) and net.extras == 2 and net.num_frames == 16
    assert inspect.signature(LatteIMG).parameters["extras"].default == 2          # latte_img.py:224
    # conditionings that are not built are refused before any argument is read (extras=78 is the CLIP text projection)
    for args in (SimpleNamespace(model="LatteIMG-XL/2"), SimpleNamespace(model="LatteIMG-S/2", latent_size=32, num_classes=101,
                                                                           num_frames=16, learn_sigma=True, extras=78)):
        with pytest.raises(NotImplementedError):
            get_models(args)
    # the parameter set is Latte's: reference checkpoints load either way
    a = LatteIMG(input_size=16, hidden_size=128, depth=2, num_heads=2, num_frames=F, num_classes=101)
    b = Latte(input_size=16, hidden_size=128, depth=2, num_heads=2, num_frames=F, num_classes=101, extras=2)
    assert {k: v.shape for k, v in a.state_dict().items()} == {k: v.shape for k, v in b.state_dict().items()}
    with pytest.raises(NotImplementedError):
        LatteIMG(input_size=16, hidden_size=128, depth=2, num_heads=2, extras=78)
    g = np.load(os.path.join(golden_dir, "train_img_tiny64_e2.npz"))
    grads = [k for k, p in a.named_parameters() if p.requires_grad]
    assert grads == [str(k) for k in g["grad_names"]]


def _small(extras=2):
    return LatteIMG(input_size=16, hidden_size=128, depth=2, num_heads=2, num_frames=F, num_classes=11, extras=extras)


def test_input_errors_are_value_errors_before_any_launch():
    m = _small().train()
    x = torch.randn(B, F + I, 4, 16, 16)
    t, y = torch.tensor([1, 2]), torch.tensor([3, 4])
    good = [torch.tensor([1, 2, 3]), torch.tensor([4, 5, 6])]
    bad = [
        dict(x=torch.randn(B, F + I + 1, 4, 16, 16), y_image=good),      # frame count != num_frames + use_image_num
        dict(x=x, y_image=None),                                          # extras=2 training needs image labels
        dict(x=x, y_image=[torch.tensor([1, 2])] * 2),                    # wrong label count per sample
        dict(x=x, y_image=good[:1]),                                      # one entry per sample
        dict(x=x, y_image=torch.zeros(B, I + 1, dtype=torch.int64)),
        dict(x=x, y_image=torch.zeros(B, I)),                             # float labels
    ]
    for kw in bad:
        with pytest.raises(ValueError):
            m(kw["x"], t, y=y, y_image=kw["y_image"], use_image_num=I)
    with pytest.raises(ValueError):
        m(x, t, y=None, y_image=good, use_image_num=I)
    with pytest.raises(ValueError, match="eval mode"):
        m.eval()(x, t, y=y, y_image=good, use_image_num=I)
    with torch.no_grad(), pytest.raises(ValueError, match="eval mode"):
        m.eval()(x, t, y=y, y_image=good, use_image_num=I)
    # well-formed input on the CPU: the loud no-CPU-fallback error, after the checks passed
    for kw in (dict(y_image=good), dict(y_image=torch.tensor([[1, 2, 3], [4, 5, 6]]))):
        with pytest.raises(RuntimeError, match="CUDA"):
            m.train()(x, t, y=y, use_image_num=I, **kw)
    with pytest.raises(RuntimeError, match="CUDA"):
        _small(1).eval()(x, t, use_image_num=I)


def test_no_images_is_latte():
    """use_image_num = 0 is the Latte call itself (same code path; the GPU tests check the bits)."""
    m = _small().eval()
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.randn(B, F, 4, 16, 16), torch.tensor([1, 2]), y=torch.tensor([3, 4]))
    assert LatteIMG.forward_with_cfg is Latte.forward_with_cfg
