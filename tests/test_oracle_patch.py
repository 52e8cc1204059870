"""CPU: the patch-4 and patch-8 Latte / LatteIMG models.

  * The oracle restatement (oracle/latte_oracle.py) against the forward goldens of the UNMODIFIED reference
    (oracle/make_golden_patch.py), as tests/test_oracle.py does at patch 2.
  * The training engine (latte_b200/training.py) on oracle/train_ops_oracle.TorchOps against the reference's gradients, in fp32
    and with bf16 operand rounding, as tests/test_train_engine.py does: this pins the zero-padded patch and head operands
    (K = C*p*p = 64 / 256, p*p*C_out = 64 .. 512 rows rounded up to the GEMM's 64-element k-block).
  * All 24 names of `get_models` (Latte and LatteIMG, S / B / L / XL at patch 2, 4 and 8) build with the reference's
    state-dict keys and shapes.
  * The library's shape rules and workspace sizes (no GPU needed: they run before anything is launched)."""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import patch_golden as PG
from latte_b200 import Latte, LatteIMG, training
from latte_b200.diffusion import create_diffusion
from oracle import latte_oracle as O
from oracle.train_ops_oracle import TorchOps


@pytest.mark.parametrize("fname", PG.FORWARD)
def test_forward_matches_reference_golden(golden_dir, fname):
    g, cfg = PG.load(golden_dir, fname)
    batch, wseed, iseed = PG.seeds(g)
    sd = O.make_weights(cfg, wseed)
    x, t, y = O.make_inputs(cfg, batch, iseed)
    assert abs(float(x.double().sum()) - float(g["x_sum"])) < 1e-9
    out = O.latte_forward(sd, cfg, x, t, y if cfg.extras == 2 else None)
    ref = torch.from_numpy(g["out"])
    assert out.shape == ref.shape == (batch, cfg.num_frames, cfg.out_channels, cfg.input_size, cfg.input_size)
    assert (out - ref).abs().max().item() < 2e-4
    out_cfg = O.latte_forward_with_cfg(sd, cfg, x, t, y if cfg.extras == 2 else None, cfg_scale=7.0)
    assert (out_cfg[: batch // 2, :, :4] - torch.from_numpy(g["out_cfg_half_eps"])).abs().max().item() < 1e-3


def _engine_step(g, cfg, dt, images=0):
    """One training step of the product engine through TorchOps(dt) under the product's training_losses; returns the model
    (with .grad set) and the loss."""
    cls = LatteIMG if images else Latte
    m = PG.build(cls, cfg)
    m.load_state_dict(O.make_weights(cfg, int(g["wseed"])), strict=True)
    m.eval()                     # the engine itself has no mode; eval keeps the label path free of dropout RNG
    ops = TorchOps(dt)
    x0, noise, t = (torch.from_numpy(g[k]) for k in ("x0", "noise", "t"))
    d = create_diffusion(timestep_respacing="")
    if images:
        def model_fn(x, tt, y=None, use_image_num=0):
            c = training.frame_conditioning(m, tt, None, None, use_image_num)
            return training.train_forward(m, ops, dt, x, c, images=use_image_num)
        kw = dict(y=None, use_image_num=images)
    else:
        def model_fn(x, tt, y):
            return training.train_forward(m, ops, dt, x, training.conditioning(m, tt, y))
        kw = dict(y=torch.from_numpy(g["y"]))
    terms = d.training_losses(model_fn, x0, t, kw, noise=noise)
    loss = terms["loss"].mean()
    loss.backward()
    return m, loss.item()


@pytest.mark.parametrize("fname", PG.TRAIN + [PG.TRAIN_IMG])
def test_engine_gradients_equal_reference(golden_dir, fname):
    g, cfg = PG.load(golden_dir, fname)
    images = int(g["images"]) if "images" in g.files else 0
    m, loss = _engine_step(g, cfg, torch.float32, images)
    assert abs(loss - float(g["loss"])) < 2e-5 * abs(float(g["loss"]))
    PG.check_grads(g, dict(m.named_parameters()), 1e-4, 1e-4)


@pytest.mark.parametrize("fname", PG.TRAIN + [PG.TRAIN_IMG])
def test_engine_with_16bit_operands_on_cpu(golden_dir, fname):
    """bf16 rounding wherever the CUDA backend rounds: within bf16 noise of the reference's fp32 gradients, every gradient fp32."""
    g, cfg = PG.load(golden_dir, fname)
    images = int(g["images"]) if "images" in g.files else 0
    m, loss = _engine_step(g, cfg, torch.bfloat16, images)
    assert abs(loss - float(g["loss"])) < 2e-2 * abs(float(g["loss"]))
    assert all(p.grad.dtype == torch.float32 for p in m.parameters() if p.grad is not None)
    PG.check_grads(g, dict(m.named_parameters()), 8e-2, 8e-2)


def test_img_eval_forward_with_images_matches_reference(golden_dir):
    """LatteIMG eval with images (extras 1) through the engine's forward without saved activations, in fp32."""
    g, cfg = PG.load(golden_dir, PG.TRAIN_IMG)
    m = PG.build(LatteIMG, cfg)
    m.load_state_dict(O.make_weights(cfg, int(g["wseed"])), strict=True)
    x0, t = torch.from_numpy(g["x0"]), torch.from_numpy(g["t"])
    c = training.frame_conditioning(m, t, None, None, int(g["images"]))
    out = training.image_forward(m, TorchOps(torch.float32), torch.float32, x0, c, int(g["images"]))
    np.testing.assert_allclose(out.numpy(), g["eval_out"], rtol=1e-4, atol=1e-5)


NAMES = [f"{fam}-{size}/{p}" for fam in ("Latte", "LatteIMG") for size in ("S", "B", "L", "XL") for p in (2, 4, 8)]


@pytest.mark.parametrize("name", NAMES)
def test_get_models_builds_reference_state_dict(name):
    """get_models(args) as sample.py / train.py call it; built on the meta device (no memory for XL's weights)."""
    from latte_b200.models import get_models
    size, p = name.split("-")[1].split("/")
    args = SimpleNamespace(model=name, latent_size=32, num_classes=101, num_frames=16, learn_sigma=True, extras=2)
    with torch.device("meta"):
        m = get_models(args)
    assert type(m) is (LatteIMG if name.startswith("LatteIMG") else Latte) and m.patch_size == int(p)
    cfg = O.make_config(f"Latte-{size}/2", patch_size=int(p), input_size=32, num_frames=16, num_classes=101)
    got = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert got == {k: tuple(s) for k, s in O.state_dict_spec(cfg)}


def _shape(**kw):
    from latte_b200 import _lib
    base = dict(depth=28, hidden=1152, heads=16, mlp_hidden=4608, patch=2, in_channels=4, out_channels=8, input_size=32,
                frames=16, num_embed=102, dtype=_lib.FP16, wide_patch=1)
    base.update(kw)
    return _lib.LatteShape(**base)


def test_workspace_sizes_with_wide_patch():
    """With `wide_patch` set, the Latte workspace is the activations plus the head's fp32 [T, p*p*C_out] buffer (32 columns
    at the least, so the patch-2 sizes are those of a 32-wide head, as without the flag); grids the spatial attention does not
    take are refused by the size query.  Without the flag the rules of ABI v6 hold: patch 2 only (tests/test_abi.py)."""
    from latte_b200 import _lib
    lib = _lib.load()
    D = 1152
    for p, n_out in ((2, 32), (4, 128), (8, 512)):
        s = _shape(patch=p)
        n = lib.b200_latte_workspace_bytes(C.byref(s), 2)
        T = 2 * 16 * (32 // p) ** 2
        lower = T * D * 4 + T * D * 2 + T * 3 * D * 2 + T * 4 * D * 2 + (T + 1) * n_out * 4  # x, h, qkv, mlp hidden, head
        assert lower <= n < lower + (1 << 21), (p, n, lower)   # + conditioning rows, stream-K flags, alignment
    # no learned sigma at patch 2: a 16-wide head still reserves the 32-wide buffer; patch 2 sizes do not depend on the flag
    assert lib.b200_latte_workspace_bytes(C.byref(_shape(out_channels=4)), 2) == lib.b200_latte_workspace_bytes(C.byref(_shape()), 2)
    assert lib.b200_latte_workspace_bytes(C.byref(_shape(wide_patch=0)), 2) == lib.b200_latte_workspace_bytes(C.byref(_shape()), 2)
    for p in (4, 8):
        assert lib.b200_latte_workspace_bytes(C.byref(_shape(patch=p, wide_patch=0)), 2) == 0
        assert "need wide_patch" in _lib.last_error()
    assert lib.b200_latte_workspace_bytes(C.byref(_shape(patch=16)), 2) == 0 and "(2, 4, 8)" in _lib.last_error()
    assert lib.b200_latte_workspace_bytes(C.byref(_shape(heads=10)), 2) == 0 and "heads" in _lib.last_error()
    # input 24 at patch 4: 6 x 6 = 36 tokens per frame
    assert lib.b200_latte_workspace_bytes(C.byref(_shape(patch=4, input_size=24)), 2) == 0
    assert "6 x 6 patches per frame" in _lib.last_error()
    assert lib.b200_latte_workspace_bytes(C.byref(_shape(patch=4, input_size=30)), 2) == 0 and "patch" in _lib.last_error()


def test_t2v_stays_at_patch_2():
    from latte_b200 import _lib
    lib = _lib.load()
    s = _lib.T2VShape(layers=2, hidden=1152, heads=16, mlp_hidden=4608, patch=2, in_channels=4, out_channels=8, input_size=64,
                      frames=4, caption_channels=4096, dtype=_lib.FP16)
    assert lib.b200_t2v_workspace_bytes(C.byref(s), 1, 120) > 0
    s.patch = 4
    assert lib.b200_t2v_workspace_bytes(C.byref(s), 1, 120) == 0 and "patch size 4 not built (only 2)" in _lib.last_error()
