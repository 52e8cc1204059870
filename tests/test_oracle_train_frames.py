"""CPU: one training step at video lengths other than 8 frames -- F = 1 (image-only training), F = 20 (not a power of two)
and F = 32 -- against the loss and gradients of the UNMODIFIED reference (tests/golden/train_tiny64_f*.npz,
oracle/make_golden_train_frames.py).  Two paths: autograd through the oracle restatements, and the product's backward
orchestration (latte_b200/training.py) driven through the torch backend (oracle/train_ops_oracle.TorchOps) in fp32."""
import os

import numpy as np
import pytest
import torch

from latte_b200 import Latte, training
from latte_b200.diffusion import create_diffusion
from oracle import latte_oracle as O
from oracle import sampler_oracle as S
from oracle.train_ops_oracle import TorchOps

FRAMES = [1, 20, 32]


def _load(golden_dir, frames):
    g = np.load(os.path.join(golden_dir, f"train_tiny64_f{frames}.npz"))
    cfg = O.make_config("Latte-tiny64/2", input_size=16, num_frames=frames)
    return g, cfg, O.make_weights(cfg, 21)


def _inputs(g):
    return (torch.from_numpy(g["x0"]), torch.from_numpy(g["noise"]), torch.from_numpy(g["t"]), torch.from_numpy(g["y"]))


def _check_grads(g, grad_of):
    for k, want in zip([str(n) for n in g["grad_names"]], g["grad_norms"]):
        got = grad_of(k).double().norm().item()
        assert abs(got - want) <= 1e-4 * want + 1e-9, (k, got, want)
    for key in g.files:
        if key.startswith("grad::"):
            ref = torch.from_numpy(g[key])
            err = (grad_of(key[6:]) - ref).abs().max().item()
            assert err <= 1e-4 * ref.abs().max().item() + 1e-8, (key, err)


@pytest.mark.parametrize("frames", FRAMES)
def test_oracle_training_step_matches_reference(golden_dir, frames):
    g, cfg, sd0 = _load(golden_dir, frames)
    sd = {k: v.clone().requires_grad_(k not in ("pos_embed", "temp_embed")) for k, v in sd0.items()}
    x0, noise, t, y = _inputs(g)
    terms = S.training_losses(S.make_schedule(""), lambda x, tt, **kw: O.latte_forward(sd, cfg, x, tt, kw["y"]), x0, t, noise,
                              dict(y=y))
    np.testing.assert_allclose(np.stack([terms[k].detach().numpy() for k in ("loss", "mse", "vb")]), g["loss_terms"],
                               rtol=2e-5, atol=1e-6)
    loss = terms["loss"].mean()
    assert abs(loss.item() - float(g["loss"])) < 2e-5 * abs(float(g["loss"]))
    loss.backward()
    assert len(g["grad_names"]) == sum(1 for v in sd.values() if v.requires_grad and v.grad is not None)
    _check_grads(g, lambda k: sd[k].grad)


@pytest.mark.parametrize("frames", FRAMES)
def test_engine_training_step_matches_reference(golden_dir, frames):
    g, cfg, sd = _load(golden_dir, frames)
    m = Latte(input_size=16, hidden_size=128, depth=2, num_heads=2, num_frames=frames, num_classes=101, extras=2)
    m.load_state_dict(sd, strict=True)
    m.eval()
    x0, noise, t, y = _inputs(g)
    ops = TorchOps(torch.float32)
    d = create_diffusion(timestep_respacing="")
    terms = d.training_losses(lambda x, tt, y: training.train_forward(m, ops, torch.float32, x, training.conditioning(m, tt, y)),
                              x0, t, dict(y=y), noise=noise)
    loss = terms["loss"].mean()
    assert abs(loss.item() - float(g["loss"])) < 2e-5 * abs(float(g["loss"]))
    loss.backward()
    named = dict(m.named_parameters())
    assert {str(k) for k in g["grad_names"]} == {k for k, p in named.items() if p.grad is not None}
    _check_grads(g, lambda k: named[k].grad)
