"""tests/golden/train_tiny64_f{1,20,32}.npz: one training step's loss and GRADIENTS from the UNMODIFIED reference at video
lengths other than the 8 frames of train_tiny64.npz -- the Latte module (/root/reference/models/latte.py, timm shim) under the
reference's own `diffusion.training_losses` (train.py:206-222 with given latents, eval-mode label path so there is no dropout
RNG).  F = 1 is image-only training (a one-frame temporal block), F = 20 is not a power of two and leaves a partial 64-row
block in the temporal attention backward, F = 32 is the smallest common training length above 16 frames.
    python oracle/make_golden_train_frames.py"""
import importlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(HERE, "ref_shim"))
sys.path.insert(0, "/root/reference")
from oracle import latte_oracle as O                          # noqa: E402
from oracle.make_golden import build_ref_model, load_reference  # noqa: E402

FRAMES = (1, 20, 32)
# blocks.1 is the temporal block of the depth-2 model: its qkv bias gradient is a column sum of the temporal attention backward
FULL = ["final_layer.linear.bias", "blocks.0.attn.qkv.bias", "blocks.1.attn.qkv.bias", "blocks.1.attn.proj.bias",
        "blocks.1.adaLN_modulation.1.bias", "x_embedder.proj.weight", "t_embedder.mlp.2.bias"]


def make(ref, ref_diffusion, frames):
    cfg = O.make_config("Latte-tiny64/2", input_size=16, num_frames=frames)
    sd = O.make_weights(cfg, 21)
    m = build_ref_model(ref, cfg, sd)          # .eval(): LabelEmbedder applies no dropout (latte.py:148-153)
    for p in m.parameters():
        p.requires_grad_(True)
    m.pos_embed.requires_grad_(False)
    m.temp_embed.requires_grad_(False)
    torch.manual_seed(5 + frames)
    x0 = torch.randn(2, frames, 4, 16, 16)
    noise = torch.randn_like(x0)
    t = torch.tensor([0, 617])
    y = torch.tensor([3, 100])
    d = ref_diffusion.create_diffusion(timestep_respacing="")
    terms = d.training_losses(m, x0, t, dict(y=y), noise=noise)
    loss = terms["loss"].mean()                # train.py:222
    loss.backward()
    blob = dict(x0=x0.numpy(), noise=noise.numpy(), t=t.numpy(), y=y.numpy(), loss=np.float32(loss.item()),
                loss_terms=np.stack([terms[k].detach().numpy() for k in ("loss", "mse", "vb")]),
                meta=np.array(f"Latte-tiny64/2 input 16 frames {frames}, weights seed 21, torch seed {5 + frames}"))
    names, norms = [], []
    for k, p in m.named_parameters():
        if p.grad is None:
            continue
        names.append(k)
        norms.append(p.grad.double().norm().item())
        if k in FULL:
            blob["grad::" + k] = p.grad.numpy()
    blob["grad_names"] = np.array(names)
    blob["grad_norms"] = np.array(norms, dtype=np.float64)
    path = os.path.join(ROOT, "tests", "golden", f"train_tiny64_f{frames}.npz")
    np.savez_compressed(path, **blob)
    print("wrote", path, f"({os.path.getsize(path) / 1e3:.0f} kB)", "loss", loss.item(), "params with grad", len(names))


def main():
    ref_diffusion = importlib.import_module("diffusion")
    ref = load_reference()
    for f in FRAMES:
        make(ref, ref_diffusion, f)


if __name__ == "__main__":
    main()
