"""tests/golden/train_img_tiny64_e{1,2}.npz: one video + image joint training step's loss and GRADIENTS from the UNMODIFIED
reference -- the LatteIMG module (/root/reference/models/latte_img.py, timm shim) in training mode under the reference's own
`diffusion.training_losses` (train_with_img.py:214-241 with given latents).  class_dropout_prob = 0, so the label path draws no
random numbers.  Latte-tiny64/2, input 16 (N = 64), F = 4 video frames + I = 3 images, B = 2; extras = 2 with a distinct label
per image, extras = 1 (timestep only) with one eval-mode forward over the same video + image frames.
    python oracle/make_golden_train_img.py"""
import importlib
import importlib.util
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

REF_IMG = "/root/reference/models/latte_img.py"
FRAMES, IMAGES, BATCH = 4, 3, 2
# blocks.1 is the temporal block of the depth-2 model (video rows only); the embedders get their gradients through the
# per-frame conditioning, image labels included
FULL = ["final_layer.linear.bias", "blocks.0.attn.qkv.bias", "blocks.1.attn.qkv.bias", "blocks.1.adaLN_modulation.1.bias",
        "blocks.0.adaLN_modulation.1.bias", "x_embedder.proj.weight", "t_embedder.mlp.2.bias", "y_embedder.embedding_table.weight"]


def load_reference_img():
    spec = importlib.util.spec_from_file_location("ref_latte_img", REF_IMG)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def make(ref, ref_diffusion, extras):
    cfg = O.make_config("Latte-tiny64/2", input_size=16, num_frames=FRAMES, extras=extras, class_dropout_prob=0.0)
    sd = O.make_weights(cfg, 21)
    m = ref.Latte(input_size=cfg.input_size, patch_size=cfg.patch_size, in_channels=cfg.in_channels, hidden_size=cfg.hidden_size,
                  depth=cfg.depth, num_heads=cfg.num_heads, mlp_ratio=cfg.mlp_ratio, num_frames=cfg.num_frames,
                  class_dropout_prob=cfg.class_dropout_prob, num_classes=cfg.num_classes, learn_sigma=cfg.learn_sigma, extras=extras)
    missing, unexpected = m.load_state_dict(sd, strict=True)
    assert not missing and not unexpected
    m.train()
    m.pos_embed.requires_grad_(False)
    m.temp_embed.requires_grad_(False)
    torch.manual_seed(40 + extras)
    x0 = torch.randn(BATCH, FRAMES + IMAGES, 4, 16, 16)
    noise = torch.randn_like(x0)
    t = torch.tensor([0, 617])
    y = torch.tensor([3, 100])
    y_image = torch.tensor([[5, 17, 42], [99, 0, 63]])       # distinct per image (train_with_img.py passes a list of B tensors)
    kw = dict(y=y, y_image=list(y_image), use_image_num=IMAGES) if extras == 2 else dict(y=None, use_image_num=IMAGES)
    d = ref_diffusion.create_diffusion(timestep_respacing="")
    terms = d.training_losses(m, x0, t, kw, noise=noise)
    loss = terms["loss"].mean()                # train_with_img.py:236
    loss.backward()
    blob = dict(x0=x0.numpy(), noise=noise.numpy(), t=t.numpy(), y=y.numpy(), y_image=y_image.numpy(), loss=np.float32(loss.item()),
                loss_terms=np.stack([terms[k].detach().numpy() for k in ("loss", "mse", "vb")]),
                meta=np.array(f"LatteIMG Latte-tiny64/2 input 16 frames {FRAMES} images {IMAGES} extras {extras}, weights seed 21, "
                              f"torch seed {40 + extras}, training mode, class_dropout_prob 0"))
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
    if extras == 1:                            # eval mode with images works for extras = 1 (latte_img.py:316-399)
        m.eval()
        with torch.no_grad():
            blob["eval_out"] = m(x0, t, use_image_num=IMAGES).numpy()
    path = os.path.join(ROOT, "tests", "golden", f"train_img_tiny64_e{extras}.npz")
    np.savez_compressed(path, **blob)
    print("wrote", path, f"({os.path.getsize(path) / 1e3:.0f} kB)", "loss", loss.item(), "params with grad", len(names))


def main():
    ref_diffusion = importlib.import_module("diffusion")
    ref = load_reference_img()
    for e in (2, 1):
        make(ref, ref_diffusion, e)


if __name__ == "__main__":
    main()
