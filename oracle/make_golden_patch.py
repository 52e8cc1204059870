"""tests/golden/patch*.npz: forwards and training steps of the patch-4 and patch-8 Latte / LatteIMG models from the UNMODIFIED
reference (/root/reference/models/latte.py and latte_img.py, timm shim), in the style of make_golden.py, make_golden_train.py and
make_golden_train_img.py.  Weights and inputs are the oracle's seeded ones (oracle/latte_oracle.make_weights / make_inputs);
every file stores its LatteConfig as JSON under `cfg`, so a test rebuilds the model from the file alone.

  forward:  S/4 and S/8 at input 32 (64 and 16 tokens per frame), tiny72/4 and tiny72/8 at input 16 (16 and 4), tiny64/4
            without learned sigma (head width 64), B/4 at input 64 (256), each with the guided half of forward_with_cfg and the
            reference's own bf16-autocast deviation.
  training: tiny64/4 and tiny64/8 at input 16, tiny72/8 at input 32 (training_losses + loss.backward(), eval-mode label
            path), and LatteIMG tiny64/4 with 3 images per video (extras 1, training mode) plus its eval forward with images.

    python oracle/make_golden_patch.py"""
import dataclasses
import importlib
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(HERE, "ref_shim"))
sys.path.insert(0, "/root/reference")
from oracle import latte_oracle as O                                            # noqa: E402
from oracle.make_golden import build_ref_model, load_reference, weights_digest  # noqa: E402
from oracle.make_golden_train_img import load_reference_img                    # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
FULL = ["final_layer.linear.bias", "blocks.0.attn.qkv.bias", "blocks.1.adaLN_modulation.1.bias", "x_embedder.proj.weight",
        "t_embedder.mlp.2.bias", "blocks.1.mlp.fc2.bias", "blocks.1.attn.qkv.bias"]


def config(base, patch, **kw):
    """The oracle's `base` size (a patch-2 name of O.CONFIGS) at patch size `patch`."""
    return O.make_config(base, patch_size=patch, **kw)


def cfg_json(cfg):
    return np.array(json.dumps(dataclasses.asdict(cfg), sort_keys=True))


def save(name, blob):
    path = os.path.join(OUT, name)
    np.savez_compressed(path, **blob)
    print(f"{path}: {os.path.getsize(path) / 1e3:.0f} kB")


def gen_forward(ref, name, cfg, batch, wseed, iseed):
    sd = O.make_weights(cfg, wseed)
    x, t, y = O.make_inputs(cfg, batch, iseed)
    yy = y if cfg.extras == 2 else None
    m = build_ref_model(ref, cfg, sd)
    with torch.no_grad():
        out = m(x, t, y=yy)
        out_cfg = m.forward_with_cfg(x, t, y=yy, cfg_scale=7.0)
        with torch.autocast("cpu", dtype=torch.bfloat16):
            out_bf16 = m(x, t, y=yy).float()
    save(name, dict(cfg=cfg_json(cfg), out=out.numpy(), out_cfg_half_eps=out_cfg[: batch // 2, :, :4].numpy(),
                    ref_bf16_maxabs=np.float32((out_bf16 - out).abs().max().item()), t=t.numpy(), y=y.numpy(),
                    x_sum=np.float64(x.double().sum().item()), weights_sha256=np.array(weights_digest(sd)),
                    meta=np.array(f"batch={batch} wseed={wseed} iseed={iseed}")))


def _grads(m, blob):
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


def gen_train(ref, ref_diffusion, name, cfg, wseed, tseed, batch=2):
    """As make_golden_train.py: eval-mode label path (no dropout RNG), training_losses, loss.backward()."""
    sd = O.make_weights(cfg, wseed)
    m = build_ref_model(ref, cfg, sd)
    for p in m.parameters():
        p.requires_grad_(True)
    m.pos_embed.requires_grad_(False)
    m.temp_embed.requires_grad_(False)
    torch.manual_seed(tseed)
    x0 = torch.randn(batch, cfg.num_frames, cfg.in_channels, cfg.input_size, cfg.input_size)
    noise = torch.randn_like(x0)
    t = torch.tensor([0, 617, 999][:batch])
    y = torch.tensor([3, 100, 7][:batch])
    d = ref_diffusion.create_diffusion(timestep_respacing="")
    terms = d.training_losses(m, x0, t, dict(y=y), noise=noise)
    loss = terms["loss"].mean()
    loss.backward()
    blob = dict(cfg=cfg_json(cfg), wseed=np.int64(wseed), x0=x0.numpy(), noise=noise.numpy(), t=t.numpy(), y=y.numpy(), loss=np.float32(loss.item()),
                loss_terms=np.stack([terms[k].detach().numpy() for k in ("loss", "mse", "vb")]),
                meta=np.array(f"weights seed {wseed}, torch seed {tseed}, eval-mode labels"))
    _grads(m, blob)
    save(name, blob)


def gen_train_img(ref_img, ref_diffusion, name, cfg, images, wseed, tseed):
    """As make_golden_train_img.py with extras = 1: a training-mode video + image step, then an eval forward with images."""
    assert cfg.extras == 1 and cfg.class_dropout_prob == 0.0
    sd = O.make_weights(cfg, wseed)
    m = ref_img.Latte(input_size=cfg.input_size, patch_size=cfg.patch_size, in_channels=cfg.in_channels,
                      hidden_size=cfg.hidden_size, depth=cfg.depth, num_heads=cfg.num_heads, mlp_ratio=cfg.mlp_ratio,
                      num_frames=cfg.num_frames, class_dropout_prob=cfg.class_dropout_prob, num_classes=cfg.num_classes,
                      learn_sigma=cfg.learn_sigma, extras=cfg.extras)
    missing, unexpected = m.load_state_dict(sd, strict=True)
    assert not missing and not unexpected
    m.train()
    m.pos_embed.requires_grad_(False)
    m.temp_embed.requires_grad_(False)
    torch.manual_seed(tseed)
    x0 = torch.randn(2, cfg.num_frames + images, cfg.in_channels, cfg.input_size, cfg.input_size)
    noise = torch.randn_like(x0)
    t = torch.tensor([0, 617])
    d = ref_diffusion.create_diffusion(timestep_respacing="")
    terms = d.training_losses(m, x0, t, dict(y=None, use_image_num=images), noise=noise)
    loss = terms["loss"].mean()
    loss.backward()
    blob = dict(cfg=cfg_json(cfg), wseed=np.int64(wseed), images=np.int64(images), x0=x0.numpy(), noise=noise.numpy(), t=t.numpy(),
                loss=np.float32(loss.item()), loss_terms=np.stack([terms[k].detach().numpy() for k in ("loss", "mse", "vb")]),
                meta=np.array(f"LatteIMG, weights seed {wseed}, torch seed {tseed}, training mode, class_dropout_prob 0"))
    _grads(m, blob)
    m.eval()
    with torch.no_grad():
        blob["eval_out"] = m(x0, t, use_image_num=images).numpy()
    save(name, blob)


def main():
    torch.manual_seed(0)
    ref = load_reference()
    gen_forward(ref, "patch_s_4_b2.npz", config("Latte-S/2", 4, num_frames=4), 2, 0, 123)
    gen_forward(ref, "patch_s_8_b2.npz", config("Latte-S/2", 8, num_frames=4), 2, 1, 124)
    gen_forward(ref, "patch_tiny72_4_b2.npz", config("Latte-tiny72/2", 4, input_size=16, num_frames=4), 2, 21, 22)
    gen_forward(ref, "patch_tiny72_8_b2.npz", config("Latte-tiny72/2", 8, input_size=16, num_frames=4), 2, 23, 24)
    gen_forward(ref, "patch_tiny64_4_nosigma_b2.npz",
                config("Latte-tiny64/2", 4, input_size=16, num_frames=8, learn_sigma=False, extras=1), 2, 11, 12)
    gen_forward(ref, "patch_b_4_b2.npz", config("Latte-B/2", 4, input_size=64, num_frames=2), 2, 2, 125)

    ref_diffusion = importlib.import_module("diffusion")
    gen_train(ref, ref_diffusion, "patch_train_tiny64_4.npz", config("Latte-tiny64/2", 4, input_size=16, num_frames=4), 21, 5)
    gen_train(ref, ref_diffusion, "patch_train_tiny64_8.npz", config("Latte-tiny64/2", 8, input_size=16, num_frames=4), 22, 6)
    gen_train(ref, ref_diffusion, "patch_train_tiny72_8.npz", config("Latte-tiny72/2", 8, input_size=32, num_frames=4), 23, 7)
    gen_train_img(load_reference_img(), ref_diffusion, "patch_train_img_tiny64_4.npz",
                  config("Latte-tiny64/2", 4, input_size=16, num_frames=4, extras=1, class_dropout_prob=0.0), 3, 24, 8)


if __name__ == "__main__":
    main()
