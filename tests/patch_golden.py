"""The patch-4 / patch-8 goldens (oracle/make_golden_patch.py): each file carries its LatteConfig as JSON under `cfg`."""
import json
import os

import numpy as np

FORWARD = ["patch_s_4_b2.npz", "patch_s_8_b2.npz", "patch_tiny72_4_b2.npz", "patch_tiny72_8_b2.npz",
           "patch_tiny64_4_nosigma_b2.npz", "patch_b_4_b2.npz"]
TRAIN = ["patch_train_tiny64_4.npz", "patch_train_tiny64_8.npz", "patch_train_tiny72_8.npz"]
TRAIN_IMG = "patch_train_img_tiny64_4.npz"


def load(golden_dir, fname):
    """(the npz, its oracle LatteConfig)."""
    from oracle import latte_oracle as O
    g = np.load(os.path.join(golden_dir, fname))
    return g, O.LatteConfig(**json.loads(str(g["cfg"])))


def seeds(g):
    """(batch, weight seed, input seed) of a forward golden."""
    kv = dict(item.split("=") for item in str(g["meta"]).split())
    return int(kv["batch"]), int(kv["wseed"]), int(kv["iseed"])


def build(cls, cfg):
    """`cls` (Latte or LatteIMG) with the golden's configuration."""
    return cls(input_size=cfg.input_size, patch_size=cfg.patch_size, in_channels=cfg.in_channels, hidden_size=cfg.hidden_size,
               depth=cfg.depth, num_heads=cfg.num_heads, mlp_ratio=cfg.mlp_ratio, num_frames=cfg.num_frames,
               class_dropout_prob=cfg.class_dropout_prob, num_classes=cfg.num_classes, learn_sigma=cfg.learn_sigma,
               extras=cfg.extras)


def check_grads(g, named, norm_tol, full_tol, frobenius=False):
    """Every parameter the reference gave a gradient has one, each norm within norm_tol (relative) of the reference's, and
    every stored full gradient within full_tol: of the reference's largest magnitude element by element, or with
    `frobenius` as a relative Frobenius error (the GPU tests' measure)."""
    import torch
    names = [str(k) for k in g["grad_names"]]
    assert set(names) == {k for k, p in named.items() if p.grad is not None}
    for k, want in zip(names, g["grad_norms"]):
        got = named[k].grad.double().norm().item()
        assert abs(got - want) <= norm_tol * want + 1e-9, (k, got, want)
    for key in g.files:
        if key.startswith("grad::"):
            grad = named[key[6:]].grad.float()
            ref = torch.from_numpy(g[key]).to(grad.device)
            if frobenius:
                err = ((grad - ref).norm() / (ref.norm() + 1e-12)).item()
                assert err < full_tol, (key, err)
            else:
                err = (grad - ref).abs().max().item()
                assert err <= full_tol * ref.abs().max().item() + 1e-8, (key, err)
