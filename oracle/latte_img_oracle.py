"""CPU oracle for the LatteIMG forward (reference models/latte_img.py) — TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A functional restatement, over the op-by-op pieces of oracle/latte_oracle.py, of the video + image joint forward that
train_with_img.py trains.  Checked against the unmodified reference by tests/test_oracle_train_img.py through the goldens
of oracle/make_golden_train_img.py.
"""
from __future__ import annotations

import torch

from oracle.latte_oracle import (LatteConfig, final_layer, patch_embed, t_embedder, transformer_block, unpatchify,
                                 y_embedder)


def latte_img_forward(sd, cfg: LatteConfig, x, t, y=None, y_image=None, use_image_num=0, training=True, dtype=torch.float32):
    """models/latte_img.py:316-399 without label dropout: x (B, F + I, C, H, W) with F = cfg.num_frames video frames, then
    I = use_image_num images.  Spatial blocks and the final layer see all F + I frames, conditioned per frame on t_b + y_b
    (video) or t_b + y_image[b, i] (image i; extras == 2 in training mode); temporal blocks and temp_embed see the video frames
    only.  y_image (B, I) int64.  extras == 2 in eval mode has no image conditioning in the reference (a shape error there)."""
    B, Fa = x.shape[0], x.shape[1]
    I = use_image_num
    Fr = Fa - I
    N, D = cfg.num_patches, cfg.hidden_size
    assert Fr == cfg.num_frames
    h = patch_embed(sd, cfg, x, dtype)                       # (B*(F+I), N, D)   :328-329
    tv = t_embedder(sd, t, dtype)                            # (B, D)            :330
    c_temp = tv
    c_spatial = tv[:, None].expand(B, Fa, D)                 # :331 timestep_spatial
    if cfg.extras == 2:
        assert training or I == 0, "latte_img.py has no image labels in eval mode"
        yv = y_embedder(sd, y, dtype)                        # :335
        c_temp = tv + yv                                     # :350, :381
        ys = yv[:, None].expand(B, Fr, D)
        if I:
            ys = torch.cat([ys, y_embedder(sd, y_image, dtype)], dim=1)      # :337-345
        c_spatial = c_spatial + ys
    c_spatial = c_spatial.reshape(B * Fa, D)
    c_temp = c_temp.repeat_interleave(N, dim=0)              # :332, :350 'n d -> (n c) d'
    for i in range(0, cfg.depth, 2):
        h = transformer_block(sd, i, h, c_spatial, cfg.num_heads)                     # :370
        h = h.reshape(B, Fa, N, D).permute(0, 2, 1, 3).reshape(B * N, Fa, D)          # :372
        hv, hi = h[:, :Fr], h[:, Fr:]                                                 # :373-374
        if i == 0:
            hv = hv + sd["temp_embed"].to(dtype)                                      # :377-378
        hv = transformer_block(sd, i + 1, hv, c_temp, cfg.num_heads)                  # :387
        h = torch.cat([hv, hi], dim=1)                                                # :388
        h = h.reshape(B, N, Fa, D).permute(0, 2, 1, 3).reshape(B * Fa, N, D)          # :389
    o = final_layer(sd, h, c_spatial)                        # :395
    o = unpatchify(cfg, o)                                   # :396
    return o.reshape(B, Fa, *o.shape[1:])                    # :397
