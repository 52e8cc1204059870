"""CPU oracle for LatteT2V.forward on latents other than sample_size x sample_size — TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The reference forward reads height and width from its input (`models/latte_t2v.py:770`) and unpatchifies with them
(`:926-935`); diffusers 0.24.0's `PatchEmbed.forward` recomputes the 2-D sin-cos table when the patch grid is not the
configured one, scaling each axis to base_size = sample_size / patch (PixArt-alpha's interpolation).  This module restates
that, and runs `oracle/t2v_oracle.py`'s blocks (spatial, temporal, adaLN-single, caption projection) on the input's grid:
  * `get_2d_sincos_pos_embed` / `install_patch_embed_interpolation`: the (height, width) form of diffusers'
    get_2d_sincos_pos_embed and PatchEmbed.forward.  `oracle/make_golden_t2v_res.py` installs the latter on the shim's
    PatchEmbed (`oracle/ref_shim`, whose forward covers the configured grid only) before it runs the reference module.
    Like every diffusers leaf this is a restatement: no diffusers package is available offline.
  * `make_inputs`, `pos_embed_table`, `t2v_forward`: `oracle/t2v_oracle.py`'s functions for a height x width latent.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from . import latte_oracle as LO
from . import t2v_oracle as T


def get_2d_sincos_pos_embed(embed_dim, grid_size, base_size, interpolation_scale, sincos_1d=LO.sincos_1d_from_grid):
    """diffusers 0.24.0 get_2d_sincos_pos_embed: grid_size an int or (height, width); index / (size / base_size) /
    interpolation_scale along each axis, w-coordinates in the first half of the channels."""
    gh, gw = (grid_size, grid_size) if isinstance(grid_size, int) else grid_size
    ch = np.arange(gh, dtype=np.float32) / (gh / base_size) / interpolation_scale
    cw = np.arange(gw, dtype=np.float32) / (gw / base_size) / interpolation_scale
    grid = np.stack(np.meshgrid(cw, ch), axis=0).reshape([2, 1, gw, gh])    # as published; the data order stays (h, w)
    return np.concatenate([sincos_1d(embed_dim // 2, grid[0]), sincos_1d(embed_dim // 2, grid[1])], axis=1)


def install_patch_embed_interpolation(embeddings):
    """Give `embeddings.PatchEmbed` (the shim module) diffusers 0.24.0's forward: a latent whose patch grid differs from
    the configured one gets a table recomputed for its (height, width) grid with the configured base_size and
    interpolation_scale; the configured grid keeps the stored table."""
    def forward(self, latent):
        height, width = latent.shape[-2] // self.patch_size, latent.shape[-1] // self.patch_size
        latent = self.proj(latent).flatten(2).transpose(1, 2)
        if self.height != height or self.width != width:
            pos = get_2d_sincos_pos_embed(self.pos_embed.shape[-1], (height, width), self.base_size, self.interpolation_scale,
                                          embeddings.get_1d_sincos_pos_embed_from_grid)
            pos = torch.from_numpy(pos).float().unsqueeze(0).to(latent.device)
        else:
            pos = self.pos_embed
        return (latent + pos).to(latent.dtype)
    embeddings.PatchEmbed.forward = forward


def make_inputs(cfg: T.T2VConfig, batch: int, text_len: int, seed: int, height: int, width: int):
    """t2v_oracle.make_inputs for a height x width latent (the same draws in the same order)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(batch, cfg.in_channels, cfg.video_length, height, width, generator=g)
    t = torch.randint(0, 1000, (batch,), generator=g)
    text = torch.randn(batch, text_len, cfg.caption_channels, generator=g) * 0.5
    return x, t, text


def pos_embed_table(cfg: T.T2VConfig, grid_h: int, grid_w: int) -> torch.Tensor:
    """PatchEmbed's table of a grid_h x grid_w patch grid: base_size = sample_size / patch, interpolation_scale =
    max(sample_size // 64, 1) (latte_t2v.py:575-582)."""
    base = cfg.sample_size // cfg.patch_size
    return torch.from_numpy(get_2d_sincos_pos_embed(cfg.inner_dim, (grid_h, grid_w), base, max(cfg.sample_size // 64, 1))).float()


def t2v_forward(sd, cfg: T.T2VConfig, x, t, text, dtype=torch.float32, enable_temporal=True, text_mask=None):
    """t2v_oracle.t2v_forward (latte_t2v.py:729-941, eval) on x (B, C, F, H, W) of any H, W divisible by the patch."""
    B, C, Fr, Hh, Ww = x.shape
    D, p, heads = cfg.inner_dim, cfg.patch_size, cfg.num_attention_heads
    gh, gw = Hh // p, Ww // p
    N = gh * gw
    xf = x.permute(0, 2, 1, 3, 4).reshape(B * Fr, C, Hh, Ww).to(dtype)
    patches = xf.reshape(B * Fr, C, gh, p, gw, p).permute(0, 2, 4, 1, 3, 5).reshape(B * Fr, N, C * p * p)
    h = patches @ sd["pos_embed.proj.weight"].to(dtype).reshape(D, -1).t() + sd["pos_embed.proj.bias"].to(dtype)
    h = h + pos_embed_table(cfg, gh, gw).to(device=h.device, dtype=dtype)
    ts, emb = T.adaln_single(sd, t, dtype)
    txt = T._lin(sd, "caption_projection.linear_2", F.gelu(T._lin(sd, "caption_projection.linear_1", text.to(dtype)), approximate="tanh"))
    txt_sp = txt.repeat_interleave(Fr, dim=0)
    bias_sp = None
    if text_mask is not None:
        bias_sp = ((1 - text_mask.to(dtype)) * -10000.0).repeat_interleave(Fr, dim=0)
    ts_sp = ts.repeat_interleave(Fr, dim=0)
    ts_tm = ts.repeat_interleave(N, dim=0)
    for i in range(cfg.num_layers):
        h = T.spatial_block(sd, i, h, txt_sp, ts_sp, heads, bias_sp)
        if enable_temporal:
            h = h.reshape(B, Fr, N, D).permute(0, 2, 1, 3).reshape(B * N, Fr, D)
            if i == 0 and Fr > 1:
                h = h + T.temp_pos_embed_table(cfg).to(device=h.device, dtype=dtype)
            h = T.temporal_block(sd, i, h, ts_tm, heads)
            h = h.reshape(B, N, Fr, D).permute(0, 2, 1, 3).reshape(B * Fr, N, D)
    shift, scale = (sd["scale_shift_table"].to(dtype)[None] + emb.repeat_interleave(Fr, dim=0)[:, None]).chunk(2, dim=1)
    h = LO.layer_norm(h) * (1 + scale) + shift
    h = T._lin(sd, "proj_out", h)
    h = h.reshape(B * Fr, gh, gw, p, p, cfg.out_channels)
    h = torch.einsum("nhwpqc->nchpwq", h).reshape(B * Fr, cfg.out_channels, Hh, Ww)
    return h.reshape(B, Fr, cfg.out_channels, Hh, Ww).permute(0, 2, 1, 3, 4).contiguous()
