"""CPU oracle for LatteT2V video + image joint training (`use_image_num` > 0) -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Restates the training-mode branch of `/root/reference/models/latte_t2v.py:729-941` with images on top of the pieces of
oracle/t2v_oracle.py (spatial / temporal block, adaLN-single, caption projection, output head).  Pinned by
`oracle/make_golden_train_t2v_img.py`, which runs the UNMODIFIED reference module in `.train()` with `use_image_num`, and by
tests/test_oracle_train_t2v_img.py, which holds this restatement's autograd to those goldens.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from . import latte_oracle as LO
from .t2v_oracle import T2VConfig, _lin, adaln_single, pos_embed_table, spatial_block, t2v_forward, temporal_block


def make_img_inputs(cfg: T2VConfig, batch: int, images: int, text_len: int, seed: int = 7):
    """Inputs of video + image joint training: x (B, C, F + I, H, W), t (B,), text (B, 1 + I, L, caption_channels)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(batch, cfg.in_channels, cfg.video_length + images, cfg.sample_size, cfg.sample_size, generator=g)
    t = torch.randint(0, 1000, (batch,), generator=g)
    text = torch.randn(batch, 1 + images, text_len, cfg.caption_channels, generator=g) * 0.5
    return x, t, text


def t2v_train_forward(sd, cfg: T2VConfig, x, t, text, use_image_num, text_mask=None, dtype=torch.float32):
    """LatteT2V.forward in training mode (not checkpointed) with video + image joint training, use_image_num = I > 0
    (latte_t2v.py:729-941).  x (B, C, F + I, H, W) with F = cfg.video_length; text (B, 1 + I, L, caption_channels); text_mask
    None or the 3-D keep-mask (B, 1 + I, L) -> (B, out_channels, F + I, H, W).
      * caption (b, 0) serves the F video frames of sample b, caption (b, 1 + i) its image i (:789-796); the mask rows are
        repeated the same way and become the bias (1 - mask) * -10000 (:756-762);
      * conditioning stays per sample: ts[b] and emb[b] repeated over all F + I frames (:801, :919);
      * spatial blocks see all F + I frames; temporal blocks see the F video frames, the image frames pass through (:876-891);
      * temp_pos_embed is not added in this branch (only the non-image branch adds it, :894)."""
    if use_image_num == 0:
        return t2v_forward(sd, cfg, x, t, text, dtype, text_mask=text_mask)
    B, C, Fa, Hh, Ww = x.shape
    Fr, I = Fa - use_image_num, use_image_num
    D, p, heads = cfg.inner_dim, cfg.patch_size, cfg.num_attention_heads
    N = (Hh // p) * (Ww // p)
    xf = x.permute(0, 2, 1, 3, 4).reshape(B * Fa, C, Hh, Ww).to(dtype)                     # :731
    patches = xf.reshape(B * Fa, C, Hh // p, p, Ww // p, p).permute(0, 2, 4, 1, 3, 5).reshape(B * Fa, N, C * p * p)
    h = patches @ sd["pos_embed.proj.weight"].to(dtype).reshape(D, -1).t() + sd["pos_embed.proj.bias"].to(dtype)
    h = h + pos_embed_table(cfg).to(device=h.device, dtype=dtype)
    ts, emb = adaln_single(sd, t, dtype)                                                    # :782-784

    def per_frame(a):
        """(B, 1 + I, ...) -> (B*(F + I), ...): row 0 of each sample repeated over its F video frames, then its I rows."""
        return torch.cat((a[:, :1].expand(B, Fr, *a.shape[2:]), a[:, 1:]), dim=1).reshape(B * Fa, *a.shape[2:])
    txt = _lin(sd, "caption_projection.linear_2", F.gelu(_lin(sd, "caption_projection.linear_1", text.to(dtype)), approximate="tanh"))
    txt_sp = per_frame(txt)                                                                 # :791-796
    bias_sp = per_frame((1 - text_mask.to(dtype)) * -10000.0) if text_mask is not None else None     # :756-762
    ts_sp = ts.repeat_interleave(Fa, dim=0)                                                 # :801
    ts_tm = ts.repeat_interleave(N, dim=0)                                                  # :802
    for i in range(cfg.num_layers):
        h = spatial_block(sd, i, h, txt_sp, ts_sp, heads, bias_sp)                          # :862-870
        h = h.reshape(B, Fa, N, D).permute(0, 2, 1, 3)                                      # :874, (b t) f d
        hv = temporal_block(sd, i, h[:, :, :Fr].reshape(B * N, Fr, D), ts_tm, heads)         # :877-888
        h = torch.cat((hv.reshape(B, N, Fr, D), h[:, :, Fr:]), dim=2)                       # :890
        h = h.permute(0, 2, 1, 3).reshape(B * Fa, N, D)                                     # :891
    shift, scale = (sd["scale_shift_table"].to(dtype)[None] + emb.repeat_interleave(Fa, dim=0)[:, None]).chunk(2, dim=1)   # :919-923
    h = LO.layer_norm(h) * (1 + scale) + shift
    h = _lin(sd, "proj_out", h)
    g = Hh // p
    h = h.reshape(B * Fa, g, g, p, p, cfg.out_channels)
    h = torch.einsum("nhwpqc->nchpwq", h).reshape(B * Fa, cfg.out_channels, Hh, Ww)
    return h.reshape(B, Fa, cfg.out_channels, Hh, Ww).permute(0, 2, 1, 3, 4).contiguous()
