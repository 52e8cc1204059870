"""CPU oracle for LatteT2V.forward — TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Restates `/root/reference/models/latte_t2v.py` (Vchitect/Latte @ b27c24a) for the configuration the reference ships
(HF `maxin-cn/Latte-1` transformer config, SURVEY.md App. C.2: `norm_type="ada_norm_single"`, no affine LayerNorms,
`activation_fn="gelu-approximate"`, `attention_bias=True`, `caption_channels=4096`).  Control flow follows
`latte_t2v.py:729-941`; the temporal block follows `BasicTransformerBlock_` (`:294-299,314-325,364-367,385,389-392`).

Pin (round 2): `oracle/make_golden_t2v.py` runs the UNMODIFIED reference module (through `oracle/ref_shim/diffusers`,
which supplies only the library leaves it imports) and commits whole-forward outputs -- with and without temporal blocks,
with padded-prompt masks, at N = 64 / 256 / 1024 tokens per frame, and the 28-layer 16x512x512 Latte-1 shape -- plus
direct outputs of `BasicTransformerBlock_`, `AdaLayerNormSingle` and `FeedForward`; `tests/test_oracle_t2v.py` holds
this restatement to them.  So the forward control flow, the temporal block, adaLN-single, the feed-forward and the
mask -> bias conversion are **pinned to reference code**.  Still only shim-restated (diffusers==0.24.0, pinned in
`environment.yml:13`, is neither vendored nor installed and there is no network): the spatial `BasicTransformerBlock`,
`Attention`/`AttnProcessor2_0`, `PatchEmbed`, `CaptionProjection`, `CombinedTimestepSizeEmbeddings`.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import torch
import torch.nn.functional as F

from . import latte_oracle as LO


@dataclass(frozen=True)
class T2VConfig:
    num_attention_heads: int = 16
    attention_head_dim: int = 72
    in_channels: int = 4
    out_channels: int = 8
    num_layers: int = 28
    patch_size: int = 2
    sample_size: int = 64
    caption_channels: int = 4096
    video_length: int = 16

    @property
    def inner_dim(self) -> int:
        return self.num_attention_heads * self.attention_head_dim

    @property
    def num_patches(self) -> int:
        return (self.sample_size // self.patch_size) ** 2


def state_dict_spec(cfg: T2VConfig):
    D, p, C = cfg.inner_dim, cfg.patch_size, cfg.in_channels
    spec = [
        ("pos_embed.proj.weight", (D, C, p, p)), ("pos_embed.proj.bias", (D,)),
        ("adaln_single.emb.timestep_embedder.linear_1.weight", (D, 256)), ("adaln_single.emb.timestep_embedder.linear_1.bias", (D,)),
        ("adaln_single.emb.timestep_embedder.linear_2.weight", (D, D)), ("adaln_single.emb.timestep_embedder.linear_2.bias", (D,)),
        ("adaln_single.linear.weight", (6 * D, D)), ("adaln_single.linear.bias", (6 * D,)),
        ("caption_projection.linear_1.weight", (D, cfg.caption_channels)), ("caption_projection.linear_1.bias", (D,)),
        ("caption_projection.linear_2.weight", (D, D)), ("caption_projection.linear_2.bias", (D,)),
    ]

    def attn(prefix):
        out = []
        for n in ("to_q", "to_k", "to_v", "to_out.0"):
            out += [(f"{prefix}.{n}.weight", (D, D)), (f"{prefix}.{n}.bias", (D,))]
        return out

    def ff(prefix):
        return [(f"{prefix}.net.0.proj.weight", (4 * D, D)), (f"{prefix}.net.0.proj.bias", (4 * D,)),
                (f"{prefix}.net.2.weight", (D, 4 * D)), (f"{prefix}.net.2.bias", (D,))]

    for i in range(cfg.num_layers):
        b = f"transformer_blocks.{i}"
        spec += [(f"{b}.scale_shift_table", (6, D))] + attn(f"{b}.attn1") + attn(f"{b}.attn2") + ff(f"{b}.ff")
    for i in range(cfg.num_layers):
        b = f"temporal_transformer_blocks.{i}"
        spec += [(f"{b}.scale_shift_table", (6, D))] + attn(f"{b}.attn1") + ff(f"{b}.ff")
    spec += [("scale_shift_table", (2, D)), ("proj_out.weight", (p * p * cfg.out_channels, D)), ("proj_out.bias", (p * p * cfg.out_channels,))]
    return spec


def make_weights(cfg: T2VConfig, seed: int = 0):
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for name, shape in state_dict_spec(cfg):
        if name.endswith(".bias"):
            t = torch.randn(shape, generator=g) * 0.05
        elif name.endswith("scale_shift_table"):
            t = torch.randn(shape, generator=g) / math.sqrt(shape[-1]) * 4.0
        elif name == "pos_embed.proj.weight":
            t = torch.randn(shape, generator=g) * 0.25
        elif name == "adaln_single.linear.weight":
            t = torch.randn(shape, generator=g) * (0.5 / math.sqrt(shape[1]))
        else:
            t = torch.randn(shape, generator=g) * (1.0 / math.sqrt(shape[-1]))
        sd[name] = t.contiguous()
    return sd


def make_inputs(cfg: T2VConfig, batch: int, text_len: int, seed: int = 7):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(batch, cfg.in_channels, cfg.video_length, cfg.sample_size, cfg.sample_size, generator=g)
    t = torch.randint(0, 1000, (batch,), generator=g)
    text = torch.randn(batch, text_len, cfg.caption_channels, generator=g) * 0.5
    return x, t, text


# ---------------------------------------------------------------------------------------------- pieces
def pos_embed_table(cfg: T2VConfig) -> torch.Tensor:
    """diffusers PatchEmbed pos_embed: 2-D sin-cos on a grid of sample_size/patch with base_size = that grid and
    interpolation_scale = max(sample_size // 64, 1) (latte_t2v.py:575-582): coordinates are grid / (grid/base) / scale."""
    import numpy as np
    grid = cfg.sample_size // cfg.patch_size
    scale = max(cfg.sample_size // 64, 1)
    coords = np.arange(grid, dtype=np.float32) / (grid / grid) / scale
    ww, hh = np.meshgrid(coords, coords)
    emb = np.concatenate([LO.sincos_1d_from_grid(cfg.inner_dim // 2, ww), LO.sincos_1d_from_grid(cfg.inner_dim // 2, hh)], axis=1)
    return torch.from_numpy(emb).float()


def temp_pos_embed_table(cfg: T2VConfig) -> torch.Tensor:
    """latte_t2v.py:669-671, :943-944 -> same 1-D table as Latte."""
    return torch.from_numpy(LO.sincos_temp(cfg.inner_dim, cfg.video_length)).float()


def _lin(sd, name, x):
    return F.linear(x, sd[name + ".weight"].to(x.dtype), sd[name + ".bias"].to(x.dtype))


def attention(sd, prefix, x, ctx, heads, key_bias=None):
    """diffusers Attention + AttnProcessor2_0: to_q(x), to_k/to_v(ctx), per-head softmax(q k^T / sqrt(hd) + bias) v,
    to_out[0].  key_bias (B, L): additive, broadcast over heads and queries (latte_t2v.py:766-771)."""
    B, S, D = x.shape
    hd = D // heads
    q = _lin(sd, prefix + ".to_q", x).reshape(B, S, heads, hd).transpose(1, 2)
    k = _lin(sd, prefix + ".to_k", ctx).reshape(B, -1, heads, hd).transpose(1, 2)
    v = _lin(sd, prefix + ".to_v", ctx).reshape(B, -1, heads, hd).transpose(1, 2)
    scores = q @ k.transpose(-1, -2) * hd ** -0.5
    if key_bias is not None:
        scores = scores + key_bias.to(scores.dtype)[:, None, None, :]
    a = torch.softmax(scores, dim=-1)
    o = (a @ v).transpose(1, 2).reshape(B, S, D)
    return _lin(sd, prefix + ".to_out.0", o)


def feed_forward(sd, prefix, x):
    """FeedForward('gelu-approximate') (latte_t2v.py:96-111): Linear -> GELU(tanh) -> Linear."""
    h = F.gelu(_lin(sd, prefix + ".net.0.proj", x), approximate="tanh")
    return _lin(sd, prefix + ".net.2", h)


def spatial_block(sd, i, x, text, ts, heads, text_bias=None):
    """diffusers BasicTransformerBlock, ada_norm_single (SURVEY.md App. C.3; call at latte_t2v.py:862-870).
    x (B*F, N, D), text (B*F, L, D), ts (B*F, 6D), text_bias (B*F, L) additive or None."""
    p = f"transformer_blocks.{i}"
    n = x.shape[0]
    sh1, sc1, g1, sh2, sc2, g2 = (sd[p + ".scale_shift_table"].to(x.dtype)[None] + ts.reshape(n, 6, -1)).chunk(6, dim=1)
    h = LO.layer_norm(x) * (1 + sc1) + sh1
    x = x + g1 * attention(sd, p + ".attn1", h, h, heads)
    x = x + attention(sd, p + ".attn2", x, text, heads, text_bias)   # no norm before attn2 in this mode
    h = LO.layer_norm(x) * (1 + sc2) + sh2
    return x + g2 * feed_forward(sd, p + ".ff", h)


def temporal_block(sd, i, x, ts, heads):
    """BasicTransformerBlock_ (latte_t2v.py:294-299,314-325,364-367,385,389-392). x (B*N, F, D), ts (B*N, 6D)."""
    p = f"temporal_transformer_blocks.{i}"
    n = x.shape[0]
    sh1, sc1, g1, sh2, sc2, g2 = (sd[p + ".scale_shift_table"].to(x.dtype)[None] + ts.reshape(n, 6, -1)).chunk(6, dim=1)
    h = LO.layer_norm(x) * (1 + sc1) + sh1
    x = x + g1 * attention(sd, p + ".attn1", h, h, heads)
    h = LO.layer_norm(x) * (1 + sc2) + sh2                        # norm3
    return x + g2 * feed_forward(sd, p + ".ff", h)


def adaln_single(sd, t, dtype=torch.float32):
    """AdaLayerNormSingle (latte_t2v.py:398-428): emb = TimestepEmbedding(Timesteps(t)); returns (Linear(SiLU(emb)), emb)."""
    tf = LO.timestep_embedding(t).to(dtype)
    emb = _lin(sd, "adaln_single.emb.timestep_embedder.linear_2", F.silu(_lin(sd, "adaln_single.emb.timestep_embedder.linear_1", tf)))
    return _lin(sd, "adaln_single.linear", F.silu(emb)), emb


def t2v_forward(sd, cfg: T2VConfig, x, t, text, dtype=torch.float32, enable_temporal=True, text_mask=None):
    """LatteT2V.forward (latte_t2v.py:729-941), eval mode, use_image_num = 0.
    x (B, C, F, H, W); t (B,); text (B, L, caption_channels); text_mask (B, L) 1 = keep / 0 = discard or None
    (encoder_attention_mask, converted to the bias (1 - mask) * -10000 and repeated per frame, :766-771)
    -> (B, out_channels, F, H, W)."""
    B, C, Fr, Hh, Ww = x.shape
    D, p, heads = cfg.inner_dim, cfg.patch_size, cfg.num_attention_heads
    N = (Hh // p) * (Ww // p)
    # :731 rearrange to (b f) c h w ; :773 PatchEmbed conv + pos_embed
    xf = x.permute(0, 2, 1, 3, 4).reshape(B * Fr, C, Hh, Ww).to(dtype)
    patches = xf.reshape(B * Fr, C, Hh // p, p, Ww // p, p).permute(0, 2, 4, 1, 3, 5).reshape(B * Fr, N, C * p * p)
    h = patches @ sd["pos_embed.proj.weight"].to(dtype).reshape(D, -1).t() + sd["pos_embed.proj.bias"].to(dtype)
    h = h + pos_embed_table(cfg).to(device=h.device, dtype=dtype)
    # :782-784 adaln_single: emb = TimestepEmbedding(Timesteps(t)); ts = Linear(SiLU(emb))
    ts, emb = adaln_single(sd, t, dtype)
    # :789 caption projection, :798 repeat per frame
    txt = _lin(sd, "caption_projection.linear_2", F.gelu(_lin(sd, "caption_projection.linear_1", text.to(dtype)), approximate="tanh"))
    txt_sp = txt.repeat_interleave(Fr, dim=0)
    bias_sp = None
    if text_mask is not None:
        bias_sp = ((1 - text_mask.to(dtype)) * -10000.0).repeat_interleave(Fr, dim=0)
    ts_sp = ts.repeat_interleave(Fr, dim=0)            # :801
    ts_tm = ts.repeat_interleave(N, dim=0)             # :802
    for i in range(cfg.num_layers):
        h = spatial_block(sd, i, h, txt_sp, ts_sp, heads, bias_sp)                          # :862-870
        if enable_temporal:
            h = h.reshape(B, Fr, N, D).permute(0, 2, 1, 3).reshape(B * N, Fr, D)            # :874
            if i == 0 and Fr > 1:
                h = h + temp_pos_embed_table(cfg).to(device=h.device, dtype=dtype)          # :894-895
            h = temporal_block(sd, i, h, ts_tm, heads)                                      # :897-905
            h = h.reshape(B, N, Fr, D).permute(0, 2, 1, 3).reshape(B * Fr, N, D)            # :907
    # :918-924 output head
    shift, scale = (sd["scale_shift_table"].to(dtype)[None] + emb.repeat_interleave(Fr, dim=0)[:, None]).chunk(2, dim=1)
    h = LO.layer_norm(h) * (1 + scale) + shift
    h = _lin(sd, "proj_out", h)
    # :929-936 unpatchify -> (b f) c H W -> b c f H W
    g = Hh // p
    h = h.reshape(B * Fr, g, g, p, p, cfg.out_channels)
    h = torch.einsum("nhwpqc->nchpwq", h).reshape(B * Fr, cfg.out_channels, Hh, Ww)
    return h.reshape(B, Fr, cfg.out_channels, Hh, Ww).permute(0, 2, 1, 3, 4).contiguous()


def gemm_flops_per_video(cfg: T2VConfig, text_len: int) -> float:
    """The Linear-layer part of `algorithmic_flops_per_video` (everything the wgmma GEMM kernel executes)."""
    D, N, Fr, L = cfg.inner_dim, cfg.num_patches, cfg.video_length, cfg.num_layers
    T = N * Fr
    sp_lin = 2.0 * T * (3 * D * D + D * D + 2 * D * D + 8 * D * D)
    tm_lin = 2.0 * T * (3 * D * D + D * D + 8 * D * D)
    kv = 2.0 * text_len * D * 2 * D
    cap = 2.0 * text_len * (cfg.caption_channels * D + D * D)
    return (sp_lin + tm_lin + kv) * L + cap


def algorithmic_flops_per_video(cfg: T2VConfig, text_len: int) -> float:
    """SURVEY.md App. A, T2V row: text K/V projected once per sample."""
    D, N, Fr, L = cfg.inner_dim, cfg.num_patches, cfg.video_length, cfg.num_layers
    T = N * Fr
    sp_lin = 2.0 * T * (3 * D * D + D * D + 2 * D * D + 8 * D * D)      # qkv, out, cross q + out, ff
    tm_lin = 2.0 * T * (3 * D * D + D * D + 8 * D * D)
    attn = 4.0 * N * N * D * Fr + 4.0 * N * text_len * D * Fr + 4.0 * Fr * Fr * D * N
    kv = 2.0 * text_len * D * 2 * D
    cap = 2.0 * text_len * (cfg.caption_channels * D + D * D)
    return (sp_lin + tm_lin + attn + kv) * L + cap
