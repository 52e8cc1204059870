"""`AutoencoderKL` — the decode half of the SD-VAE the reference samplers call once after the loop
(`vae.decode(samples / 0.18215).sample`, sample/sample.py:114, sample_ddp.py:167, pipeline_latte.py:758,771), backed by
TMA implicit-GEMM convolutions on the wgmma GEMM kernel (`b200_vae_decode`), and the encode half train.py calls on every
batch (`vae.encode(x).latent_dist.sample()`, train.py:206-211; `b200_vae_encode`, SURVEY.md §8(f) rank 4).  Parameter names
follow the diffusers 0.24.0 `AutoencoderKL` state dict (encoder.*, quant_conv.*, post_quant_conv.*, decoder.*), so
`vae/diffusion_pytorch_model.safetensors` loads unchanged.  **Parity unpinned** (diffusers absent offline).  No CPU path."""
from __future__ import annotations

import ctypes as C
import json
import os
from types import SimpleNamespace

import torch
import torch.nn as nn

from . import _lib
from ._cache import DeviceCacheMixin


# ---- weight layouts of the native layers (the packers below and the op-level tests both use these) -------------------
def pack_conv3x3(wt):
    """Conv2d 3x3 weight OIHW -> [O][tap = ky*3+kx][I] as a 2-D [O, 9I] view (b200_vae_conv, B200_VAE_CONV3X3)."""
    return wt.detach().permute(0, 2, 3, 1).reshape(wt.shape[0], -1)


def pack_linear(wt):
    """nn.Linear [O, I] or 1x1 Conv2d [O, I, 1, 1] weight -> [O, I]."""
    return wt.detach().reshape(wt.shape[0], -1)


def pack_conv_t3(wt, scale=1.0):
    """Conv3d (3,1,1) weight [O][I][kt][1][1] -> fp32 [O][kt][I] as [O, 3I], times `scale` (B200_VAE_CONV_T3)."""
    return (wt.detach().float() * scale).reshape(wt.shape[0], wt.shape[1], 3).permute(0, 2, 1).reshape(wt.shape[0], -1)


def pack_down2(wt):
    """Conv2d(C, C, 3, stride 2) after F.pad (0,1,0,1) -> 2x2-tap conv over the space-to-depth input: input pixel (2y+dy,
    2x+dx) is phase (dy & 1, dx & 1) at offset (dy >> 1, dx >> 1); fp32 [O][tap = oy*2+ox][phase = py*2+px][I] as [O, 16I],
    zeros at (phase 1, offset 1), which no 3x3 tap reaches (B200_VAE_CONV_DOWN2)."""
    O, I = wt.shape[:2]
    out = torch.zeros(O, 2, 2, 2, 2, I, dtype=torch.float32, device=wt.device)     # [O][oy][ox][py][px][I]
    w = wt.detach().float()
    for dy in range(3):
        for dx in range(3):
            out[:, dy >> 1, dx >> 1, dy & 1, dx & 1, :] = w[:, :, dy, dx]
    return out.reshape(O, -1)


def fold_v_bias(o_w, o_b, v_b):
    """softmax rows sum to 1, so P (V + 1 b_v^T) W_o^T + b_o = P V W_o^T + (W_o b_v + b_o): the fp32 output bias of the
    mid-block attention with the v bias folded in (b200_vae_mid_attention takes no v bias)."""
    return o_b.detach().float() + o_w.detach().float() @ v_b.detach().float()


class _Resnet(nn.Module):
    def __init__(self, cin, cout, groups):
        super().__init__()
        self.norm1 = nn.GroupNorm(groups, cin, eps=1e-6)
        self.conv1 = nn.Conv2d(cin, cout, 3, padding=1)
        self.norm2 = nn.GroupNorm(groups, cout, eps=1e-6)
        self.conv2 = nn.Conv2d(cout, cout, 3, padding=1)
        if cin != cout:
            self.conv_shortcut = nn.Conv2d(cin, cout, 1)


class _Attention(nn.Module):
    def __init__(self, c, groups):
        super().__init__()
        self.group_norm = nn.GroupNorm(groups, c, eps=1e-6)
        self.to_q = nn.Linear(c, c)
        self.to_k = nn.Linear(c, c)
        self.to_v = nn.Linear(c, c)
        self.to_out = nn.ModuleList([nn.Linear(c, c), nn.Dropout(0.0)])


class _Mid(nn.Module):
    def __init__(self, c, groups):
        super().__init__()
        self.attentions = nn.ModuleList([_Attention(c, groups)])
        self.resnets = nn.ModuleList([_Resnet(c, c, groups), _Resnet(c, c, groups)])


class _Upsampler(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.conv = nn.Conv2d(c, c, 3, padding=1)


class _UpBlock(nn.Module):
    def __init__(self, cin, cout, n, groups, add_upsample):
        super().__init__()
        self.resnets = nn.ModuleList([_Resnet(cin if i == 0 else cout, cout, groups) for i in range(n)])
        if add_upsample:
            self.upsamplers = nn.ModuleList([_Upsampler(cout)])


class _Decoder(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        up = tuple(reversed(cfg.block_out_channels))
        g = cfg.norm_num_groups
        self.conv_in = nn.Conv2d(cfg.latent_channels, up[0], 3, padding=1)
        self.mid_block = _Mid(up[0], g)
        blocks, cin = [], up[0]
        for i, co in enumerate(up):
            blocks.append(_UpBlock(cin, co, cfg.layers_per_block + 1, g, i + 1 < len(up)))
            cin = co
        self.up_blocks = nn.ModuleList(blocks)
        self.conv_norm_out = nn.GroupNorm(g, up[-1], eps=1e-6)
        self.conv_out = nn.Conv2d(up[-1], cfg.out_channels, 3, padding=1)


class DecoderOutput(SimpleNamespace):
    pass


class AutoencoderKLOutput(SimpleNamespace):
    pass


class _Downsampler(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.conv = nn.Conv2d(c, c, 3, stride=2, padding=0)     # diffusers Downsample2D(padding=0): F.pad (0,1,0,1) first


class _DownBlock(nn.Module):
    def __init__(self, cin, cout, n, groups, add_downsample):
        super().__init__()
        self.resnets = nn.ModuleList([_Resnet(cin if i == 0 else cout, cout, groups) for i in range(n)])
        if add_downsample:
            self.downsamplers = nn.ModuleList([_Downsampler(cout)])


class _Encoder(nn.Module):
    """diffusers 0.24.0 `Encoder` parameter layout (encoder.conv_in, down_blocks.i.resnets.j, downsamplers.0.conv, mid_block,
    conv_norm_out, conv_out with 2 * latent_channels outputs)."""

    def __init__(self, cfg):
        super().__init__()
        ch, g = tuple(cfg.block_out_channels), cfg.norm_num_groups
        self.conv_in = nn.Conv2d(cfg.in_channels, ch[0], 3, padding=1)
        blocks, cin = [], ch[0]
        for i, co in enumerate(ch):
            blocks.append(_DownBlock(cin, co, cfg.layers_per_block, g, i + 1 < len(ch)))
            cin = co
        self.down_blocks = nn.ModuleList(blocks)
        self.mid_block = _Mid(ch[-1], g)
        self.conv_norm_out = nn.GroupNorm(g, ch[-1], eps=1e-6)
        self.conv_out = nn.Conv2d(ch[-1], 2 * cfg.latent_channels, 3, padding=1)


class DiagonalGaussianDistribution:
    """diffusers.models.vae.DiagonalGaussianDistribution on the (n, 2L, h, w) moments: mean | logvar, logvar clamped to
    [-30, 20]; `sample()` = mean + std * randn (train.py:210), `mode()` = mean."""

    def __init__(self, parameters, deterministic=False):
        self.parameters = parameters
        self.mean, self.logvar = torch.chunk(parameters, 2, dim=1)
        self.logvar = torch.clamp(self.logvar, -30.0, 20.0)
        self.deterministic = deterministic
        self.std = torch.exp(0.5 * self.logvar)
        self.var = torch.exp(self.logvar)
        if deterministic:
            self.var = self.std = torch.zeros_like(self.mean)

    def sample(self, generator=None):
        noise = torch.randn(self.mean.shape, generator=generator, device=self.parameters.device, dtype=self.parameters.dtype)
        return self.mean + self.std * noise

    def mode(self):
        return self.mean

    def kl(self, other=None):
        if self.deterministic:
            return torch.zeros(self.mean.shape[0], device=self.mean.device)
        if other is None:
            return 0.5 * torch.sum(torch.pow(self.mean, 2) + self.var - 1.0 - self.logvar, dim=[1, 2, 3])
        return 0.5 * torch.sum(torch.pow(self.mean - other.mean, 2) / other.var + self.var / other.var - 1.0 - self.logvar + other.logvar,
                               dim=[1, 2, 3])


# ---- AutoencoderKLTemporalDecoder containers (diffusers 0.24.0 names) --------------------------------------------
class _TemporalResnet(nn.Module):
    def __init__(self, c, groups):
        super().__init__()
        self.norm1 = nn.GroupNorm(groups, c, eps=1e-5)
        self.conv1 = nn.Conv3d(c, c, (3, 1, 1), padding=(1, 0, 0))
        self.norm2 = nn.GroupNorm(groups, c, eps=1e-5)
        self.conv2 = nn.Conv3d(c, c, (3, 1, 1), padding=(1, 0, 0))


class _Mixer(nn.Module):
    def __init__(self):
        super().__init__()
        self.mix_factor = nn.Parameter(torch.zeros(1))


class _STBlock(nn.Module):
    def __init__(self, cin, cout, groups):
        super().__init__()
        self.spatial_res_block = _Resnet(cin, cout, groups)
        self.temporal_res_block = _TemporalResnet(cout, groups)
        self.time_mixer = _Mixer()


class _TMid(nn.Module):
    def __init__(self, c, groups):
        super().__init__()
        self.attentions = nn.ModuleList([_Attention(c, groups)])
        self.resnets = nn.ModuleList([_STBlock(c, c, groups), _STBlock(c, c, groups)])


class _TUpBlock(nn.Module):
    def __init__(self, cin, cout, n, groups, add_upsample):
        super().__init__()
        self.resnets = nn.ModuleList([_STBlock(cin if i == 0 else cout, cout, groups) for i in range(n)])
        if add_upsample:
            self.upsamplers = nn.ModuleList([_Upsampler(cout)])


class _TemporalDecoder(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        up = tuple(reversed(cfg.block_out_channels))
        g = cfg.norm_num_groups
        self.conv_in = nn.Conv2d(cfg.latent_channels, up[0], 3, padding=1)
        self.mid_block = _TMid(up[0], g)
        blocks, cin = [], up[0]
        for i, co in enumerate(up):
            blocks.append(_TUpBlock(cin, co, cfg.layers_per_block + 1, g, i + 1 < len(up)))
            cin = co
        self.up_blocks = nn.ModuleList(blocks)
        self.conv_norm_out = nn.GroupNorm(g, up[-1], eps=1e-6)
        self.conv_out = nn.Conv2d(up[-1], cfg.out_channels, 3, padding=1)
        self.time_conv_out = nn.Conv3d(cfg.out_channels, cfg.out_channels, (3, 1, 1), padding=(1, 0, 0))


class AutoencoderKL(DeviceCacheMixin, nn.Module):
    def __init__(self, in_channels=3, out_channels=3, block_out_channels=(128, 256, 512, 512), layers_per_block=2,
                 latent_channels=4, norm_num_groups=32, scaling_factor=0.18215, **unused):
        super().__init__()
        self.config = SimpleNamespace(in_channels=in_channels, out_channels=out_channels, block_out_channels=tuple(block_out_channels),
                                      layers_per_block=layers_per_block, latent_channels=latent_channels,
                                      norm_num_groups=norm_num_groups, scaling_factor=scaling_factor)
        self._temporal = type(self).__name__ == "AutoencoderKLTemporalDecoder"
        if self._temporal:
            self.decoder = _TemporalDecoder(self.config)     # no post_quant_conv in the SVD decoder
        else:
            self.encoder = _Encoder(self.config)
            self.quant_conv = nn.Conv2d(2 * latent_channels, 2 * latent_channels, 1)
            self.post_quant_conv = nn.Conv2d(latent_channels, latent_channels, 1)
            self.decoder = _Decoder(self.config)
        self.compute_dtype = torch.float16
        self._packed = None
        self._packed_key = None
        self._workspace = None
        self._packed_enc = None

    @property
    def dtype(self):
        return self.decoder.conv_in.weight.dtype

    @classmethod
    def from_pretrained(cls, path, subfolder=None, torch_dtype=None, **kw):
        root = os.path.join(path, subfolder) if subfolder else path
        with open(os.path.join(root, "config.json")) as f:
            cfg = {k: v for k, v in json.load(f).items() if not k.startswith("_")}
        model = cls(**cfg)
        st = os.path.join(root, "diffusion_pytorch_model.safetensors")
        if os.path.exists(st):
            from safetensors.torch import load_file
            sd = load_file(st)
        else:
            sd = torch.load(os.path.join(root, "diffusion_pytorch_model.bin"), map_location="cpu")
        own = model.state_dict()
        # the SVD temporal decoder checkpoint also carries the image encoder; this class keeps only what its decode uses
        missing = [k for k in own if k not in sd and not k.startswith(("encoder.", "quant_conv."))]
        if missing:
            raise RuntimeError(f"checkpoint {st} lacks {missing[:4]} ...")
        model.load_state_dict({k: v for k, v in sd.items() if k in own}, strict=False)
        return model.to(torch_dtype) if torch_dtype is not None else model

    # ---------------------------------------------------------------------------------------------
    @torch.no_grad()
    def _pack_encoder(self):
        enc = self.encoder
        ver = sum(p._version for p in enc.parameters()) + sum(p._version for p in self.quant_conv.parameters())
        w0 = enc.conv_in.weight
        key = (ver, w0.data_ptr(), w0.device, w0.dtype, self.compute_dtype)
        if self._packed_enc is not None and self._packed_enc[2] == key:
            return self._packed_enc
        dev, c = w0.device, self.config
        od = w0.dtype if w0.dtype in (torch.float16, torch.bfloat16) else self.compute_dtype
        keep = []

        def f32(t):
            t = t.detach().to(device=dev, dtype=torch.float32).contiguous()
            keep.append(t)
            return t.data_ptr()

        def t16(t):
            t = t.to(device=dev, dtype=od).contiguous()
            keep.append(t)
            return t.data_ptr()

        conv16 = lambda wt: t16(pack_conv3x3(wt))      # noqa: E731
        lin16 = lambda wt: t16(pack_linear(wt))        # noqa: E731
        down16 = lambda wt: t16(pack_down2(wt))        # noqa: E731

        def resnet(r):
            s = _lib.VaeResnet()
            s.gn1_g, s.gn1_b, s.conv1_w16, s.conv1_b = f32(r.norm1.weight), f32(r.norm1.bias), conv16(r.conv1.weight), f32(r.conv1.bias)
            s.gn2_g, s.gn2_b, s.conv2_w16, s.conv2_b = f32(r.norm2.weight), f32(r.norm2.bias), conv16(r.conv2.weight), f32(r.conv2.bias)
            s.cin, s.cout = r.conv1.weight.shape[1], r.conv1.weight.shape[0]
            if hasattr(r, "conv_shortcut"):
                s.short_w16, s.short_b = lin16(r.conv_shortcut.weight), f32(r.conv_shortcut.bias)
            else:
                s.short_w16, s.short_b = None, None
            return s

        e = _lib.VaeEncoder()
        ch = tuple(c.block_out_channels)
        e.in_channels, e.n_down, e.groups, e.latent_channels = c.in_channels, len(ch), c.norm_num_groups, c.latent_channels
        for i in range(4):
            e.down_channels[i] = ch[i] if i < len(ch) else 0
        e.dtype = _lib.BF16 if od == torch.bfloat16 else _lib.FP16
        e.eps = 1e-6
        e.conv_in_w, e.conv_in_b = f32(enc.conv_in.weight), f32(enc.conv_in.bias)
        for b, blk in enumerate(enc.down_blocks):
            for r in range(2):
                e.down[b * 2 + r] = resnet(blk.resnets[r])
            if hasattr(blk, "downsamplers"):
                e.down_w16[b], e.down_b[b] = down16(blk.downsamplers[0].conv.weight), f32(blk.downsamplers[0].conv.bias)
        e.mid[0], e.mid[1] = resnet(enc.mid_block.resnets[0]), resnet(enc.mid_block.resnets[1])
        at = enc.mid_block.attentions[0]
        e.attn_gn_g, e.attn_gn_b = f32(at.group_norm.weight), f32(at.group_norm.bias)
        e.attn_q_w16, e.attn_q_b = lin16(at.to_q.weight), f32(at.to_q.bias)
        e.attn_k_w16, e.attn_k_b = lin16(at.to_k.weight), f32(at.to_k.bias)
        e.attn_v_w16, e.attn_o_w16 = lin16(at.to_v.weight), lin16(at.to_out[0].weight)
        e.attn_o_b = f32(fold_v_bias(at.to_out[0].weight, at.to_out[0].bias, at.to_v.bias))
        e.norm_out_g, e.norm_out_b = f32(enc.conv_norm_out.weight), f32(enc.conv_norm_out.bias)
        M = 2 * c.latent_channels
        wo = torch.zeros(32, *enc.conv_out.weight.shape[1:], dtype=torch.float32, device=dev)
        wo[:M] = enc.conv_out.weight.detach().float()
        bo = torch.zeros(32, dtype=torch.float32, device=dev)
        bo[:M] = enc.conv_out.bias.detach().float()
        e.conv_out_w16, e.conv_out_b = conv16(wo), f32(bo)
        e.quant_w, e.quant_b = f32(self.quant_conv.weight.reshape(M, M)), f32(self.quant_conv.bias)
        self._packed_enc = (e, keep, key)
        return self._packed_enc

    def encode(self, x, return_dict=True):
        """x (n, 3, H, W) in [-1, 1] -> AutoencoderKLOutput(latent_dist=DiagonalGaussianDistribution) -- the call train.py:206-211
        makes on every batch (`vae.encode(x).latent_dist.sample().mul_(0.18215)`).  The moments (n, 2L, H/8, W/8) come from
        `b200_vae_encode`; the reparameterised sample stays a torch expression on that small tensor (its RNG is the caller's)."""
        if self._temporal:
            raise NotImplementedError("AutoencoderKLTemporalDecoder.encode is outside the built path (the pipelines only decode with it)")
        if not x.is_cuda:
            raise RuntimeError("latte_b200.AutoencoderKL runs on CUDA (sm_90a) only; there is no CPU fallback")
        lib = _lib.load()
        dev = x.device
        n, ci, h, w = x.shape
        f = 2 ** (len(self.config.block_out_channels) - 1)
        with torch.cuda.device(dev):
            e, _, _ = self._pack_encoder()
            xf = x.detach().to(torch.float32).contiguous()
            moments = torch.empty(n, 2 * self.config.latent_channels, h // f, w // f, dtype=torch.float32, device=dev)
            need = lib.b200_vae_encode_workspace_bytes(C.byref(e), n, h, w)
            if need == 0:
                raise RuntimeError("latte_b200: unsupported VAE encode configuration: " + _lib.last_error())
            base = self._aligned_workspace(need, dev)
            rc = lib.b200_vae_encode(C.byref(e), xf.data_ptr(), n, h, w, moments.data_ptr(), base, need,
                                     torch.cuda.current_stream(dev).cuda_stream)
            _lib.check(rc, "b200_vae_encode")
        pd = self.dtype
        dist = DiagonalGaussianDistribution(moments if pd == torch.float32 else moments.to(pd))
        return AutoencoderKLOutput(latent_dist=dist) if return_dict else (dist,)

    # ---------------------------------------------------------------------------------------------
    @torch.no_grad()
    def _pack(self):
        ver = sum(p._version for p in self.parameters())
        w0 = self.decoder.conv_in.weight
        key = (ver, w0.data_ptr(), w0.device, w0.dtype, self.compute_dtype)
        if self._packed is not None and key == self._packed_key:
            return self._packed
        dev, c = w0.device, self.config
        od = w0.dtype if w0.dtype in (torch.float16, torch.bfloat16) else self.compute_dtype
        keep = []

        def f32(t):
            t = t.detach().to(device=dev, dtype=torch.float32).contiguous()
            keep.append(t)
            return t.data_ptr()

        def t16(t):
            t = t.to(device=dev, dtype=od).contiguous()
            keep.append(t)
            return t.data_ptr()

        conv16 = lambda wt: t16(pack_conv3x3(wt))                           # noqa: E731
        lin16 = lambda wt: t16(pack_linear(wt))                             # noqa: E731
        conv16_t = lambda wt, scale=1.0: t16(pack_conv_t3(wt, scale))       # noqa: E731

        def resnet(blk):
            r = blk.spatial_res_block if self._temporal else blk
            s = _lib.VaeResnet()
            s.gn1_g, s.gn1_b, s.conv1_w16, s.conv1_b = f32(r.norm1.weight), f32(r.norm1.bias), conv16(r.conv1.weight), f32(r.conv1.bias)
            s.gn2_g, s.gn2_b, s.conv2_w16, s.conv2_b = f32(r.norm2.weight), f32(r.norm2.bias), conv16(r.conv2.weight), f32(r.conv2.bias)
            s.cin, s.cout = r.conv1.weight.shape[1], r.conv1.weight.shape[0]
            if hasattr(r, "conv_shortcut"):
                s.short_w16, s.short_b = lin16(r.conv_shortcut.weight), f32(r.conv_shortcut.bias)
            else:
                s.short_w16, s.short_b = None, None
            if self._temporal:
                t = blk.temporal_res_block
                # AlphaBlender(learned, switch_spatial_to_temporal_mix): alpha = 1 - sigmoid(mix); out = x_s + (1 - alpha) * conv2(...)
                one_minus_alpha = float(torch.sigmoid(blk.time_mixer.mix_factor.detach().float()))
                s.t_gn1_g, s.t_gn1_b, s.t_conv1_w16, s.t_conv1_b = f32(t.norm1.weight), f32(t.norm1.bias), conv16_t(t.conv1.weight), f32(t.conv1.bias)
                s.t_gn2_g, s.t_gn2_b = f32(t.norm2.weight), f32(t.norm2.bias)
                s.t_conv2_w16, s.t_conv2_b = conv16_t(t.conv2.weight, one_minus_alpha), f32(t.conv2.bias.detach().float() * one_minus_alpha)
            return s

        dec = self.decoder
        up = tuple(reversed(c.block_out_channels))
        d = _lib.VaeDecoder()
        d.latent_channels, d.layers_per_block, d.n_up, d.groups = c.latent_channels, c.layers_per_block, len(up), c.norm_num_groups
        for i in range(4):
            d.up_channels[i] = up[i] if i < len(up) else 0
        d.dtype = _lib.BF16 if od == torch.bfloat16 else _lib.FP16
        d.eps = 1e-6
        if self._temporal:
            d.pq_w, d.pq_b = None, None
            d.temporal_eps = 1e-5
            d.time_conv_w, d.time_conv_b = f32(dec.time_conv_out.weight.reshape(c.out_channels, c.out_channels, 3)), f32(dec.time_conv_out.bias)
        else:
            d.pq_w, d.pq_b = f32(self.post_quant_conv.weight.reshape(c.latent_channels, c.latent_channels)), f32(self.post_quant_conv.bias)
            d.temporal_eps = 1e-5
            d.time_conv_w, d.time_conv_b = None, None
        d.conv_in_w, d.conv_in_b = f32(dec.conv_in.weight), f32(dec.conv_in.bias)
        d.mid[0], d.mid[1] = resnet(dec.mid_block.resnets[0]), resnet(dec.mid_block.resnets[1])
        at = dec.mid_block.attentions[0]
        d.attn_gn_g, d.attn_gn_b = f32(at.group_norm.weight), f32(at.group_norm.bias)
        d.attn_q_w16, d.attn_q_b = lin16(at.to_q.weight), f32(at.to_q.bias)
        d.attn_k_w16, d.attn_k_b = lin16(at.to_k.weight), f32(at.to_k.bias)
        d.attn_v_w16 = lin16(at.to_v.weight)
        d.attn_o_w16 = lin16(at.to_out[0].weight)
        d.attn_o_b = f32(fold_v_bias(at.to_out[0].weight, at.to_out[0].bias, at.to_v.bias))
        for b, blk in enumerate(dec.up_blocks):
            for r in range(3):
                d.up[b * 3 + r] = resnet(blk.resnets[r])
            if hasattr(blk, "upsamplers"):
                d.ups_w16[b], d.ups_b[b] = conv16(blk.upsamplers[0].conv.weight), f32(blk.upsamplers[0].conv.bias)
        d.norm_out_g, d.norm_out_b = f32(dec.conv_norm_out.weight), f32(dec.conv_norm_out.bias)
        wo = torch.zeros(32, *dec.conv_out.weight.shape[1:], dtype=torch.float32, device=dec.conv_out.weight.device)
        wo[: c.out_channels] = dec.conv_out.weight.detach().float()
        bo = torch.zeros(32, dtype=torch.float32, device=wo.device)
        bo[: c.out_channels] = dec.conv_out.bias.detach().float()
        d.conv_out_w16, d.conv_out_b = conv16(wo), f32(bo)
        d.out_channels = c.out_channels
        self._packed, self._packed_key = (d, keep), key
        return self._packed

    def decode(self, z, return_dict=True, num_frames=None, **kwargs):
        """z (n, latent_channels, h, w) -> DecoderOutput(sample=(n, 3, 8h, 8w)).  `num_frames` is ignored by AutoencoderKL
        and required by AutoencoderKLTemporalDecoder (one clip per call: n == num_frames, as pipeline_latte.py:785-792 does)."""
        if not z.is_cuda:
            raise RuntimeError("latte_b200.AutoencoderKL runs on CUDA (sm_90a) only; there is no CPU fallback")
        lib = _lib.load()
        dev = z.device
        n, cz, h, w = z.shape
        scale = 2 ** (len(self.config.block_out_channels) - 1)
        with torch.cuda.device(dev):
            d, _ = self._pack()
            zf = z.detach().to(torch.float32).contiguous()
            out = torch.empty(n, self.config.out_channels, h * scale, w * scale, dtype=torch.float32, device=dev)
            need = lib.b200_vae_workspace_bytes(C.byref(d), n, h, w)
            if need == 0:
                raise RuntimeError("latte_b200: unsupported VAE configuration: " + _lib.last_error())
            base = self._aligned_workspace(need, dev)
            if self._temporal:
                if num_frames is None:
                    raise ValueError("AutoencoderKLTemporalDecoder.decode needs num_frames")
                rc = lib.b200_vae_decode_temporal(C.byref(d), zf.data_ptr(), n, h, w, int(num_frames), out.data_ptr(), base, need,
                                                  torch.cuda.current_stream(dev).cuda_stream)
            else:
                rc = lib.b200_vae_decode(C.byref(d), zf.data_ptr(), n, h, w, out.data_ptr(), base, need,
                                         torch.cuda.current_stream(dev).cuda_stream)
            _lib.check(rc, "b200_vae_decode")
        pd = self.dtype
        out = out if pd == torch.float32 else out.to(pd)
        return DecoderOutput(sample=out) if return_dict else (out,)


class AutoencoderKLTemporalDecoder(AutoencoderKL):
    """The SVD temporal decoder `sample_t2x.py:31-34` loads for `enable_vae_temporal_decoder` (pipeline_latte.py:779-798):
    every resnet is spatial ResnetBlock2D + temporal Conv3d(3,1,1) resnet blended by a learned alpha; `time_conv_out` last.
    Same kernels as AutoencoderKL; the temporal convolutions are 3-tap implicit GEMMs shifted along the frame index."""
