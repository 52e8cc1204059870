"""Training step of `LatteT2V` (the text-to-video denoiser of Latte-1): the step of `training._EngineBase`, which `Latte` shares,
with LatteT2V's operand table, modulation, caption projection and cross-attention.

Derivatives follow the reference forward (models/latte_t2v.py:677-941 with use_image_num = 0; the spatial block is diffusers'
`BasicTransformerBlock` with ada_norm_single, restated in oracle/t2v_oracle.spatial_block):
  spatial block    x += g1 * attn1(LNmod1(x));  x += attn2(x, caption) (no norm, no gate);  x += g2 * ff(LNmod2(x))
  temporal block   x += g1 * attn1(LNmod1(x));  x += g2 * ff(LNmod2(x))         (temp_pos_embed before the first one, F > 1)
  conditioning     mod of block j = scale_shift_table_j + ts,  ts = adaln_single.linear(silu(emb)),  emb = adaln_single.emb(t)
  output head      LN(x)(1 + table_f[1] + emb) + table_f[0] + emb -> proj_out -> unpatchify
Rows stay in (b, f, n) order for spatial and temporal blocks, as in the sampling path.  The caption is projected once per sample
(`caption_projection`, B*L rows), and the K/V of every layer's attn2 come from ONE GEMM over the stacked [layers*2D, D] weight;
the backward collects every layer's dK/dV in one [B*L, layers*2D] buffer (b200_cross_attention_bwd writes its column window) and
runs one weight gradient and one input gradient over it after the block loop.  Row counts of the caption GEMMs are padded to 64
with zero rows.

Video + image joint training (`images` = I > 0, latte_t2v.py:730-919 in training mode): each sample is F video frames plus I
still images, every image with its own caption, in the row layout of `training._EngineBase`.  Caption rows: the B video
captions, then the B*I image captions in (b, i) order (the stacked K/V, the dK | dV buffer and the key-bias rows follow it).
The modulation rows are one per frame, each table_j + ts[b]; each spatial block issues two cross-attention calls on row views,
the videos (batch B, F*N query rows per caption) and the images (batch B*I, N query rows per caption).  temp_pos_embed is not
added (the reference's plain image-joint branch, :876-891, has no such term).

`emb` (B, D) stays on torch autograd (a handful of kernels); the engine returns its gradient `dc`, which collects the SiLU path
into every block's modulation and the output head's direct use of it.  Backend-agnostic: latte_b200.train_ops.NativeOps on the
GPU, the torch restatement oracle/train_t2v_ops_oracle.T2VTorchOps in the CPU tests.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from .training import _EngineBase, _pad64


class T2VTrainEngine(_EngineBase):
    """One training forward + backward of a `LatteT2V` on `ops` with operand type `dtype`.  text (B, L, caption_channels) fp32;
    key_bias None or (B, 128) fp32 additive score bias per caption token ((1 - mask) * -10000, latte_t2v.py:766-771).  With
    `images` = I > 0 still images per sample, text is (B, 1 + I, L, caption_channels) and key_bias None or (B, 1 + I, 128):
    caption (b, 0) serves the video frames of sample b, caption (b, 1 + i) its image i (latte_t2v.py:756-762, 791-796).
    Inputs and outputs are (B, C, F[+I], H, W)."""

    def __init__(self, model, ops, dtype, text, key_bias=None, checkpoint=False, images=0):
        super().__init__(model, ops, dtype, images, checkpoint)
        m, cfg = model, model.config
        self.D, self.H, self.Fr = m.inner_dim, cfg.num_attention_heads, cfg.video_length
        self.N, self.p, self.nblocks = (cfg.sample_size // cfg.patch_size) ** 2, cfg.patch_size, 2 * cfg.num_layers
        self.patch_conv, self.final_linear, self.pos_table = m.pos_embed.proj, m.proj_out, m.pos_table
        #: scale_shift_table of block j, in block order (spatial and temporal alternate)
        self.tables = [t for pair in zip([b.scale_shift_table for b in m.transformer_blocks],
                                         [b.scale_shift_table for b in m.temporal_transformer_blocks]) for t in pair]
        self.text = self._caption_rows(text)
        self.key_bias = self._caption_rows(key_bias)

    def _operands(self):
        """Per spatial block q|k|v, attn1 out, attn2 q, attn2 out, fc1, fc2; per temporal block q|k|v, out, fc1, fc2; every
        layer's attn2 k|v; adaln_single.linear; caption_projection linear_1, linear_2."""
        m = self.m
        t = []
        for i, b in enumerate(m.transformer_blocks):
            a1 = b.attn1
            t += [((2 * i, "qkv"), [a1.to_q.weight, a1.to_k.weight, a1.to_v.weight], [a1.to_q.bias, a1.to_k.bias, a1.to_v.bias])]
            t += [((2 * i, k), [lin.weight], [lin.bias]) for k, lin in
                  (("out", a1.to_out[0]), ("q2", b.attn2.to_q), ("o2", b.attn2.to_out[0]), ("fc1", b.ff.net[0].proj),
                   ("fc2", b.ff.net[2]))]
        for i, b in enumerate(m.temporal_transformer_blocks):
            a1 = b.attn1
            t += [((2 * i + 1, "qkv"), [a1.to_q.weight, a1.to_k.weight, a1.to_v.weight], [a1.to_q.bias, a1.to_k.bias, a1.to_v.bias])]
            t += [((2 * i + 1, k), [lin.weight], [lin.bias]) for k, lin in
                  (("out", a1.to_out[0]), ("fc1", b.ff.net[0].proj), ("fc2", b.ff.net[2]))]
        kv = [lin for b in m.transformer_blocks for lin in (b.attn2.to_k, b.attn2.to_v)]
        t.append(("kv", [lin.weight for lin in kv], [lin.bias for lin in kv]))
        for k, lin in (("ada", m.adaln_single.linear), ("cap1", m.caption_projection.linear_1),
                       ("cap2", m.caption_projection.linear_2)):
            t.append((k, [lin.weight], [lin.bias]))
        return t

    def _extra_params(self):
        return self.tables + [self.m.scale_shift_table]

    # ---------------------------------------------------------------------------------------------------------------
    def _caption_rows(self, t):
        """(B, 1 + I, ...) per-sample captions -> (B*(1 + I), ...): the B video captions, then the B*I image captions."""
        if t is None or not self.images:
            return t
        return torch.cat((t[:, 0], t[:, 1:].flatten(0, 1))).contiguous()

    def _frame_rows(self, t, B):
        """Per-sample rows (B, n) -> one row per frame in row order (the video frames, then the images); as is without images."""
        if not self.images:
            return t
        return torch.cat((t.repeat_interleave(self.Fr, dim=0), t.repeat_interleave(self.images, dim=0)))

    def _sample_sum(self, t, B):
        """Adjoint of `_frame_rows`: the rows of each sample's frames summed into one row per sample."""
        if not self.images:
            return t
        Fr = self.Fr
        return t[:B * Fr].reshape(B, Fr, -1).sum(1) + t[B * Fr:].reshape(B, self.images, -1).sum(1)

    def _cross_calls(self, B):
        """One (query rows, batch, query rows per caption, caption rows) per cross-attention call: the videos, then the images."""
        L, Tv = self.text.shape[1], B * self.Fr * self.N
        calls = [(slice(0, Tv), B, self.Fr * self.N, slice(0, B * L))]
        if self.images:
            calls.append((slice(Tv, None), B * self.images, self.N, slice(B * L, None)))
        return calls

    def _key_bias(self, nb, rows):
        """key_bias rows of one cross-attention call (row b*L of the caption buffer <-> key_bias row b)."""
        if self.key_bias is None:
            return None
        L = self.text.shape[1]
        return self.key_bias[rows.start // L:rows.start // L + nb]

    # ---------------------------------------------------------------------------------------------------------------
    def forward(self, x, c, save=True):
        """x (B, C, F[+I], H, W) fp32, c = emb (B, D) fp32 -> (B, out_channels, F[+I], H, W) fp32: a transposed view without
        images, contiguous with them (the layouts LatteT2V's training call returns)."""
        out = super().forward(x.transpose(1, 2), c, save).transpose(1, 2)
        return out.contiguous() if self.images else out

    def backward(self, dout):
        """dout (B, out_channels, F[+I], H, W) -> ({parameter name: fp32 gradient}, dc (B, D) fp32)."""
        return super().backward(dout.transpose(1, 2))

    def _modulation(self, ts, c, B):
        """Block j's six rows = table_j + ts, output head = table_f + emb (one row per sample, or per frame with images: the
        conditioning stays per sample, latte_t2v.py:801, :919)."""
        D = self.D
        tables = torch.cat([t.detach().float().reshape(-1) for t in self.tables]).reshape(1, self.nblocks * 6 * D)
        final_table = self.m.scale_shift_table.detach().float().reshape(1, 2 * D)
        return torch.cat((tables + self._frame_rows(ts, B).repeat(1, self.nblocks),
                          final_table + self._frame_rows(c.float(), B).repeat(1, 2)), dim=1).contiguous()

    def _modulation_backward(self, dmod, S, grads):
        """-> (d ts, the output head's direct terms of dc); puts the tables' gradients into grads."""
        D, B = self.D, S["B"]
        base = self.nblocks * 6 * D
        name = self.names
        dtab = dmod[:, :base].sum(0)
        for j, t in enumerate(self.tables):
            grads[name[id(t)]] = dtab[j * 6 * D:(j + 1) * 6 * D].reshape(6, D)
        dfin = self._sample_sum(dmod[:, base:], B)
        grads[name[id(self.m.scale_shift_table)]] = dfin.sum(0).reshape(2, D)
        dts = self._sample_sum(dmod[:, :base], B).reshape(B, self.nblocks, 6 * D).sum(1).contiguous()
        return dts, (dfin[:, :D], dfin[:, D:])

    def _temp_embed(self):
        """temp_pos_embed joins after the first spatial block, before the first temporal one (latte_t2v.py:894-895); the
        image-joint branch adds none (:876-891)."""
        if self.Fr == 1 or self.images:
            return None
        return self.m.temp_pos_embed.detach().float().reshape(-1, self.D)[:self.Fr].contiguous()

    def _context_forward(self, S, save):
        """The caption projection (B*L rows, padded to 64) and every layer's K/V in one GEMM."""
        ops, W = self.ops, self.w
        R = self.text.shape[0] * self.text.shape[1]
        tp = torch.zeros(_pad64(R), self.text.shape[2], dtype=torch.float32, device=self.text.device)
        tp[:R] = self.text.reshape(R, -1).float()
        text16 = ops.to_operand(tp)
        del tp
        cu, ca = ops.linear_gelu_both(text16, *W["cap1"])
        txt = ops.linear(ca, *W["cap2"])
        S["kv"] = ops.linear(txt, *W["kv"])                                                # (Rp, layers*2D)
        if save:
            S.update(text16=text16, cu=cu, ca=ca, txt=txt)

    def _cross_forward(self, j, xm, S):
        """x += to_out(attn2(to_q(x), caption K/V)), one call per caption group."""
        ops, W, D = self.ops, self.w, self.D
        xa = ops.to_operand(xm)
        q2 = ops.linear(xa, *W[j, "q2"])
        kvl = S["kv"][:, j * D:(j + 2) * D]                 # layer j // 2's [k | v] columns
        o2 = [ops.cross_attention(q2[qr], kvl[cr], nb, rows, self.text.shape[1], self.H, self._key_bias(nb, cr))
              for qr, nb, rows, cr in self._cross_calls(S["B"])]
        o2 = o2[0] if len(o2) == 1 else torch.cat(o2)
        ops.linear_accum(xm, o2, *W[j, "o2"])
        return xa, q2, o2

    def _begin_backward(self, S, dev):
        S["dkv"] = torch.zeros(S["kv"].shape[0], self.nblocks * self.D, dtype=self.dtype, device=dev)   # every layer's [dK | dV]
        S["unit"] = torch.ones(1, self.D, dtype=torch.float32, device=dev)                             # the ungated residual's gate

    def _cross_backward(self, j, cross, dx, S, G, bgrad):
        """Backward of x_mid = x_attn + to_out(attn2(to_q(x_attn))): writes the layer's caption dK | dV into S["dkv"] and
        returns the gradient of x_attn."""
        ops, W, D = self.ops, self.w, self.D
        xa, q2, o2 = cross
        ops.colsum(dx, bgrad[j, "o2"])
        dx16 = ops.to_operand(dx)
        G[j, "o2"] = self._wgrad(dx16, o2)
        do2 = ops.dgrad(dx16, W[j, "o2"][0])
        del dx16
        kvl = S["kv"][:, j * D:(j + 2) * D]
        dq2 = [ops.cross_attention_bwd(q2[qr], kvl[cr], o2[qr], do2[qr], nb, rows, self.text.shape[1], self.H,
                                       self._key_bias(nb, cr), S["dkv"][cr], j * D) for qr, nb, rows, cr in self._cross_calls(S["B"])]
        dq2 = dq2[0] if len(dq2) == 1 else torch.cat(dq2)
        del do2, o2
        ops.colsum(dq2, bgrad[j, "q2"])
        G[j, "q2"] = self._wgrad(dq2, xa)
        return ops.gate_residual(dx, ops.dgrad(dq2, W[j, "q2"][0]), S["unit"], dx.shape[0])

    def _context_backward(self, S, G, bgrad):
        """Every layer's K/V projection, then the caption projection (linear_1 -> GELU(tanh) -> linear_2)."""
        ops, W = self.ops, self.w
        dkv = S.pop("dkv")
        ops.colsum(dkv, bgrad["kv"])
        G["kv"] = self._wgrad(dkv, S["txt"])
        dtxt = ops.dgrad(dkv, W["kv"][0])
        del dkv
        ops.colsum(dtxt, bgrad["cap2"])
        G["cap2"] = self._wgrad(dtxt, S["ca"])
        dcu = ops.gelu_bwd(ops.dgrad(dtxt, W["cap2"][0]), S["cu"], bgrad["cap1"])
        G["cap1"] = self._wgrad(dcu, S["text16"])


def trainable_names(model):
    """Every parameter except adaln_single.emb (the timestep embedder, whose (B, D) graph stays on torch autograd and gets its
    gradient from `dc`), in named_parameters order."""
    return T2VTrainEngine(model, None, None, None).trainable_names()


def conditioning(model, t):
    """emb = adaln_single.emb(t): Timesteps(256, flip_sin_to_cos, shift 0) -> linear_1 -> SiLU -> linear_2 (latte_t2v.py:
    782-784, AdaLayerNormSingle :398-428), on torch autograd."""
    te = model.adaln_single.emb.timestep_embedder
    half = 128
    freqs = torch.exp(-math.log(10000) * torch.arange(0, half, dtype=torch.float32, device=t.device) / half)
    args = t[:, None].float() * freqs[None]
    e = torch.cat([torch.cos(args), torch.sin(args)], dim=-1)
    return te.linear_2(F.silu(te.linear_1(e.to(te.linear_1.weight.dtype)))).float()


def train_forward(model, ops, dtype, x, c, text, key_bias=None, images=0):
    """Forward of one training step with the backward attached; c = `conditioning(model, t)`.  With `images` still images per
    sample, x is (B, C, F + images, H, W) and text / key_bias carry 1 + images captions per sample (see T2VTrainEngine).
    Checkpoints each block when `model.gradient_checkpointing` is set."""
    eng = T2VTrainEngine(model, ops, dtype, text, key_bias, checkpoint=model.gradient_checkpointing, images=images)
    return eng.train_forward(x, c)
