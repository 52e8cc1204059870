"""Training step of `LatteT2V` (the text-to-video denoiser of Latte-1): forward that keeps its activations + the backward written
out op by op, behind one autograd node, like `training.TrainEngine` for `Latte`.

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
still images, every image with its own caption.  Row order as in `training.TrainEngine`: the B*F*N video rows first, (b, f, n),
then the B*I*N image rows, (b, i, n).  Caption rows: the B video captions, then the B*I image captions in (b, i) order (the
stacked K/V, the dK | dV buffer and the key-bias rows follow it).  Spatial blocks and the output head run over every row with
one modulation row per frame (rows_per_batch = N, each row table_j + ts[b]); each spatial block issues two cross-attention calls
on row views, the videos (batch B, F*N query rows per caption) and the images (batch B*I, N query rows per caption).  Temporal
blocks run on the video prefix x[:B*F*N], exactly a batch of B videos, through a strided view with one modulation row per
video, and carry the image rows through unchanged.  temp_pos_embed is not added (the reference's plain image-joint branch,
:876-891, has no such term).

`emb` (B, D) stays on torch autograd (a handful of kernels); the engine returns its gradient `dc`, which collects the SiLU path
into every block's modulation and the output head's direct use of it.  Backend-agnostic: latte_b200.train_ops.NativeOps on the
GPU, the torch restatement oracle/train_t2v_ops_oracle.T2VTorchOps in the CPU tests.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from .training import _LatteTrainFn, _patch_rows


def _pad64(n):
    return (n + 63) // 64 * 64


class T2VTrainEngine:
    """One training forward + backward of a `LatteT2V` on `ops` with operand type `dtype`.  text (B, L, caption_channels) fp32;
    key_bias None or (B, 128) fp32 additive score bias per caption token ((1 - mask) * -10000, latte_t2v.py:766-771).  With
    `images` = I > 0 still images per sample, text is (B, 1 + I, L, caption_channels) and key_bias None or (B, 1 + I, 128):
    caption (b, 0) serves the video frames of sample b, caption (b, 1 + i) its image i (latte_t2v.py:756-762, 791-796)."""

    def __init__(self, model, ops, dtype, text, key_bias=None, checkpoint=False, images=0):
        self.m = model
        self.ops = ops
        self.dtype = dtype
        self.images = images
        self.text = self._caption_rows(text)
        self.key_bias = self._caption_rows(key_bias)
        #: gradient checkpointing: the forward keeps each block's input only and the backward reruns the block before its backward
        self.checkpoint = checkpoint
        self.saved = None
        self.w = None

    # ---------------------------------------------------------------------------------------------------------------
    def _weight_groups(self):
        """(cache key, [source parameters stacked by rows]) of every GEMM operand."""
        m = self.m
        g = []
        for i, b in enumerate(m.transformer_blocks):
            g += [(f"s{i}.qkv", [b.attn1.to_q.weight, b.attn1.to_k.weight, b.attn1.to_v.weight]),
                  (f"s{i}.out", [b.attn1.to_out[0].weight]), (f"s{i}.q2", [b.attn2.to_q.weight]),
                  (f"s{i}.o2", [b.attn2.to_out[0].weight]),
                  (f"s{i}.fc1", [b.ff.net[0].proj.weight]), (f"s{i}.fc2", [b.ff.net[2].weight])]
        for i, b in enumerate(m.temporal_transformer_blocks):
            g += [(f"t{i}.qkv", [b.attn1.to_q.weight, b.attn1.to_k.weight, b.attn1.to_v.weight]),
                  (f"t{i}.out", [b.attn1.to_out[0].weight]),
                  (f"t{i}.fc1", [b.ff.net[0].proj.weight]), (f"t{i}.fc2", [b.ff.net[2].weight])]
        g.append(("kv", [w for b in m.transformer_blocks for w in (b.attn2.to_k.weight, b.attn2.to_v.weight)]))
        g += [("ada", [m.adaln_single.linear.weight]), ("cap1", [m.caption_projection.linear_1.weight]),
              ("cap2", [m.caption_projection.linear_2.weight])]
        return g

    def _bias_groups(self):
        m = self.m
        g = {}
        for i, b in enumerate(m.transformer_blocks):
            g[f"s{i}.qkv"] = [b.attn1.to_q.bias, b.attn1.to_k.bias, b.attn1.to_v.bias]
            g[f"s{i}.out"], g[f"s{i}.q2"], g[f"s{i}.o2"] = [b.attn1.to_out[0].bias], [b.attn2.to_q.bias], [b.attn2.to_out[0].bias]
            g[f"s{i}.fc1"], g[f"s{i}.fc2"] = [b.ff.net[0].proj.bias], [b.ff.net[2].bias]
        for i, b in enumerate(m.temporal_transformer_blocks):
            g[f"t{i}.qkv"] = [b.attn1.to_q.bias, b.attn1.to_k.bias, b.attn1.to_v.bias]
            g[f"t{i}.out"], g[f"t{i}.fc1"], g[f"t{i}.fc2"] = [b.attn1.to_out[0].bias], [b.ff.net[0].proj.bias], [b.ff.net[2].bias]
        g["kv"] = [t for b in m.transformer_blocks for t in (b.attn2.to_k.bias, b.attn2.to_v.bias)]
        g["ada"], g["cap1"], g["cap2"] = [m.adaln_single.linear.bias], [m.caption_projection.linear_1.bias], [m.caption_projection.linear_2.bias]
        return g

    def prepare(self):
        """Operand copies of the parameters in the compute type, refreshed by one multi-tensor cast per step into buffers that
        persist on the model (`model._train_operands`), as `TrainEngine.prepare` does.  Stacked operands (q|k|v, every layer's
        k|v) are one buffer whose row slices are the parameters' copies.  Patch embedding / proj_out are zero-padded to the
        GEMM's 64-element k-block."""
        m, ops = self.m, self.ops
        D = m.inner_dim
        dev = m.proj_out.weight.device
        groups = self._weight_groups()
        cache = getattr(m, "_train_operands", None)
        key = (self.dtype, dev, type(ops).__name__)
        if cache is None or cache["key"] != key:
            cache = {"key": key, "w": {}}
            for name, ps in groups:
                cache["w"][name] = torch.empty(sum(p.shape[0] for p in ps), ps[0].shape[1], dtype=self.dtype, device=dev)
            m._train_operands = cache
        srcs, dsts = [], []
        for name, ps in groups:
            row = 0
            for p in ps:
                srcs.append(p.detach())
                dsts.append(cache["w"][name][row:row + p.shape[0]])
                row += p.shape[0]
        if all(t.dtype == torch.float32 and t.is_contiguous() for t in srcs):
            ops.cast_into(srcs, dsts)
        else:
            for a, b in zip(srcs, dsts):
                b.copy_(a)
        W = {}
        for name, bs in self._bias_groups().items():
            W[name] = (cache["w"][name], torch.cat([b.detach().float() for b in bs]).contiguous())
        pw = m.pos_embed.proj.weight.detach().reshape(D, -1).float()
        self.kp = pw.shape[1]
        pad = torch.zeros(D, 64, dtype=torch.float32, device=dev)
        pad[:, : self.kp] = pw
        W["patch"] = (ops.cast(pad), m.pos_embed.proj.bias.detach().float().contiguous())
        fw = m.proj_out.weight.detach().float()
        self.nf = fw.shape[0]
        padk = torch.zeros(64, D, dtype=torch.float32, device=dev)
        padk[: self.nf] = fw
        W["final_wk"] = ops.cast(padk)
        W["final"] = (W["final_wk"][: self.nf], m.proj_out.bias.detach().float().contiguous())
        NB = 2 * m.config.num_layers
        tabs = [t for pair in zip([b.scale_shift_table for b in m.transformer_blocks],
                                  [b.scale_shift_table for b in m.temporal_transformer_blocks]) for t in pair]
        W["tables"] = torch.cat([t.detach().float().reshape(-1) for t in tabs]).reshape(1, NB * 6 * D)
        W["final_table"] = m.scale_shift_table.detach().float().reshape(1, 2 * D)
        self.w = W

    # ---------------------------------------------------------------------------------------------------------------
    def _geometry(self):
        c = self.m.config
        g = c.sample_size // c.patch_size
        return c.video_length, g * g, g

    def _rows(self, B):
        """(rows of all frames, rows of the video frames, rows_per_batch of spatial blocks / output head, of temporal blocks)."""
        Fr, N, _ = self._geometry()
        Tv = B * Fr * N
        if not self.images:
            return Tv, Tv, Fr * N, Fr * N
        return Tv + B * self.images * N, Tv, N, Fr * N

    def _caption_rows(self, t):
        """(B, 1 + I, ...) per-sample captions -> (B*(1 + I), ...): the B video captions, then the B*I image captions."""
        if t is None or not self.images:
            return t
        return torch.cat((t[:, 0], t[:, 1:].flatten(0, 1))).contiguous()

    def _frame_rows(self, t, B):
        """Per-sample rows (B, n) -> one row per frame in row order (the video frames, then the images); as is without images."""
        if not self.images:
            return t
        Fr = self._geometry()[0]
        return torch.cat((t.repeat_interleave(Fr, dim=0), t.repeat_interleave(self.images, dim=0)))

    def _sample_sum(self, t, B):
        """Adjoint of `_frame_rows`: the rows of each sample's frames summed into one row per sample."""
        if not self.images:
            return t
        Fr = self._geometry()[0]
        return t[:B * Fr].reshape(B, Fr, -1).sum(1) + t[B * Fr:].reshape(B, self.images, -1).sum(1)

    def _temporal_rows(self, t, B):
        """The modulation rows (of mod / dmod) a temporal block addresses: per sample without images, else the first frame's row
        of each video (a strided view)."""
        Fr = self._geometry()[0]
        return t[0:B * Fr:Fr] if self.images else t

    def _cross_calls(self, B):
        """One (query rows, batch, query rows per caption, caption rows) per cross-attention call: the videos, then the images."""
        Fr, N, _ = self._geometry()
        L, Tv = self.text.shape[1], B * Fr * N
        calls = [(slice(0, Tv), B, Fr * N, slice(0, B * L))]
        if self.images:
            calls.append((slice(Tv, None), B * self.images, N, slice(B * L, None)))
        return calls

    def _key_bias(self, nb, rows):
        """key_bias rows of one cross-attention call (row b*L of the caption buffer <-> key_bias row b)."""
        if self.key_bias is None:
            return None
        L = self.text.shape[1]
        return self.key_bias[rows.start // L:rows.start // L + nb]

    def _unit(self, n, dev):
        return torch.ones(1, n, dtype=torch.float32, device=dev)

    def _block_forward(self, j, xs, mod, kv, B, temp, rerun=False):
        """Block j (spatial for even j, temporal for odd j) on its input xs (T x D fp32) -> (its output, the list of
        activations its backward reads); kv = every layer's caption K/V.  rerun=True is the checkpointed backward's
        recomputation: it stops before the last residual update, whose output the backward does not read, and returns None
        in its place."""
        m, ops, W = self.m, self.ops, self.w
        D, H = m.inner_dim, m.config.num_attention_heads
        Fr, N, _ = self._geometry()
        _, Tv, rpb, rpb_t = self._rows(B)
        L = self.text.shape[1]
        i, temporal = j // 2, bool(j % 2)
        mv = (self._temporal_rows(mod, B) if temporal else mod)[:, j * 6 * D:(j + 1) * 6 * D]
        sh1, sc1, g1, sh2, sc2, g2 = (mv[:, k * D:(k + 1) * D] for k in range(6))
        p = f"{'t' if temporal else 's'}{i}."
        rp = rpb_t if temporal else rpb
        xi = xs[:Tv] if temporal else xs    # temporal blocks see the video rows only (latte_t2v.py:876-891)
        h1 = ops.ln_modulate(xi, sh1, sc1, rp)
        qkv = ops.linear(h1, *W[p + "qkv"])
        o = ops.attention(qkv, B, Fr if temporal else Fr + self.images, N, H, temporal)
        m1 = ops.linear(o, *W[p + "out"])
        xm = ops.gate_residual(xi, m1, g1, rp)
        cross = None
        if not temporal:                # x += to_out(attn2(to_q(x), caption K/V)), one call per caption group
            xa = ops.to_operand(xm)
            q2 = ops.linear(xa, *W[p + "q2"])
            kvl = kv[:, i * 2 * D:(i + 1) * 2 * D]
            o2 = [ops.cross_attention(q2[qr], kvl[cr], nb, rows, L, H, self._key_bias(nb, cr))
                  for qr, nb, rows, cr in self._cross_calls(B)]
            o2 = o2[0] if len(o2) == 1 else torch.cat(o2)
            ops.linear_accum(xm, o2, *W[p + "o2"])
            cross = (xa, q2, o2)
        h2 = ops.ln_modulate(xm, sh2, sc2, rp)
        u, a = ops.linear_gelu_both(h2, *W[p + "fc1"])
        m2 = ops.linear(a, *W[p + "fc2"])
        acts = [xi, h1, qkv, o, m1, cross, xm, h2, u, a, m2]
        if rerun:
            return None, acts
        # temp_pos_embed joins after the first spatial block, before the first temporal one (latte_t2v.py:894-895); the
        # image-joint branch adds none (:876-891)
        add = temp if (j == 0 and Fr > 1 and not self.images) else None
        xo = ops.gate_residual(xm, m2, g2, rp, row_add=add, tokens=N)
        if temporal and self.images:        # image rows pass through the temporal block unchanged
            xo = torch.cat((xo, xs[Tv:]))
        return xo, acts

    def _block_backward(self, j, acts, dx, mod, dmod, dkv, kv, unit, B, G):
        """Backward of block j from the list `_block_forward` returned, which it empties so that each buffer is freed as soon
        as it is used.  Accumulates into dx (T x D fp32) and dmod, writes the layer's caption dK | dV into dkv and puts the
        block's weight and bias gradients into G.  Returns dx, which the ungated cross-attention replaces (unit: its gate of
        ones)."""
        m, ops, W = self.m, self.ops, self.w
        D, H = m.inner_dim, m.config.num_attention_heads
        Fr, N, _ = self._geometry()
        T, Tv, rpb, rpb_t = self._rows(B)
        L = self.text.shape[1]
        xs, h1, qkv, o, m1, cross, xm, h2, u, a, m2 = acts
        acts.clear()
        i, temporal = j // 2, bool(j % 2)
        mv = (self._temporal_rows(mod, B) if temporal else mod)[:, j * 6 * D:(j + 1) * 6 * D]
        sh1, sc1, g1, sh2, sc2, g2 = (mv[:, k * D:(k + 1) * D] for k in range(6))
        dv = (self._temporal_rows(dmod, B) if temporal else dmod)[:, j * 6 * D:(j + 1) * 6 * D]
        dsh1, dsc1, dg1, dsh2, dsc2, dg2 = (dv[:, k * D:(k + 1) * D] for k in range(6))
        p = f"{'t' if temporal else 's'}{i}."
        rp = rpb_t if temporal else rpb
        dxb = dx[:Tv] if temporal else dx   # a temporal block passes the image rows' gradient through untouched
        wgrad, bgrad = self._wgrad, self._bgrad
        db = {n: bgrad(p + n, dx.device) for n in ("qkv", "out", "fc1", "fc2")}
        # x_out = x_mid + g2 * fc2(gelu(fc1(LNmod2(x_mid))))
        dm2 = ops.gate_bwd(dxb, m2, g2, rp, dg2, db["fc2"])
        G[p + "fc2"] = wgrad(dm2, a)
        du = ops.gelu_bwd(ops.dgrad(dm2, W[p + "fc2"][0]), u, db["fc1"])
        del dm2, a
        G[p + "fc1"] = wgrad(du, h2)
        dh2 = ops.dgrad(du, W[p + "fc1"][0])
        del du
        ops.ln_modulate_bwd(dh2, xm, sh2, sc2, rp, dxb, dsh2, dsc2)
        del dh2
        if cross is not None:           # x_mid = x_attn + to_out(attn2(to_q(x_attn)))
            xa, q2, o2 = cross
            db["q2"], db["o2"] = bgrad(p + "q2", dx.device), bgrad(p + "o2", dx.device)
            ops.colsum(dx, db["o2"])
            dx16 = ops.to_operand(dx)
            G[p + "o2"] = wgrad(dx16, o2)
            do2 = ops.dgrad(dx16, W[p + "o2"][0])
            del dx16
            kvl = kv[:, i * 2 * D:(i + 1) * 2 * D]
            dq2 = [ops.cross_attention_bwd(q2[qr], kvl[cr], o2[qr], do2[qr], nb, rows, L, H, self._key_bias(nb, cr), dkv[cr],
                                           i * 2 * D) for qr, nb, rows, cr in self._cross_calls(B)]
            dq2 = dq2[0] if len(dq2) == 1 else torch.cat(dq2)
            del do2, o2
            ops.colsum(dq2, db["q2"])
            G[p + "q2"] = wgrad(dq2, xa)
            dx = dxb = ops.gate_residual(dx, ops.dgrad(dq2, W[p + "q2"][0]), unit, T)
            del dq2, xa, q2
        # x_attn = x_in + g1 * out(attn1(qkv(LNmod1(x_in))))
        dm1 = ops.gate_bwd(dxb, m1, g1, rp, dg1, db["out"])
        G[p + "out"] = wgrad(dm1, o)
        do = ops.dgrad(dm1, W[p + "out"][0])
        del dm1
        dqkv = ops.attention_bwd(qkv, o, do, B, Fr if temporal else Fr + self.images, N, H, temporal)
        del do
        ops.colsum(dqkv, db["qkv"])
        G[p + "qkv"] = wgrad(dqkv, h1)
        dh1 = ops.dgrad(dqkv, W[p + "qkv"][0])
        del dqkv
        ops.ln_modulate_bwd(dh1, xs, sh1, sc1, rp, dxb, dsh1, dsc1)
        for n, t in db.items():
            G[p + n + ".bias"] = t
        return dx

    def _wgrad(self, dy, x):
        return self.ops.wgrad(torch.zeros(dy.shape[1], x.shape[1], dtype=torch.float32, device=dy.device), dy, x)

    def _bgrad(self, name, dev):
        return torch.zeros(self.w[name][1].shape[0], dtype=torch.float32, device=dev)

    def forward(self, x, c, save=True):
        """x (B, C, F[+I], H, W) fp32, c = emb (B, D) fp32 -> (B, out_channels, F[+I], H, W) fp32."""
        if self.w is None:
            self.prepare()
        m, ops, W = self.m, self.ops, self.w
        cfg = m.config
        B = x.shape[0]
        D, nl = m.inner_dim, cfg.num_layers
        Fr, N, _ = self._geometry()
        T, _, rpb, _ = self._rows(B)
        L = self.text.shape[1]
        R = self.text.shape[0] * L
        Rp = _pad64(R)
        dev = x.device
        # ---- conditioning: ts = adaln_single.linear(silu(emb)); block j's six rows = table_j + ts; output head = table_f + emb
        # (one row per sample, or per frame with images: the conditioning stays per sample, latte_t2v.py:801, :919)
        sc = ops.to_operand(F.silu(c.float()).contiguous())
        ts = ops.linear(sc, *W["ada"]).float()                                             # (B, 6D)
        NB = 2 * nl
        mod = torch.cat((W["tables"] + self._frame_rows(ts, B).repeat(1, NB),
                         W["final_table"] + self._frame_rows(c.float(), B).repeat(1, 2)), dim=1).contiguous()
        S = {"B": B, "c": c, "sc": sc, "mod": mod, "blocks": []}
        # ---- caption projection (B*L rows, padded to 64) and every layer's K/V in one GEMM
        tp = torch.zeros(Rp, self.text.shape[2], dtype=torch.float32, device=dev)
        tp[:R] = self.text.reshape(R, -1).float()
        text16 = ops.to_operand(tp)
        del tp
        cu, ca = ops.linear_gelu_both(text16, *W["cap1"])
        txt = ops.linear(ca, *W["cap2"])
        kv = ops.linear(txt, *W["kv"])                                                     # (Rp, layers*2D)
        if save:
            S.update(text16=text16, cu=cu, ca=ca, txt=txt, kv=kv)
        # ---- patch embedding + the frozen sin-cos table
        xp = torch.zeros(T, 64, dtype=torch.float32, device=dev)
        xf = x.float().permute(0, 2, 1, 3, 4)
        if self.images:
            xp[:, : self.kp] = torch.cat((_patch_rows(xf[:, :Fr], cfg.patch_size), _patch_rows(xf[:, Fr:], cfg.patch_size)))
        else:
            xp[:, : self.kp] = _patch_rows(xf, cfg.patch_size)
        del xf
        xp = ops.to_operand(xp)
        xs = m.pos_table.detach().float().reshape(1, N, D).expand(B * (Fr + self.images), N, D).reshape(T, D).contiguous()
        ops.linear_accum(xs, xp, *W["patch"])
        if save:
            S["xp"] = xp
        del xp
        temp = m.temp_pos_embed.detach().float().reshape(-1, D)[:Fr].contiguous()
        for j in range(NB):
            xo, acts = self._block_forward(j, xs, mod, kv, B, temp)
            if save:
                S["blocks"].append(xs if self.checkpoint else acts)
            del acts                        # a checkpointed block's activations are freed before the next block runs
            xs = xo
        base = NB * 6 * D
        hf = ops.ln_modulate(xs, mod[:, base:base + D], mod[:, base + D:base + 2 * D], rpb)
        tok = torch.zeros(T, self.nf, dtype=torch.float32, device=dev)
        ops.linear_accum(tok, hf, *W["final"])
        S["x_last"], S["hf"] = xs, hf
        self.saved = S if save else None
        return self._unpatchify(tok, B)

    def _unpatchify(self, tok, B):
        """rows (b, f, h, w) x (p, q, c) -> (B, c, F, h*p, w*q) (latte_t2v.py:929-936); image rows follow as frames F.."""
        cfg = self.m.config
        Fr, N, g = self._geometry()
        p, c = cfg.patch_size, cfg.out_channels

        def unp(rows, frames):
            t = rows.view(B * frames, g, g, p, p, c).permute(0, 5, 1, 3, 2, 4).reshape(B, frames, c, g * p, g * p)
            return t.permute(0, 2, 1, 3, 4)
        if self.images:
            Tv = B * Fr * N
            return torch.cat((unp(tok[:Tv], Fr), unp(tok[Tv:], self.images)), dim=2)
        return unp(tok, Fr)

    def _patchify_out(self, dout):
        cfg = self.m.config
        Fr, _, g = self._geometry()
        p, c = cfg.patch_size, cfg.out_channels

        def pat(d):
            B, frames = d.shape[0], d.shape[2]
            t = d.permute(0, 2, 1, 3, 4).reshape(B * frames, c, g, p, g, p).permute(0, 2, 4, 3, 5, 1)
            return t.reshape(B * frames * g * g, p * p * c)
        if self.images:
            return torch.cat((pat(dout[:, :, :Fr]), pat(dout[:, :, Fr:])))
        return pat(dout).contiguous()

    # ---------------------------------------------------------------------------------------------------------------
    def backward(self, dout):
        """dout (B, c, F[+I], H, W) -> ({parameter name: fp32 gradient}, dc (B, D) fp32).  Frees the saved activations."""
        m, ops, W, S = self.m, self.ops, self.w, self.saved
        self.saved = None
        cfg = m.config
        B = S["B"]
        D, nl = m.inner_dim, cfg.num_layers
        NB = 2 * nl
        T, _, rpb, _ = self._rows(B)
        Rp = S["kv"].shape[0]
        dev = dout.device
        mod = S["mod"]
        dmod = torch.zeros_like(mod)
        unit = self._unit(D, dev)
        G = {}
        wgrad = self._wgrad

        def bgrad(name):
            return self._bgrad(name, dev)

        # ---- output head
        dtok = self._patchify_out(dout.float())
        G["proj_out.bias"] = ops.colsum(dtok, torch.zeros(self.nf, dtype=torch.float32, device=dev))
        G["proj_out.weight"] = wgrad(ops.to_operand(dtok), S["hf"])
        dtp = torch.zeros(T, 64, dtype=torch.float32, device=dev)
        dtp[:, : self.nf] = dtok
        dhf = ops.dgrad(ops.to_operand(dtp), W["final_wk"])
        dx = torch.zeros(T, D, dtype=torch.float32, device=dev)
        base = NB * 6 * D
        ops.ln_modulate_bwd(dhf, S["x_last"], mod[:, base:base + D], mod[:, base + D:base + 2 * D], rpb, dx,
                            dmod[:, base:base + D], dmod[:, base + D:base + 2 * D])
        del dhf, dtp, dtok

        dkv = torch.zeros(Rp, nl * 2 * D, dtype=self.dtype, device=dev)   # every layer's [dK | dV]; padding rows stay zero
        # blocks, last to first; a checkpointed block first reruns its forward from its saved input
        for j in reversed(range(NB)):
            acts = S["blocks"].pop()
            if self.checkpoint:
                acts = self._block_forward(j, acts, mod, S["kv"], B, None, rerun=True)[1]
            dx = self._block_backward(j, acts, dx, mod, dmod, dkv, S["kv"], unit, B, G)

        # ---- patch embedding (pos_table / temp_pos_embed are frozen buffers)
        G["patch.bias"] = ops.colsum(dx, torch.zeros(D, dtype=torch.float32, device=dev))
        G["patch"] = wgrad(ops.to_operand(dx), S["xp"])[:, : self.kp]
        del dx

        # ---- every layer's K/V projection, then the caption projection (linear_1 -> GELU(tanh) -> linear_2)
        G["kv.bias"] = ops.colsum(dkv, bgrad("kv"))
        G["kv"] = wgrad(dkv, S["txt"])
        dtxt = ops.dgrad(dkv, W["kv"][0])
        del dkv
        G["cap2.bias"] = ops.colsum(dtxt, bgrad("cap2"))
        G["cap2"] = wgrad(dtxt, S["ca"])
        G["cap1.bias"] = bgrad("cap1")
        dcu = ops.gelu_bwd(ops.dgrad(dtxt, W["cap2"][0]), S["cu"], G["cap1.bias"])
        G["cap1"] = wgrad(dcu, S["text16"])
        del dtxt, dcu

        # ---- conditioning: block tables, ts = linear(silu(emb)), output head's direct use of emb
        dtab = dmod[:, :base].sum(0)
        dts = self._sample_sum(dmod[:, :base], B).reshape(B, NB, 6 * D).sum(1).contiguous()
        G["ada"] = ops.ada_outer(dts, S["sc"])
        G["ada.bias"] = dts.sum(0)
        dsc = ops.ada_dsc(dts, W["ada"][0])
        c = S["c"].float()
        sg = torch.sigmoid(c)
        dfin = self._sample_sum(dmod[:, base:], B)
        dc = dsc * (sg * (1 + c * (1 - sg))) + dfin[:, :D] + dfin[:, D:]
        return self._named(G, dtab, dfin.sum(0)), dc

    def _named(self, G, dtab, dfin_tab):
        """Engine gradient keys -> parameter names (stacked operands split back by rows)."""
        m = self.m
        D = m.inner_dim
        out = {"pos_embed.proj.weight": G["patch"].reshape(m.pos_embed.proj.weight.shape).contiguous(),
               "pos_embed.proj.bias": G["patch.bias"], "proj_out.weight": G["proj_out.weight"], "proj_out.bias": G["proj_out.bias"],
               "scale_shift_table": dfin_tab.reshape(2, D), "adaln_single.linear.weight": G["ada"],
               "adaln_single.linear.bias": G["ada.bias"]}
        for n, mod in (("cap1", "caption_projection.linear_1"), ("cap2", "caption_projection.linear_2")):
            out[mod + ".weight"], out[mod + ".bias"] = G[n], G[n + ".bias"]
        for kind, blocks in (("s", "transformer_blocks"), ("t", "temporal_transformer_blocks")):
            for i in range(m.config.num_layers):
                p, q = f"{kind}{i}.", f"{blocks}.{i}."
                j = 2 * i + (kind == "t")
                out[q + "scale_shift_table"] = dtab[j * 6 * D:(j + 1) * 6 * D].reshape(6, D)
                for k, n in enumerate(("to_q", "to_k", "to_v")):
                    out[q + f"attn1.{n}.weight"] = G[p + "qkv"][k * D:(k + 1) * D]
                    out[q + f"attn1.{n}.bias"] = G[p + "qkv.bias"][k * D:(k + 1) * D]
                out[q + "attn1.to_out.0.weight"], out[q + "attn1.to_out.0.bias"] = G[p + "out"], G[p + "out.bias"]
                out[q + "ff.net.0.proj.weight"], out[q + "ff.net.0.proj.bias"] = G[p + "fc1"], G[p + "fc1.bias"]
                out[q + "ff.net.2.weight"], out[q + "ff.net.2.bias"] = G[p + "fc2"], G[p + "fc2.bias"]
                if kind == "s":
                    out[q + "attn2.to_q.weight"], out[q + "attn2.to_q.bias"] = G[p + "q2"], G[p + "q2.bias"]
                    out[q + "attn2.to_out.0.weight"], out[q + "attn2.to_out.0.bias"] = G[p + "o2"], G[p + "o2.bias"]
                    r = i * 2 * D
                    out[q + "attn2.to_k.weight"], out[q + "attn2.to_k.bias"] = G["kv"][r:r + D], G["kv.bias"][r:r + D]
                    out[q + "attn2.to_v.weight"], out[q + "attn2.to_v.bias"] = G["kv"][r + D:r + 2 * D], G["kv.bias"][r + D:r + 2 * D]
        return out


def trainable_names(model):
    """Every parameter except adaln_single.emb (the timestep embedder, whose (B, D) graph stays on torch autograd and gets its
    gradient from `dc`), in named_parameters order."""
    return [n for n, _ in model.named_parameters() if not n.startswith("adaln_single.emb.")]


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
    names = trainable_names(model)
    named = dict(model.named_parameters())
    return _LatteTrainFn.apply(eng, names, x, c, *[named[n] for n in names])
