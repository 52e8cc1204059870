"""Training step of `Latte` (BASELINE config 5: train.py:206-222 — forward + backward under `loss.backward()`).

The reference trains through torch autograd over ~1000 eager kernels per forward.  Here the forward keeps the activations the
backward needs and the backward is written out explicitly, op by op, over the same hand-written kernels as the sampling path
(the wgmma GEMM does every dgrad and wgrad; wgrads accumulate in fp32 straight into the gradient buffers through the
residual epilogue) plus the kernels of csrc/train.cu (LayerNorm-modulate backward, gate / GELU backward with the bias and
per-sample reductions fused, attention backward on tensor cores, 16-bit transposes, adaLN outer products).

Derivatives follow the reference forward (models/latte.py): block :177-181, modulate :28-29, attention 'math' :48-77, Mlp
:169-171, FinalLayer :197-201, PatchEmbed + pos_embed :330-331, temp_embed :357-358.  Rows stay in (b, f, n) order for
spatial AND temporal blocks (the regrouping of :355/:368 is index arithmetic inside the attention kernels), so every
per-sample adaLN vector addresses `rows_per_batch = F*N` consecutive rows.

Gradient checkpointing (`checkpoint=True`, the module's `gradient_checkpointing` flag): the forward keeps each block's input
only, and the backward reruns that block's forward right before its backward.  Both steps run the same `_block_forward` /
`_block_backward`; only the loops around them differ.

`TrainEngine` is backend-agnostic: the product backend is latte_b200.train_ops.NativeOps (C ABI, CUDA only, raises without
the extension); tests drive the same orchestration through oracle/train_ops_oracle.TorchOps on the CPU and compare with
gradients produced by the unmodified reference (tests/golden/train_tiny64.npz).
"""
from __future__ import annotations

import torch

_BLOCK_LINEARS = ("attn.qkv", "attn.proj", "mlp.fc1", "mlp.fc2")


class GradientCheckpointingMixin:
    """Gradient checkpointing under the names of diffusers' ModelMixin (the reference LatteT2V inherits them, and
    train_with_img.py:120-122 calls `enable_gradient_checkpointing()` when its config asks for it).  With the flag set, a
    training step keeps only each block's input and reruns the block's forward in the backward: the saved activations shrink
    from roughly 40-46 bytes per token and channel per block to 4, at the cost of one more forward through the blocks.  It
    changes no result, and no call other than the training step."""
    _supports_gradient_checkpointing = True
    gradient_checkpointing = False

    def enable_gradient_checkpointing(self):
        self.gradient_checkpointing = True

    def disable_gradient_checkpointing(self):
        self.gradient_checkpointing = False

    @property
    def is_gradient_checkpointing(self):
        return self.gradient_checkpointing


def _patch_rows(x, p):
    """(B, F, C, H, W) -> rows (b, f, gh, gw) x columns (c, i, j)."""
    B, Fr, C, H, Wd = x.shape
    xx = x.reshape(B * Fr, C, H // p, p, Wd // p, p).permute(0, 2, 4, 1, 3, 5)
    return xx.reshape(B * Fr * (H // p) * (Wd // p), C * p * p)


class TrainEngine:
    """`images` = I still frames per sample after the F = num_frames video frames (LatteIMG, latte_img.py:316-399).  With I > 0
    the rows of all video frames come first, in (b, f, n) order (T_v = B*F*N rows), then the rows of all images in (b, i, n)
    order.  Spatial blocks and the final layer run over every row with one adaLN row per frame (rows_per_batch = N); temporal
    blocks run on the prefix x[:T_v] -- exactly a Latte batch of B videos -- with one adaLN row per video (a strided view of the
    per-frame rows), and carry the image rows through unchanged."""

    def __init__(self, model, ops, dtype, images=0, checkpoint=False):
        self.m = model
        self.ops = ops
        self.dtype = dtype
        self.images = images
        #: gradient checkpointing: the forward keeps each block's input only and the backward reruns the block before its backward
        self.checkpoint = checkpoint
        self.saved = None
        self.w = None

    # ---------------------------------------------------------------------------------------------------------------
    def prepare(self):
        """Operand copies of the current parameters in the compute type -- ONE copy per weight: the forward GEMM reads it as
        [N][K], dgrad reads the same memory as an MN-major operand.  The 16-bit buffers persist on the model between steps
        (`model._train_operands`); a step refreshes all of them with one multi-tensor cast launch.  adaLN weights of all blocks
        + final layer land in one stacked buffer; patch-embed / final-layer operands are zero-padded to the GEMM's 64-element
        k-block (K = 16 and 32)."""
        m, ops = self.m, self.ops
        D = m.hidden_size
        dev = m.pos_embed.device
        lin = lambda blk, name: (getattr(getattr(blk, name.split(".")[0]), name.split(".")[1]))   # noqa: E731
        ada = [b.adaLN_modulation[1] for b in m.blocks] + [m.final_layer.adaLN_modulation[1]]
        cache = getattr(m, "_train_operands", None)
        key = (self.dtype, dev, type(ops).__name__)
        if cache is None or cache["key"] != key:
            NA = sum(a.weight.shape[0] for a in ada)
            cache = {"key": key, "ada_w": torch.empty(NA, D, dtype=self.dtype, device=dev), "w": {}}
            for i, blk in enumerate(m.blocks):
                for name in _BLOCK_LINEARS:
                    cache["w"][f"{i}.{name}"] = torch.empty(lin(blk, name).weight.shape, dtype=self.dtype, device=dev)
            m._train_operands = cache
        srcs, dsts = [], []
        for i, blk in enumerate(m.blocks):
            for name in _BLOCK_LINEARS:
                srcs.append(lin(blk, name).weight.detach())
                dsts.append(cache["w"][f"{i}.{name}"])
        row = 0
        for a in ada:
            srcs.append(a.weight.detach())
            dsts.append(cache["ada_w"][row:row + a.weight.shape[0]])
            row += a.weight.shape[0]
        if all(t.dtype == torch.float32 and t.is_contiguous() for t in srcs):
            ops.cast_into(srcs, dsts)
        else:                                   # 16-bit or non-contiguous parameters: plain copies
            for a, b in zip(srcs, dsts):
                b.copy_(a)
        W = {}
        for i, blk in enumerate(m.blocks):
            for name in _BLOCK_LINEARS:
                W[f"{i}.{name}"] = (cache["w"][f"{i}.{name}"], lin(blk, name).bias.detach().float().contiguous())
        W["ada_w"] = cache["ada_w"]
        W["ada_b"] = torch.cat([a.bias.detach() for a in ada]).float().contiguous()
        pw = m.x_embedder.proj.weight.detach().reshape(D, -1).float()
        self.kp = pw.shape[1]
        pad = torch.zeros(D, 64, dtype=torch.float32, device=dev)
        pad[:, : self.kp] = pw
        W["patch_w"] = ops.cast(pad)
        W["patch_b"] = m.x_embedder.proj.bias.detach().float().contiguous()
        fw = m.final_layer.linear.weight.detach().float()             # [p*p*Cout, D]
        self.nf = fw.shape[0]
        padk = torch.zeros(64, D, dtype=torch.float32, device=dev)
        padk[: self.nf] = fw
        W["final_wk"] = ops.cast(padk)                                # rows [0, nf) = the weight (forward), all 64 rows = dgrad operand
        W["final_w"] = W["final_wk"][: self.nf]
        W["final_b"] = m.final_layer.linear.bias.detach().float().contiguous()
        self.w = W

    # ---------------------------------------------------------------------------------------------------------------
    def _patchify(self, x):
        """(B, F[+I], C, H, W) -> rows (b, f, gh, gw) [then (b, i, gh, gw)] x columns (c, i, j): timm PatchEmbed's
        Conv2d(k = s = p) as a GEMM operand."""
        p, Fr = self.m.patch_size, self.m.num_frames
        if self.images:
            return torch.cat((_patch_rows(x[:, :Fr], p), _patch_rows(x[:, Fr:], p)))
        return _patch_rows(x, p)

    def _unpatchify(self, tok, B):
        """rows (b, f, h, w) x (p, q, c) -> (B, F, c, h*p, w*q) (latte.py:297-310, :375-376); image rows follow as frames F.."""
        m = self.m
        c, p = m.out_channels, m.patch_size
        g = m.input_size // p

        def unp(rows, frames):
            t = rows.view(B * frames, g, g, p, p, c).permute(0, 5, 1, 3, 2, 4)
            return t.reshape(B, frames, c, g * p, g * p)
        if self.images:
            Tv = B * m.num_frames * g * g
            return torch.cat((unp(tok[:Tv], m.num_frames), unp(tok[Tv:], self.images)), dim=1)
        return unp(tok, m.num_frames)

    def _patchify_out(self, dout):
        m = self.m
        c, p = m.out_channels, m.patch_size
        g = m.input_size // p

        def pat(d):
            B, frames = d.shape[:2]
            t = d.reshape(B * frames, c, g, p, g, p).permute(0, 2, 4, 3, 5, 1)
            return t.reshape(B * frames * g * g, p * p * c)
        if self.images:
            return torch.cat((pat(dout[:, :m.num_frames]), pat(dout[:, m.num_frames:])))
        return pat(dout).contiguous()

    # ---------------------------------------------------------------------------------------------------------------
    def _geometry(self, B):
        """(rows of all frames, rows of the video frames, rows_per_batch of spatial blocks / final layer, of temporal blocks)."""
        m = self.m
        Fr, N = m.num_frames, m.x_embedder.num_patches
        Tv = B * Fr * N
        if not self.images:
            return Tv, Tv, Fr * N, Fr * N
        return Tv + B * self.images * N, Tv, N, Fr * N

    def _temporal_rows(self, t, B):
        """The adaLN rows (of mod / dmod) a temporal block addresses: per sample without images, else the first frame's row of
        each video (every video frame carries the same conditioning)."""
        return t[0:B * self.m.num_frames:self.m.num_frames] if self.images else t

    @staticmethod
    def _join_rows(video, images):
        """One buffer of the video rows followed by the image rows: the output of a temporal block, whose image rows are its
        input's, copied device to device (B*I*N*D*4 bytes)."""
        return torch.cat((video, images))

    def _block_forward(self, i, xs, mod, B, temp, rerun=False):
        """Block i (latte.py:177-181) on its input xs (T x D fp32) -> (its output, the list of activations its backward reads).
        rerun=True is the checkpointed backward's recomputation: it stops before the last residual update, whose output the
        backward does not read, and returns None in its place."""
        m, ops, W = self.m, self.ops, self.w
        D, Fr, N, H = m.hidden_size, m.num_frames, m.x_embedder.num_patches, m.num_heads
        _, Tv, rpb, rpb_t = self._geometry(B)
        mod_t = self._temporal_rows(mod, B)
        temporal = bool(i % 2)
        mv = (mod_t if temporal else mod)[:, i * 6 * D:(i + 1) * 6 * D]
        sh1, sc1, g1, sh2, sc2, g2 = (mv[:, k * D:(k + 1) * D] for k in range(6))
        wq, wp, w1, w2 = (W[f"{i}.{n}"] for n in _BLOCK_LINEARS)
        rp = rpb_t if temporal else rpb
        xi = xs[:Tv] if temporal else xs        # temporal blocks see the video rows only (latte_img.py:373-374, 387-388)
        h1 = ops.ln_modulate(xi, sh1, sc1, rp)
        qkv = ops.linear(h1, wq[0], wq[1])
        o = ops.attention(qkv, B, Fr if temporal else Fr + self.images, N, H, temporal)
        m1 = ops.linear(o, wp[0], wp[1])
        # two passes: a kernel fusing the residual update with this LayerNorm-modulate measured slower (101 vs 45 + 40 us)
        xm = ops.gate_residual(xi, m1, g1, rp)
        h2 = ops.ln_modulate(xm, sh2, sc2, rp)
        u, a = ops.linear_gelu_both(h2, w1[0], w1[1])
        m2 = ops.linear(a, w2[0], w2[1])
        acts = [xi, h1, qkv, o, m1, xm, h2, u, a, m2]
        if rerun:
            return None, acts
        if i == 0 and self.images:
            # temp_embed goes to the video rows only (latte_img.py:377-378).  All frames of a video share one gate row, so
            # the video rows take the per-video view, like a temporal block.
            g2v = mod_t[:, 5 * D:6 * D]
            xo = self._join_rows(ops.gate_residual(xm[:Tv], m2[:Tv], g2v, rpb_t, row_add=temp, tokens=N),
                                 ops.gate_residual(xm[Tv:], m2[Tv:], g2[B * Fr:], rp))
        else:
            xo = ops.gate_residual(xm, m2, g2, rp, row_add=temp if i == 0 else None, tokens=N)
            if temporal and self.images:        # image rows pass through the temporal block unchanged
                xo = self._join_rows(xo, xs[Tv:])
        return xo, acts

    def _block_backward(self, i, acts, dx, mod, dmod, B, G, bias_flat):
        """Backward of block i from the list `_block_forward` returned, which it empties so that each buffer is freed as soon
        as it is used.  Accumulates into dx (T x D fp32; a temporal block touches the video rows only), dmod and the bias
        gradients in bias_flat; puts the weight gradients and bias views into G."""
        m, ops, W = self.m, self.ops, self.w
        D, Fr, N, H, Hm = m.hidden_size, m.num_frames, m.x_embedder.num_patches, m.num_heads, m.mlp_hidden
        _, Tv, rpb, rpb_t = self._geometry(B)
        xs, h1, qkv, o, m1, xm, h2, u, a, m2 = acts
        acts.clear()
        temporal = bool(i % 2)
        mv = (self._temporal_rows(mod, B) if temporal else mod)[:, i * 6 * D:(i + 1) * 6 * D]
        sh1, sc1, g1, sh2, sc2, g2 = (mv[:, k * D:(k + 1) * D] for k in range(6))
        dv = (self._temporal_rows(dmod, B) if temporal else dmod)[:, i * 6 * D:(i + 1) * 6 * D]
        dsh1, dsc1, dg1, dsh2, dsc2, dg2 = (dv[:, k * D:(k + 1) * D] for k in range(6))
        rp = rpb_t if temporal else rpb
        dxb = dx[:Tv] if temporal else dx       # a temporal block passes the image rows' gradient through untouched
        wq, wp, w1, w2 = (W[f"{i}.{n}"] for n in _BLOCK_LINEARS)
        p = f"blocks.{i}."
        off = i * (3 * D + D + Hm + D)
        G[p + "attn.qkv.bias"], G[p + "attn.proj.bias"] = bias_flat[off:off + 3 * D], bias_flat[off + 3 * D:off + 4 * D]
        G[p + "mlp.fc1.bias"], G[p + "mlp.fc2.bias"] = bias_flat[off + 4 * D:off + 4 * D + Hm], bias_flat[off + 4 * D + Hm:off + 5 * D + Hm]
        # x_out = x_mid + g2 * fc2(gelu(fc1(LNmod(x_mid))))
        dm2 = ops.gate_bwd(dxb, m2, g2, rp, dg2, G[p + "mlp.fc2.bias"])
        G[p + "mlp.fc2.weight"] = self._wgrad(dm2, a)
        del a
        # gelu'(u) is a separate pass: in this dgrad's epilogue it made the GEMM the bottleneck (327 us vs 153 + 129 us)
        da = ops.dgrad(dm2, w2[0])
        du = ops.gelu_bwd(da, u, G[p + "mlp.fc1.bias"])
        del da, dm2
        G[p + "mlp.fc1.weight"] = self._wgrad(du, h2)
        dh2 = ops.dgrad(du, w1[0])
        del du
        ops.ln_modulate_bwd(dh2, xm, sh2, sc2, rp, dxb, dsh2, dsc2)
        del dh2
        # x_mid = x_in + g1 * proj(attn(qkv(LNmod(x_in))))
        dm1 = ops.gate_bwd(dxb, m1, g1, rp, dg1, G[p + "attn.proj.bias"])
        G[p + "attn.proj.weight"] = self._wgrad(dm1, o)
        do = ops.dgrad(dm1, wp[0])
        del dm1
        dqkv = ops.attention_bwd(qkv, o, do, B, Fr if temporal else Fr + self.images, N, H, temporal)
        del do
        ops.colsum(dqkv, G[p + "attn.qkv.bias"])
        G[p + "attn.qkv.weight"] = self._wgrad(dqkv, h1)
        dh1 = ops.dgrad(dqkv, wq[0])
        del dqkv
        ops.ln_modulate_bwd(dh1, xs, sh1, sc1, rp, dxb, dsh1, dsc1)

    def _wgrad(self, dy, x):
        g = torch.zeros(dy.shape[1], x.shape[1], dtype=torch.float32, device=dy.device)
        return self.ops.wgrad(g, dy, x)

    def forward(self, x, c, save=True):
        """x (B, F[+I], C, H, W) fp32 -> (B, F[+I], 2C, H, W) fp32.  c: (B, D) fp32 = t_embedder(t) + y_embedder(y)
        (latte.py:332-348) without images, else (B*(F+I), D) per-frame conditioning in row order (`frame_conditioning`).
        save=False runs the forward without keeping the activations the backward needs.  With `checkpoint`, each block keeps
        only its input xs (T x D fp32)."""
        if self.w is None:
            self.prepare()
        m, ops, W = self.m, self.ops, self.w
        B = x.shape[0]
        D, Fr, N = m.hidden_size, m.num_frames, m.x_embedder.num_patches
        T, _, rpb, _ = self._geometry(B)
        Fs = Fr + self.images                   # frames a spatial block sees
        dev = x.device
        sc = ops.to_operand(torch.nn.functional.silu(c.float()).contiguous())            # adaLN_modulation[0], final too
        mod = ops.linear(sc, W["ada_w"], W["ada_b"]).float()                               # (B or B(F+I), depth*6D + 2D)
        S = {"B": B, "c": c, "sc": sc, "mod": mod, "blocks": []}

        xp = torch.zeros(T, 64, dtype=torch.float32, device=dev)
        xp[:, : self.kp] = self._patchify(x.float())
        xp = ops.to_operand(xp)
        xs = m.pos_embed.detach().float().reshape(1, N, D).expand(B * Fs, N, D).reshape(T, D).contiguous()
        ops.linear_accum(xs, xp, W["patch_w"], W["patch_b"])
        if save:
            S["xp"] = xp
        del xp
        temp = m.temp_embed.detach().float().reshape(Fr, D).contiguous()
        for i in range(m.depth):
            xo, acts = self._block_forward(i, xs, mod, B, temp)
            if save:
                S["blocks"].append(xs if self.checkpoint else acts)
            del acts                            # a checkpointed block's activations are freed before the next block runs
            xs = xo
        base = m.depth * 6 * D
        shf, scf = mod[:, base:base + D], mod[:, base + D:base + 2 * D]
        hf = ops.ln_modulate(xs, shf, scf, rpb)
        tok = torch.zeros(T, self.nf, dtype=torch.float32, device=dev)
        ops.linear_accum(tok, hf, W["final_w"], W["final_b"])
        S["x_last"], S["hf"] = xs, hf
        self.saved = S if save else None
        return self._unpatchify(tok, B)

    # ---------------------------------------------------------------------------------------------------------------
    def backward(self, dout):
        """dout (B, F, 2C, H, W) -> (grads: {parameter name: fp32 tensor}, dc (B, D) fp32).  Frees the saved activations.
        Bias gradients, the per-sample adaLN gradients (dmod) and every weight gradient are views of buffers zeroed once here;
        the kernels accumulate into them (wgrad through the GEMM's fp32 residual epilogue, reductions with atomics)."""
        m, ops, W, S = self.m, self.ops, self.w, self.saved
        self.saved = None
        B = S["B"]
        D, Hm = m.hidden_size, m.mlp_hidden
        T, _, rpb, _ = self._geometry(B)
        dev = dout.device
        mod = S["mod"]
        G = {}
        dmod = torch.zeros_like(mod)
        # all bias gradients in one zeroed buffer: per block [qkv 3D | proj D | fc1 Hm | fc2 D], then final (nf), patch (D)
        per_blk = 3 * D + D + Hm + D
        bias_flat = torch.zeros(m.depth * per_blk + self.nf + D, dtype=torch.float32, device=dev)
        wgrad = self._wgrad

        # ---- final layer (latte.py:197-201) ----
        dtok = self._patchify_out(dout.float())                                         # (T, nf) fp32
        G["final_layer.linear.bias"] = ops.colsum(dtok, bias_flat[m.depth * per_blk: m.depth * per_blk + self.nf])
        dtok16 = ops.to_operand(dtok)
        G["final_layer.linear.weight"] = wgrad(dtok16, S["hf"])
        dtp = torch.zeros(T, 64, dtype=torch.float32, device=dev)
        dtp[:, : self.nf] = dtok
        dhf = ops.dgrad(ops.to_operand(dtp), W["final_wk"])
        dx = torch.zeros(T, D, dtype=torch.float32, device=dev)
        base = m.depth * 6 * D
        ops.ln_modulate_bwd(dhf, S["x_last"], mod[:, base:base + D], mod[:, base + D:base + 2 * D], rpb, dx,
                            dmod[:, base:base + D], dmod[:, base + D:base + 2 * D])
        del dhf, dtp, dtok16

        # ---- blocks, last to first (latte.py:177-181); a checkpointed block first reruns its forward from its saved input
        for i in reversed(range(m.depth)):
            acts = S["blocks"].pop()
            if self.checkpoint:
                acts = self._block_forward(i, acts, mod, B, None, rerun=True)[1]
            self._block_backward(i, acts, dx, mod, dmod, B, G, bias_flat)

        # ---- patch embedding (latte.py:330-331; pos_embed / temp_embed are frozen, :246-247) ----
        G["x_embedder.proj.bias"] = ops.colsum(dx, bias_flat[m.depth * per_blk + self.nf:])
        gpe = wgrad(ops.to_operand(dx), S["xp"])
        G["x_embedder.proj.weight"] = gpe[:, : self.kp].reshape(m.x_embedder.proj.weight.shape).contiguous()

        # ---- adaLN_modulation of every block + final layer: mod = Linear(SiLU(c)) (latte.py:160-163, 192-195) ----
        dW = ops.ada_outer(dmod, S["sc"])                                               # (depth*6D + 2D, D)
        db = dmod.sum(0)
        for i in range(m.depth):
            G[f"blocks.{i}.adaLN_modulation.1.weight"] = dW[i * 6 * D:(i + 1) * 6 * D]
            G[f"blocks.{i}.adaLN_modulation.1.bias"] = db[i * 6 * D:(i + 1) * 6 * D]
        G["final_layer.adaLN_modulation.1.weight"] = dW[base:base + 2 * D]
        G["final_layer.adaLN_modulation.1.bias"] = db[base:base + 2 * D]
        dsc = ops.ada_dsc(dmod, W["ada_w"])
        c = S["c"].float()
        sg = torch.sigmoid(c)
        dc = dsc * (sg * (1 + c * (1 - sg)))                                            # d silu
        return G, dc


def trainable_names(model):
    """Names, in a fixed order, of the parameters the engine produces gradients for (everything except the embedders that
    feed `c`, whose few-kilobyte graph stays on torch autograd, and the frozen sin-cos tables)."""
    names = ["x_embedder.proj.weight", "x_embedder.proj.bias"]
    for i in range(model.depth):
        for n in _BLOCK_LINEARS:
            names += [f"blocks.{i}.{n}.weight", f"blocks.{i}.{n}.bias"]
        names += [f"blocks.{i}.adaLN_modulation.1.weight", f"blocks.{i}.adaLN_modulation.1.bias"]
    names += ["final_layer.linear.weight", "final_layer.linear.bias",
              "final_layer.adaLN_modulation.1.weight", "final_layer.adaLN_modulation.1.bias"]
    return names


class _LatteTrainFn(torch.autograd.Function):
    """Autograd boundary: inputs (x, c, *parameters) -> output; backward hands each parameter its gradient, so optimizers,
    `clip_grad_norm_`, gradient accumulation and DistributedDataParallel's bucketed all-reduce hooks see ordinary `.grad`s."""

    @staticmethod
    def forward(ctx, engine, names, x, c, *params):
        ctx.engine, ctx.names = engine, names
        ctx.dtypes = [p.dtype for p in params]
        with torch.no_grad():
            engine.prepare()
            out = engine.forward(x.detach(), c.detach())
        return out

    @staticmethod
    def backward(ctx, dout):
        eng = ctx.engine
        if eng.saved is None:
            raise RuntimeError("latte_b200: backward called twice on one training forward (activations are freed after the first)")
        with torch.no_grad():
            G, dc = eng.backward(dout.contiguous())
        grads = tuple(G[n].to(dt) if G[n].dtype != dt else G[n] for n, dt in zip(ctx.names, ctx.dtypes))
        return (None, None, None, dc) + grads


def train_forward(model, ops, dtype, x, c, images=0):
    """Forward of one training step with the backward attached.  c = t_embedder(t) + y_embedder(y), computed by the caller with
    torch autograd (a (B, D) graph); with `images` still frames per sample, the per-frame `frame_conditioning` instead.
    Checkpoints each block when `model.gradient_checkpointing` is set."""
    eng = TrainEngine(model, ops, dtype, images, checkpoint=model.gradient_checkpointing)
    names = trainable_names(model)
    named = dict(model.named_parameters())
    params = [named[n] for n in names]
    return _LatteTrainFn.apply(eng, names, x, c, *params)


def conditioning(model, t, y):
    """c = t_embedder(t) [+ y_embedder(y)] with torch autograd (latte.py:98-123 sincos + MLP, :148-153 table lookup): a
    (B, D) graph of a handful of kernels whose parameters get their gradients from `dc`."""
    c = _timestep_embedding(model, t)
    if model.extras == 2:
        c = c + model.y_embedder.embedding_table(y).float()
    return c


def _timestep_embedding(model, t):
    import math
    half = model.t_embedder.frequency_embedding_size // 2
    freqs = torch.exp(-math.log(10000) * torch.arange(0, half, dtype=torch.float32, device=t.device) / half)
    args = t[:, None].float() * freqs[None]
    emb = torch.cat([torch.cos(args), torch.sin(args)], dim=-1)
    return model.t_embedder.mlp(emb.to(model.t_embedder.mlp[0].weight.dtype)).float()


def frame_conditioning(model, t, y, y_image, images):
    """Per-frame conditioning of video + image joint training (latte_img.py:331, 336-349), (B*(F+I), D) in the engine's row
    order: the B*F video frames first, (b, f) -> t_emb[b] [+ y_emb(y[b])], then the B*I images, (b, i) -> t_emb[b]
    [+ y_emb(y_image[b, i])].  y_image (B, I) int64; labels already dropped by the caller.  Torch autograd carries `dc` back to
    the embedders, as for `conditioning`."""
    temb = _timestep_embedding(model, t)
    B, D = temb.shape
    cv, ci = temb, temb[:, None].expand(B, images, D)
    if model.extras == 2:
        table = model.y_embedder.embedding_table
        cv = cv + table(y).float()
        ci = ci + table(y_image).float()
    return torch.cat((cv.repeat_interleave(model.num_frames, dim=0), ci.reshape(B * images, D)))


def image_forward(model, ops, dtype, x, c, images):
    """Forward only (no activations kept, no autograd node) of a video + image batch through the training engine."""
    eng = TrainEngine(model, ops, dtype, images)
    with torch.no_grad():
        eng.prepare()
        return eng.forward(x.detach().float(), c.detach(), save=False)
