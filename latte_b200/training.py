"""Training step of `Latte` (BASELINE config 5: train.py:206-222 — forward + backward under `loss.backward()`), and the engine
base that the step of `LatteT2V` (training_t2v.py) shares.

The reference trains through torch autograd over ~1000 eager kernels per forward.  Here the forward keeps the activations the
backward needs and the backward is written out explicitly, op by op, over the same hand-written kernels as the sampling path
(the wgmma GEMM does every dgrad and wgrad; wgrads accumulate in fp32 straight into the gradient buffers through the
residual epilogue) plus the kernels of csrc/train.cu (LayerNorm-modulate backward, gate / GELU backward with the bias and
per-sample reductions fused, attention backward on tensor cores, 16-bit transposes, adaLN outer products).

Derivatives follow the reference forward (models/latte.py): block :177-181, modulate :28-29, attention 'math' :48-77, Mlp
:169-171, FinalLayer :197-201, PatchEmbed + pos_embed :330-331, temp_embed :357-358.  Rows stay in (b, f, n) order for
spatial AND temporal blocks (the regrouping of :355/:368 is index arithmetic inside the attention kernels), so every
per-sample adaLN vector addresses `rows_per_batch = F*N` consecutive rows.

`_EngineBase` holds the step once: the operand cache, the row layout, patchify / unpatchify, the block (LN-modulate ->
attention -> gated residual -> LN-modulate -> fc1 / GELU -> fc2 -> gated residual) and its backward, the step loop and the
mapping of gradients back to parameter names.  `TrainEngine` (Latte, LatteIMG) and `training_t2v.T2VTrainEngine` (LatteT2V)
supply their operand table and override what differs: how the modulation rows come from `linear(silu(c))`, where the
temporal embedding joins, and LatteT2V's caption projection and cross-attention.

Gradient checkpointing (`checkpoint=True`, the module's `gradient_checkpointing` flag): the forward keeps each block's input
only, and the backward reruns that block's forward right before its backward.  Both steps run the same `_block_forward` /
`_block_backward`; only the loops around them differ.

The engines are backend-agnostic: the product backend is latte_b200.train_ops.NativeOps (C ABI, CUDA only, raises without
the extension); tests drive the same orchestration through oracle/train_ops_oracle.TorchOps on the CPU and compare with
gradients produced by the unmodified reference (tests/golden/train_tiny64.npz).
"""
from __future__ import annotations

import functools
import math

import torch


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


def native_backend(model, param_dtype):
    """(operand type, NativeOps) of a training step: the autocast dtype under `torch.autocast` (the reference's mixed-precision
    recipe), else the parameter dtype if it is 16-bit, else `model.train_dtype`.  One backend object per operand type stays on
    the model: it caches the multi-cast pointer table and its workspaces."""
    from . import train_ops
    od = param_dtype if param_dtype in (torch.float16, torch.bfloat16) else model.train_dtype
    if torch.is_autocast_enabled("cuda"):
        od = torch.get_autocast_dtype("cuda")
        if od not in (torch.float16, torch.bfloat16):
            raise TypeError(f"latte_b200: autocast dtype {od} is not a tensor-core operand type")
    if model._train_backend is None:
        model._train_backend = {}
    ops = model._train_backend.get(od)
    if ops is None:
        ops = model._train_backend[od] = train_ops.NativeOps(od)
    return od, ops


def _patch_rows(x, p):
    """(B, F, C, H, W) -> rows (b, f, gh, gw) x columns (c, i, j)."""
    B, Fr, C, H, Wd = x.shape
    xx = x.reshape(B * Fr, C, H // p, p, Wd // p, p).permute(0, 2, 4, 1, 3, 5)
    return xx.reshape(B * Fr * (H // p) * (Wd // p), C * p * p)


def _pad64(n):
    """n rounded up to the GEMM's 64-element k-block."""
    return (n + 63) // 64 * 64


def _f32(ts):
    """fp32 copy of parameters stacked by rows (the parameter itself when it is one fp32 tensor)."""
    return ts[0].detach().float().contiguous() if len(ts) == 1 else torch.cat([t.detach().float() for t in ts])


class _EngineBase:
    """One training forward + backward of a Latte-family denoiser on `ops` with operand type `dtype`.

    `images` = I still frames per sample after the F video frames.  With I > 0 the rows of all video frames come first, in
    (b, f, n) order (T_v = B*F*N rows), then the rows of all images in (b, i, n) order.  Spatial blocks and the output head
    run over every row with one modulation row per frame (rows_per_batch = N); temporal blocks run on the prefix x[:T_v] --
    exactly a batch of B videos -- with one modulation row per video (a strided view of the per-frame rows), and carry the
    image rows through unchanged.  Inputs and outputs are (B, F[+I], C, H, W).

    A subclass sets the geometry (D, H, Fr, N, p, nblocks), `patch_conv`, `final_linear` and `pos_table`, and defines
    `_operands`, `_temp_embed`, `_modulation` and `_modulation_backward`; blocks alternate spatial (even j) and temporal
    (odd j)."""

    def __init__(self, model, ops, dtype, images=0, checkpoint=False):
        self.m = model
        self.ops = ops
        self.dtype = dtype
        self.images = images
        #: gradient checkpointing: the forward keeps each block's input only and the backward reruns the block before its backward
        self.checkpoint = checkpoint
        self.saved = None
        self.w = None
        #: (key, weights, biases) of every GEMM operand: the parameters stacked by rows into one 16-bit buffer (and one fp32 bias)
        self.table = self._operands()

    @functools.cached_property
    def params(self):
        """name -> parameter, in named_parameters order: one walk over the module tree per training step (none for a forward
        without backward)."""
        return dict(self.m.named_parameters())

    @functools.cached_property
    def names(self):
        """id(parameter) -> name."""
        return {id(p): n for n, p in self.params.items()}

    # ---------------------------------------------------------------------------------------------------------------
    def _operands(self):
        raise NotImplementedError

    def _extra_params(self):
        """Trained parameters outside the operand table, the patch embedding and the output projection."""
        return ()

    def trainable_names(self):
        """Names, in named_parameters order, of the parameters the engine produces gradients for."""
        own = [p for _, ws, bs in self.table for p in ws + bs] + list(self._extra_params())
        own += [self.patch_conv.weight, self.patch_conv.bias, self.final_linear.weight, self.final_linear.bias]
        ids = {id(p) for p in own}
        return [n for i, n in self.names.items() if i in ids]

    def prepare(self):
        """Operand copies of the current parameters in the compute type -- ONE copy per weight: the forward GEMM reads it as
        [N][K], dgrad reads the same memory as an MN-major operand.  The 16-bit buffers persist on the model between steps
        (`model._train_operands`); a step refreshes all of them with one multi-tensor cast launch.  Stacked operands (the adaLN
        weights of all Latte blocks, q|k|v, every LatteT2V layer's k|v) are one buffer whose row slices are the parameters'
        copies.  Patch-embed / output-projection operands are zero-padded to a multiple of the GEMM's 64-element k-block
        (`_pad64`: K = C*p*p = 16 -> 64, 64, 256; the head's p*p*C_out rows 32 -> 64, 64, 128, 256, 512)."""
        m, ops, D = self.m, self.ops, self.D
        dev = self.final_linear.weight.device
        cache = getattr(m, "_train_operands", None)
        key = (self.dtype, dev, type(ops).__name__)
        if cache is None or cache["key"] != key:
            cache = {"key": key, "w": {k: torch.empty(sum(p.shape[0] for p in ws), ws[0].shape[1], dtype=self.dtype, device=dev)
                                       for k, ws, _ in self.table}}
            m._train_operands = cache
        srcs, dsts = [], []
        for k, ws, _ in self.table:
            row = 0
            for p in ws:
                srcs.append(p.detach())
                dsts.append(cache["w"][k][row:row + p.shape[0]])
                row += p.shape[0]
        if all(t.dtype == torch.float32 and t.is_contiguous() for t in srcs):
            ops.cast_into(srcs, dsts)
        else:                                   # 16-bit or non-contiguous parameters: plain copies
            for a, b in zip(srcs, dsts):
                b.copy_(a)
        W = {k: (cache["w"][k], _f32(bs)) for k, _, bs in self.table}
        pw = self.patch_conv.weight.detach().reshape(D, -1).float()
        self.kp = pw.shape[1]
        pad = torch.zeros(D, _pad64(self.kp), dtype=torch.float32, device=dev)
        pad[:, : self.kp] = pw
        W["patch"] = (ops.cast(pad), self.patch_conv.bias.detach().float().contiguous())
        fw = self.final_linear.weight.detach().float()              # [p*p*Cout, D]
        self.nf = fw.shape[0]
        padk = torch.zeros(_pad64(self.nf), D, dtype=torch.float32, device=dev)
        padk[: self.nf] = fw
        W["final_wk"] = ops.cast(padk)                              # rows [0, nf) = the weight (forward), all rows = dgrad operand
        W["final"] = (W["final_wk"][: self.nf], self.final_linear.bias.detach().float().contiguous())
        self.w = W

    # ---------------------------------------------------------------------------------------------------------------
    def _geometry(self, B):
        """(rows of all frames, rows of the video frames, rows_per_batch of spatial blocks / output head, of temporal blocks)."""
        Tv = B * self.Fr * self.N
        if not self.images:
            return Tv, Tv, self.Fr * self.N, self.Fr * self.N
        return Tv + B * self.images * self.N, Tv, self.N, self.Fr * self.N

    def _temporal_rows(self, t, B):
        """The modulation rows (of mod / dmod) a temporal block addresses: per sample without images, else the first frame's row
        of each video (a strided view: every video frame carries the same conditioning)."""
        return t[0:B * self.Fr:self.Fr] if self.images else t

    @staticmethod
    def _join_rows(video, images):
        """One buffer of the video rows followed by the image rows: the output of a temporal block, whose image rows are its
        input's, copied device to device (B*I*N*D*4 bytes)."""
        return torch.cat((video, images))

    def _patchify(self, x):
        """(B, F[+I], C, H, W) -> rows (b, f, gh, gw) [then (b, i, gh, gw)] x columns (c, i, j): PatchEmbed's Conv2d(k = s = p)
        as a GEMM operand."""
        if self.images:
            return torch.cat((_patch_rows(x[:, :self.Fr], self.p), _patch_rows(x[:, self.Fr:], self.p)))
        return _patch_rows(x, self.p)

    def _unpatchify(self, tok, B):
        """rows (b, f, h, w) x (p, q, c) -> (B, F, c, h*p, w*q) (latte.py:297-310, :375-376); image rows follow as frames F.."""
        c, p, g = self.nf // self.p ** 2, self.p, math.isqrt(self.N)

        def unp(rows, frames):
            t = rows.view(B * frames, g, g, p, p, c).permute(0, 5, 1, 3, 2, 4)
            return t.reshape(B, frames, c, g * p, g * p)
        if self.images:
            Tv = B * self.Fr * self.N
            return torch.cat((unp(tok[:Tv], self.Fr), unp(tok[Tv:], self.images)), dim=1)
        return unp(tok, self.Fr)

    def _patchify_out(self, dout):
        """Adjoint of `_unpatchify`: the output gradient as (rows, p*p*c)."""
        c, p, g = self.nf // self.p ** 2, self.p, math.isqrt(self.N)

        def pat(d):
            B, frames = d.shape[:2]
            t = d.reshape(B * frames, c, g, p, g, p).permute(0, 2, 4, 3, 5, 1)
            return t.reshape(B * frames * g * g, p * p * c)
        if self.images:
            return torch.cat((pat(dout[:, :self.Fr]), pat(dout[:, self.Fr:])))
        return pat(dout).contiguous()

    # ---------------------------------------------------------------------------------------------------------------
    # What a model does differently.  The defaults are those of a model without a caption.
    def _context_forward(self, S, save):
        """Per-step state every block reads (LatteT2V: the caption K/V), put into S."""

    def _cross_forward(self, j, xm, S):
        """Between the two halves of spatial block j: updates xm in place, returns what `_cross_backward` reads."""
        return None

    def _begin_backward(self, S, dev):
        """Per-step gradient buffers of `_context_forward`'s state, put into S."""

    def _context_backward(self, S, G, bgrad):
        """Backward of `_context_forward`, after the block loop."""

    def _add_temp(self, xm, m2, g2, mod_t, B, temp):
        """Last residual update of block 0, which adds the temporal embedding `temp` (None: nothing to add)."""
        return self.ops.gate_residual(xm, m2, g2, self._geometry(B)[2], row_add=temp, tokens=self.N)

    # ---------------------------------------------------------------------------------------------------------------
    def _block_forward(self, j, xs, S, temp=None, rerun=False):
        """Block j on its input xs (T x D fp32) -> (its output, the list of activations its backward reads).  rerun=True is the
        checkpointed backward's recomputation: it stops before the last residual update, whose output the backward does not
        read, and returns None in its place."""
        ops, W, D, N = self.ops, self.w, self.D, self.N
        B, mod = S["B"], S["mod"]
        _, Tv, rpb, rpb_t = self._geometry(B)
        mod_t = self._temporal_rows(mod, B)
        temporal = bool(j % 2)
        mv = (mod_t if temporal else mod)[:, j * 6 * D:(j + 1) * 6 * D]
        sh1, sc1, g1, sh2, sc2, g2 = (mv[:, k * D:(k + 1) * D] for k in range(6))
        rp = rpb_t if temporal else rpb
        xi = xs[:Tv] if temporal else xs        # temporal blocks see the video rows only (latte_img.py:373-374, 387-388)
        h1 = ops.ln_modulate(xi, sh1, sc1, rp)
        qkv = ops.linear(h1, *W[j, "qkv"])
        o = ops.attention(qkv, B, self.Fr if temporal else self.Fr + self.images, N, self.H, temporal)
        m1 = ops.linear(o, *W[j, "out"])
        # two passes: a kernel fusing the residual update with this LayerNorm-modulate measured slower (101 vs 45 + 40 us)
        xm = ops.gate_residual(xi, m1, g1, rp)
        cross = None if temporal else self._cross_forward(j, xm, S)
        h2 = ops.ln_modulate(xm, sh2, sc2, rp)
        u, a = ops.linear_gelu_both(h2, *W[j, "fc1"])
        m2 = ops.linear(a, *W[j, "fc2"])
        acts = [xi, h1, qkv, o, m1, cross, xm, h2, u, a, m2]
        if rerun:
            return None, acts
        if j == 0:
            return self._add_temp(xm, m2, g2, mod_t, B, temp), acts
        xo = ops.gate_residual(xm, m2, g2, rp, tokens=N)
        if temporal and self.images:            # image rows pass through the temporal block unchanged
            xo = self._join_rows(xo, xs[Tv:])
        return xo, acts

    def _block_backward(self, j, acts, dx, S, dmod, G, bgrad):
        """Backward of block j from the list `_block_forward` returned, which it empties so that each buffer is freed as soon
        as it is used.  Accumulates into dx (T x D fp32; a temporal block touches the video rows only), dmod and the bias
        gradients bgrad; puts the weight gradients into G.  Returns dx, which a cross-attention replaces."""
        ops, W, D = self.ops, self.w, self.D
        B, mod = S["B"], S["mod"]
        _, Tv, rpb, rpb_t = self._geometry(B)
        xs, h1, qkv, o, m1, cross, xm, h2, u, a, m2 = acts
        acts.clear()
        temporal = bool(j % 2)
        mv = (self._temporal_rows(mod, B) if temporal else mod)[:, j * 6 * D:(j + 1) * 6 * D]
        sh1, sc1, g1, sh2, sc2, g2 = (mv[:, k * D:(k + 1) * D] for k in range(6))
        dv = (self._temporal_rows(dmod, B) if temporal else dmod)[:, j * 6 * D:(j + 1) * 6 * D]
        dsh1, dsc1, dg1, dsh2, dsc2, dg2 = (dv[:, k * D:(k + 1) * D] for k in range(6))
        rp = rpb_t if temporal else rpb
        dxb = dx[:Tv] if temporal else dx       # a temporal block passes the image rows' gradient through untouched
        # x_out = x_mid + g2 * fc2(gelu(fc1(LNmod(x_mid))))
        dm2 = ops.gate_bwd(dxb, m2, g2, rp, dg2, bgrad[j, "fc2"])
        G[j, "fc2"] = self._wgrad(dm2, a)
        del a
        # gelu'(u) is a separate pass: in this dgrad's epilogue it made the GEMM the bottleneck (327 us vs 153 + 129 us)
        da = ops.dgrad(dm2, W[j, "fc2"][0])
        du = ops.gelu_bwd(da, u, bgrad[j, "fc1"])
        del da, dm2
        G[j, "fc1"] = self._wgrad(du, h2)
        dh2 = ops.dgrad(du, W[j, "fc1"][0])
        del du
        ops.ln_modulate_bwd(dh2, xm, sh2, sc2, rp, dxb, dsh2, dsc2)
        del dh2
        if cross is not None:
            dx = dxb = self._cross_backward(j, cross, dx, S, G, bgrad)
        # x_mid = x_in + g1 * proj(attn(qkv(LNmod(x_in))))
        dm1 = ops.gate_bwd(dxb, m1, g1, rp, dg1, bgrad[j, "out"])
        G[j, "out"] = self._wgrad(dm1, o)
        do = ops.dgrad(dm1, W[j, "out"][0])
        del dm1
        dqkv = ops.attention_bwd(qkv, o, do, B, self.Fr if temporal else self.Fr + self.images, self.N, self.H, temporal)
        del do
        ops.colsum(dqkv, bgrad[j, "qkv"])
        G[j, "qkv"] = self._wgrad(dqkv, h1)
        dh1 = ops.dgrad(dqkv, W[j, "qkv"][0])
        del dqkv
        ops.ln_modulate_bwd(dh1, xs, sh1, sc1, rp, dxb, dsh1, dsc1)
        return dx

    def _wgrad(self, dy, x):
        g = torch.zeros(dy.shape[1], x.shape[1], dtype=torch.float32, device=dy.device)
        return self.ops.wgrad(g, dy, x)

    # ---------------------------------------------------------------------------------------------------------------
    def forward(self, x, c, save=True):
        """x (B, F[+I], C, H, W) fp32 -> (B, F[+I], 2C or out_channels, H, W) fp32.  c:
        the (B, D) fp32 conditioning, or with images (Latte) one row per frame.  save=False runs the forward without keeping the
        activations the backward needs.  With `checkpoint`, each block keeps only its input xs (T x D fp32)."""
        if self.w is None:
            self.prepare()
        ops, W, D, N = self.ops, self.w, self.D, self.N
        B = x.shape[0]
        T, _, rpb, _ = self._geometry(B)
        dev = x.device
        sc = ops.to_operand(torch.nn.functional.silu(c.float()).contiguous())            # adaLN_modulation[0], final too
        mod = self._modulation(ops.linear(sc, *W["ada"]).float(), c, B)
        S = {"B": B, "c": c, "sc": sc, "mod": mod, "blocks": []}
        self._context_forward(S, save)

        xp = torch.zeros(T, _pad64(self.kp), dtype=torch.float32, device=dev)
        xp[:, : self.kp] = self._patchify(x.float())
        xp = ops.to_operand(xp)
        xs = self.pos_table.detach().float().reshape(1, N, D).expand(B * (self.Fr + self.images), N, D).reshape(T, D).contiguous()
        ops.linear_accum(xs, xp, *W["patch"])
        if save:
            S["xp"] = xp
        del xp
        temp = self._temp_embed()
        for j in range(self.nblocks):
            xo, acts = self._block_forward(j, xs, S, temp)
            if save:
                S["blocks"].append(xs if self.checkpoint else acts)
            del acts                            # a checkpointed block's activations are freed before the next block runs
            xs = xo
        base = self.nblocks * 6 * D
        hf = ops.ln_modulate(xs, mod[:, base:base + D], mod[:, base + D:base + 2 * D], rpb)
        tok = torch.zeros(T, self.nf, dtype=torch.float32, device=dev)
        ops.linear_accum(tok, hf, *W["final"])
        S["x_last"], S["hf"] = xs, hf
        self.saved = S if save else None
        return self._unpatchify(tok, B)

    def backward(self, dout):
        """dout (B, F[+I], 2C or out_channels, H, W) -> (grads: {parameter name: fp32 tensor}, dc fp32).  Frees the saved activations.
        Bias gradients, the modulation gradients (dmod) and every weight gradient are views of buffers zeroed once here; the
        kernels accumulate into them (wgrad through the GEMM's fp32 residual epilogue, reductions with atomics)."""
        ops, W, S = self.ops, self.w, self.saved
        self.saved = None
        B, mod = S["B"], S["mod"]
        D = self.D
        T, _, rpb, _ = self._geometry(B)
        dev = dout.device
        dmod = torch.zeros_like(mod)
        G = {}
        bgrad = self._bias_grads(dev)

        # ---- output head (latte.py:197-201)
        dtok = self._patchify_out(dout.float())                                         # (T, nf) fp32
        ops.colsum(dtok, bgrad["final"])
        G["final"] = self._wgrad(ops.to_operand(dtok), S["hf"])
        dtp = torch.zeros(T, _pad64(self.nf), dtype=torch.float32, device=dev)
        dtp[:, : self.nf] = dtok
        dhf = ops.dgrad(ops.to_operand(dtp), W["final_wk"])
        dx = torch.zeros(T, D, dtype=torch.float32, device=dev)
        base = self.nblocks * 6 * D
        ops.ln_modulate_bwd(dhf, S["x_last"], mod[:, base:base + D], mod[:, base + D:base + 2 * D], rpb, dx,
                            dmod[:, base:base + D], dmod[:, base + D:base + 2 * D])
        del dhf, dtp, dtok
        self._begin_backward(S, dev)

        # ---- blocks, last to first; a checkpointed block first reruns its forward from its saved input
        for j in reversed(range(self.nblocks)):
            acts = S["blocks"].pop()
            if self.checkpoint:
                acts = self._block_forward(j, acts, S, rerun=True)[1]
            dx = self._block_backward(j, acts, dx, S, dmod, G, bgrad)

        # ---- patch embedding (latte.py:330-331; the sin-cos tables are frozen, :246-247)
        ops.colsum(dx, bgrad["patch"])
        G["patch"] = self._wgrad(ops.to_operand(dx), S["xp"])
        del dx
        self._context_backward(S, G, bgrad)

        # ---- the modulation's linear(silu(c)) (latte.py:160-163, 192-195): dA = its output's gradient
        grads = {}
        dA, dc_terms = self._modulation_backward(dmod, S, grads)
        G["ada"] = ops.ada_outer(dA, S["sc"])
        bgrad["ada"] = dA.sum(0)
        dsc = ops.ada_dsc(dA, W["ada"][0])
        c = S["c"].float()
        sg = torch.sigmoid(c)
        dc = dsc * (sg * (1 + c * (1 - sg)))                                            # d silu
        for t in dc_terms:
            dc = dc + t
        return self._named(G, bgrad, grads), dc

    def _bias_grads(self, dev):
        """{operand key: zeroed fp32 bias gradient}: views of one buffer, for every operand but "ada" (whose bias gradient is a
        row sum of dA), then "final" and "patch"."""
        sizes = [(k, sum(b.shape[0] for b in bs)) for k, _, bs in self.table if k != "ada"] + [("final", self.nf), ("patch", self.D)]
        flat = torch.zeros(sum(n for _, n in sizes), dtype=torch.float32, device=dev)
        out, off = {}, 0
        for k, n in sizes:
            out[k] = flat[off:off + n]
            off += n
        return out

    def _named(self, G, bgrad, grads):
        """Operand gradients -> parameter names: stacked weight and bias gradients split back by rows."""
        name = self.names
        for k, ws, bs in self.table:
            for ps, g in ((ws, G[k]), (bs, bgrad[k])):
                row = 0
                for p in ps:
                    grads[name[id(p)]] = g[row:row + p.shape[0]]
                    row += p.shape[0]
        pc, fl = self.patch_conv, self.final_linear
        grads[name[id(pc.weight)]] = G["patch"][:, : self.kp].reshape(pc.weight.shape).contiguous()
        grads[name[id(pc.bias)]] = bgrad["patch"]
        grads[name[id(fl.weight)]], grads[name[id(fl.bias)]] = G["final"], bgrad["final"]
        return grads

    def train_forward(self, x, c):
        """Forward of one training step with the backward attached as one autograd node."""
        names = self.trainable_names()
        return _LatteTrainFn.apply(self, names, x, c, *[self.params[n] for n in names])


class TrainEngine(_EngineBase):
    """The step of `Latte`, and of `LatteIMG` with `images` = I still frames per sample (latte_img.py:316-399)."""

    def __init__(self, model, ops, dtype, images=0, checkpoint=False):
        super().__init__(model, ops, dtype, images, checkpoint)
        m = model
        self.D, self.H, self.Fr, self.N = m.hidden_size, m.num_heads, m.num_frames, m.x_embedder.num_patches
        self.p, self.nblocks = m.patch_size, m.depth
        self.patch_conv, self.final_linear, self.pos_table = m.x_embedder.proj, m.final_layer.linear, m.pos_embed

    def _operands(self):
        """qkv, proj, fc1, fc2 of every block, then the adaLN weights of every block and the final layer in one operand."""
        m = self.m
        t = []
        for i, b in enumerate(m.blocks):
            for k, lin in (("qkv", b.attn.qkv), ("out", b.attn.proj), ("fc1", b.mlp.fc1), ("fc2", b.mlp.fc2)):
                t.append(((i, k), [lin.weight], [lin.bias]))
        ada = [b.adaLN_modulation[1] for b in m.blocks] + [m.final_layer.adaLN_modulation[1]]
        t.append(("ada", [a.weight for a in ada], [a.bias for a in ada]))
        return t

    def _modulation(self, ada, c, B):
        """mod = the stacked adaLN output, (B or B(F+I), depth*6D + 2D)."""
        return ada

    def _modulation_backward(self, dmod, S, grads):
        return dmod, ()

    def _temp_embed(self):
        return self.m.temp_embed.detach().float().reshape(self.Fr, self.D).contiguous()

    def _add_temp(self, xm, m2, g2, mod_t, B, temp):
        if not self.images:
            return super()._add_temp(xm, m2, g2, mod_t, B, temp)
        # temp_embed goes to the video rows only (latte_img.py:377-378).  All frames of a video share one gate row, so the
        # video rows take the per-video view, like a temporal block.
        _, Tv, rpb, rpb_t = self._geometry(B)
        g2v = mod_t[:, 5 * self.D:6 * self.D]
        return self._join_rows(self.ops.gate_residual(xm[:Tv], m2[:Tv], g2v, rpb_t, row_add=temp, tokens=self.N),
                               self.ops.gate_residual(xm[Tv:], m2[Tv:], g2[B * self.Fr:], rpb))


def trainable_names(model):
    """Names, in a fixed order, of the parameters the engine produces gradients for (everything except the embedders that
    feed `c`, whose few-kilobyte graph stays on torch autograd, and the frozen sin-cos tables)."""
    return TrainEngine(model, None, None).trainable_names()


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
    return TrainEngine(model, ops, dtype, images, checkpoint=model.gradient_checkpointing).train_forward(x, c)


def conditioning(model, t, y):
    """c = t_embedder(t) [+ y_embedder(y)] with torch autograd (latte.py:98-123 sincos + MLP, :148-153 table lookup): a
    (B, D) graph of a handful of kernels whose parameters get their gradients from `dc`."""
    c = _timestep_embedding(model, t)
    if model.extras == 2:
        c = c + model.y_embedder.embedding_table(y).float()
    return c


def _timestep_embedding(model, t):
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
