"""TEST INFRASTRUCTURE — torch restatement of every op the training engine (latte_b200/training.py) calls on its backend.

Two uses, both from tests/ only:
  * CPU, fp32 "operands": the engine's ORCHESTRATION (saved activations, chain rule, per-sample reductions) driven through
    these ops must reproduce the gradients the unmodified reference produced (tests/golden/train_tiny64.npz);
  * GPU: each hand-written kernel of latte_b200/csrc/train.cu is compared with the op of the same name here on the same
    16-bit inputs (fp32 math, one rounding at the output, like the kernels).
Formulas follow the reference's forward (models/latte.py:28-29 modulate, :48-77 attention 'math', :169-181 block) and are
the analytic derivatives of those expressions; nothing here is shipped or called by the product path.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F


class TorchOps:
    """`dtype` = the engine's operand type (bf16/fp16 on the GPU, fp32 for the exact CPU check)."""

    def __init__(self, dtype=torch.float32):
        self.dtype = dtype

    # ------------------------------------------------------------------ forward ops
    def ln_modulate(self, x, shift, scale, rpb):
        B = x.shape[0] // rpb
        xf = x.float().view(B, rpb, -1)
        mu = xf.mean(-1, keepdim=True)
        var = ((xf - mu) ** 2).mean(-1, keepdim=True)
        xh = (xf - mu) / torch.sqrt(var + 1e-6)
        return (xh * (1 + scale.float()[:, None]) + shift.float()[:, None]).reshape(x.shape).to(self.dtype)

    def linear(self, a, w, bias=None, gelu=False):
        out = a.float() @ w.float().t()
        if bias is not None:
            out = out + bias.float()
        if gelu:
            out = F.gelu(out, approximate="tanh")
        return out.to(self.dtype)

    def linear_accum(self, out32, a, w, bias=None):
        r = a.float() @ w.float().t()
        if bias is not None:
            r = r + bias.float()
        out32 += r
        return out32

    def dgrad(self, dy, w):
        """dx [rows, n_in] = dy [rows, n_out] @ w [n_out, n_in]."""
        return (dy.float() @ w.float()).to(self.dtype)

    def linear_gelu_both(self, a, w, bias):
        u = self.linear(a, w, bias)
        return u, self.gelu(u)

    def wgrad(self, dW32, dy, x):
        """dW [n_out, n_in] += dy [rows, n_out]^T @ x [rows, n_in]."""
        dW32 += dy.float().t() @ x.float()
        return dW32

    @staticmethod
    def _split(qkv, B, Fr, N, H, temporal):
        T, D3 = qkv.shape
        hd = D3 // 3 // H
        t = qkv.float().view(B, Fr, N, 3, H, hd)
        if temporal:
            t = t.permute(3, 0, 2, 4, 1, 5).reshape(3, B * N, H, Fr, hd)      # (b n) h f d
        else:
            t = t.permute(3, 0, 1, 4, 2, 5).reshape(3, B * Fr, H, N, hd)      # (b f) h n d
        return t[0], t[1], t[2], hd

    @staticmethod
    def _merge(o, B, Fr, N, H, temporal):
        hd = o.shape[-1]
        if temporal:
            o = o.view(B, N, H, Fr, hd).permute(0, 3, 1, 2, 4)                # b f n h d
        else:
            o = o.view(B, Fr, H, N, hd).permute(0, 1, 3, 2, 4)
        return o.reshape(B * Fr * N, H * hd)

    def attention(self, qkv, B, Fr, N, H, temporal):
        q, k, v, hd = self._split(qkv, B, Fr, N, H, temporal)
        p = ((q @ k.transpose(-1, -2)) * hd ** -0.5).softmax(-1)
        return self._merge(p @ v, B, Fr, N, H, temporal).to(self.dtype)

    def gate_residual(self, x, m, gate, rpb, row_add=None, tokens=1):
        B = x.shape[0] // rpb
        out = x.view(B, rpb, -1) + gate.float()[:, None] * m.float().view(B, rpb, -1)
        if row_add is not None:                                              # row (b, f, n) gets row_add[f]
            Fr = row_add.shape[0]
            out = out.view(B, Fr, tokens, -1) + row_add.float()[None, :, None]
        return out.reshape(x.shape).contiguous()

    def gelu(self, u):
        return F.gelu(u.float(), approximate="tanh").to(self.dtype)

    # ------------------------------------------------------------------ backward ops
    # reduction outputs accumulate (+=) into the views handed in, like the kernels
    def gate_bwd(self, dx, m, gate, rpb, dgate, dbias):
        B = dx.shape[0] // rpb
        d = dx.view(B, rpb, -1)
        dm = d * gate.float()[:, None]
        dgate += (d * m.float().view(B, rpb, -1)).sum(1)
        dbias += dm.sum((0, 1))
        return dm.reshape(dx.shape).to(self.dtype)

    def gelu_bwd(self, da, u, dbias):
        uf = u.float()
        k0, k1 = math.sqrt(2.0 / math.pi), 0.044715
        th = torch.tanh(k0 * (uf + k1 * uf ** 3))
        dg = 0.5 * (1 + th) + 0.5 * uf * (1 - th * th) * k0 * (1 + 3 * k1 * uf * uf)
        du = da.float() * dg
        dbias += du.sum(0)
        return du.to(self.dtype)

    def ln_modulate_bwd(self, dh, x, shift, scale, rpb, dx, dshift, dscale):
        B = x.shape[0] // rpb
        xf = x.float().view(B, rpb, -1)
        mu = xf.mean(-1, keepdim=True)
        var = ((xf - mu) ** 2).mean(-1, keepdim=True)
        rstd = 1.0 / torch.sqrt(var + 1e-6)
        xh = (xf - mu) * rstd
        d = dh.float().view(B, rpb, -1)
        dshift += d.sum(1)
        dscale += (d * xh).sum(1)
        g = d * (1 + scale.float()[:, None])
        dxr = rstd * (g - g.mean(-1, keepdim=True) - xh * (g * xh).mean(-1, keepdim=True))
        dx += dxr.reshape(dx.shape)

    def attention_bwd(self, qkv, o, do, B, Fr, N, H, temporal):
        q, k, v, hd = self._split(qkv, B, Fr, N, H, temporal)
        sc = hd ** -0.5
        p = ((q @ k.transpose(-1, -2)) * sc).softmax(-1)
        T, D = do.shape
        d_o = do.float().view(B, Fr, N, H, hd)
        d_o = (d_o.permute(0, 2, 3, 1, 4).reshape(B * N, H, Fr, hd) if temporal
               else d_o.permute(0, 1, 3, 2, 4).reshape(B * Fr, H, N, hd))
        dv = p.transpose(-1, -2) @ d_o
        dp = d_o @ v.transpose(-1, -2)
        ds = p * (dp - (p * dp).sum(-1, keepdim=True)) * sc
        dq = ds @ k
        dk = ds.transpose(-1, -2) @ q
        parts = [self._merge(t, B, Fr, N, H, temporal) for t in (dq, dk, dv)]
        return torch.cat(parts, dim=1).to(self.dtype)

    def colsum(self, a, out):
        out += a.float().sum(0)
        return out

    def transpose(self, a):
        return a.t().contiguous()

    def cast(self, w32):
        return w32.detach().to(self.dtype).contiguous()

    def cast_into(self, srcs, dsts):
        for a, b in zip(srcs, dsts):
            b.copy_(a.detach())

    def to_operand(self, x32):
        return x32.to(self.dtype)

    def ada_outer(self, dmod, sc):
        """dW[n, k] = sum_b dmod[b, n] * sc[b, k]."""
        return dmod.float().t() @ sc.float()

    def ada_dsc(self, dmod, w):
        """dsc[b, k] = sum_n dmod[b, n] * w[n, k]."""
        return dmod.float() @ w.float()
