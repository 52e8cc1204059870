"""TEST INFRASTRUCTURE — torch restatement of the two ops the LatteT2V training engine (latte_b200/training_t2v.py) calls on top of
those of `train_ops_oracle.TorchOps`: the text cross-attention and its backward (diffusers Attention attn2 with the padded-prompt
bias, latte_t2v.py:766-771, 862-870).  fp32 math, one rounding at the output, like the kernels."""
from __future__ import annotations

import torch

from .train_ops_oracle import TorchOps


class T2VTorchOps(TorchOps):
    def to_operand(self, x32):
        """A fresh buffer, as b200_cast16 writes one: the engine accumulates into the fp32 residual after casting it."""
        return x32.to(self.dtype, copy=True)

    @staticmethod
    def _heads(q, kv, B, q_rows, L, H):
        D = q.shape[1]
        hd = D // H
        qh = q.float().reshape(B, q_rows, H, hd).transpose(1, 2)                  # (B, H, q_rows, hd)
        kvh = kv[: B * L].float().reshape(B, L, 2, H, hd)
        return qh, kvh[:, :, 0].transpose(1, 2), kvh[:, :, 1].transpose(1, 2), hd

    @staticmethod
    def _probs(qh, k, hd, key_bias, L):
        s = qh @ k.transpose(-1, -2) * hd ** -0.5
        if key_bias is not None:
            s = s + key_bias.float()[:, None, None, :L]
        return s.softmax(-1)

    def cross_attention(self, q, kv, B, q_rows, L, H, key_bias=None):
        qh, k, v, hd = self._heads(q, kv, B, q_rows, L, H)
        o = self._probs(qh, k, hd, key_bias, L) @ v
        return o.transpose(1, 2).reshape(q.shape).to(self.dtype)

    def cross_attention_bwd(self, q, kv, o, do, B, q_rows, L, H, key_bias, dkv, col0):
        qh, k, v, hd = self._heads(q, kv, B, q_rows, L, H)
        p = self._probs(qh, k, hd, key_bias, L)
        d_o = do.float().reshape(B, q_rows, H, hd).transpose(1, 2)
        delta = (d_o * o.float().reshape(B, q_rows, H, hd).transpose(1, 2)).sum(-1, keepdim=True)    # rowsum(dO . O)
        dv = p.transpose(-1, -2) @ d_o
        ds = p * (d_o @ v.transpose(-1, -2) - delta) * hd ** -0.5
        dq = ds @ k
        dk = ds.transpose(-1, -2) @ qh
        D = q.shape[1]
        dkv[: B * L, col0:col0 + 2 * D] = torch.cat((dk.transpose(1, 2).reshape(B * L, D), dv.transpose(1, 2).reshape(B * L, D)),
                                                    dim=1).to(dkv.dtype)
        return dq.transpose(1, 2).reshape(q.shape).to(self.dtype)
