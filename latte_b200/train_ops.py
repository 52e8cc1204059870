"""Native backend of the training engines (latte_b200.training.TrainEngine, training_t2v.T2VTrainEngine): every op is a
latte_b200.ops call into liblatte_b200.so (csrc/train.cu for the backward passes and the cross-attention, the wgmma GEMM /
attention / LayerNorm kernels of the sampling path for the rest).  What lives here is the routing: operands in one 16-bit
type, shapes the GEMM kernels do not take sent through zero rows or transposes, small adaLN batches to their own passes, and
the buffers reused across calls.  CUDA only — a CPU tensor raises; the torch restatements of the same ops live in
oracle/train_ops_oracle.py and oracle/train_t2v_ops_oracle.py and are test infrastructure."""
from __future__ import annotations

import torch

from . import ops


class NativeOps:
    def __init__(self, dtype=torch.bfloat16):
        if dtype not in (torch.float16, torch.bfloat16):
            raise TypeError("NativeOps computes in float16 or bfloat16")
        self.dtype = dtype
        self._ones = {}
        self._xattn_ws = None

    def _unit_gate(self, n, dev):
        g = self._ones.get((n, dev))
        if g is None:
            g = self._ones[(n, dev)] = torch.ones(1, n, dtype=torch.float32, device=dev)
        return g

    # ------------------------------------------------------------------ forward ops
    def ln_modulate(self, x, shift, scale, rpb):
        return ops.ln_modulate(x, shift, scale, rpb, self.dtype)

    def linear(self, a, w, bias=None, gelu=False):
        return ops.linear(a, w, bias, gelu=gelu)

    def linear_accum(self, out32, a, w, bias=None):
        """out32 [M, N] += a [M, K] @ w [N, K]^T (+ bias): the GEMM's residual epilogue with a unit gate (ordered stream-K)."""
        return ops.linear_gate_residual_(out32, a, w, bias, self._unit_gate(out32.shape[1], out32.device), max(out32.shape[0], 1))

    def wgrad(self, dW32, dy, x):
        """dW32 [n_out, n_in] += dy [rows, n_out]^T @ x [rows, n_in]: the GEMM reads both activations untransposed (MN-major
        operand mode); shapes it does not take (n_in not a multiple of 128) go through explicit 16-bit transposes.  rows is
        the GEMM's K: a count that is not a multiple of 64 (patch 4 and 8 give 16 or 4 tokens per frame) gets zero rows."""
        rows, n_out = dy.shape
        n_in = x.shape[1]
        if rows % 64:
            pad = 64 - rows % 64
            dy, x = torch.cat((dy, dy.new_zeros(pad, n_out))), torch.cat((x, x.new_zeros(pad, n_in)))
            rows += pad
        if n_in % 128 == 0 and n_out % 8 == 0 and rows % 64 == 0:
            return ops.wgrad(dW32, dy, x, self._unit_gate(n_in, dy.device))
        return self.linear_accum(dW32, self.transpose(dy), self.transpose(x))

    def dgrad(self, dy, w):
        """dx [rows, n_in] = dy [rows, n_out] @ w [n_out, n_in] with the weight in its nn.Linear layout (MN-major W operand)."""
        if w.shape[1] % 128 == 0 and dy.shape[1] % 64 == 0:
            return ops.dgrad(dy, w)
        return self.linear(dy, self.transpose(w))

    def linear_gelu_both(self, a, w, bias):
        """(u, gelu_tanh(u)) with u = a @ w^T + bias, both from one GEMM epilogue (training-mode fc1)."""
        return ops.linear_gelu_both(a, w, bias)

    def attention(self, qkv, B, Fr, N, H, temporal):
        return ops.attention(qkv, B, Fr, N, H, temporal)

    def gate_residual(self, x, m, gate, rpb, row_add=None, tokens=1):
        return ops.gate_residual(x, m, gate, rpb, row_add, tokens)

    # ------------------------------------------------------------------ backward ops
    # Reduction outputs (dgate, dbias, dshift, dscale, column sums) ACCUMULATE into the fp32 views the engine hands in -- slices of
    # gradient buffers it zeroed once for the step -- so no pass needs a memset or a copy of its result.
    def gate_bwd(self, dx, m, gate, rpb, dgate, dbias):
        return ops.gate_bwd(dx, m, gate, rpb, dgate, dbias)

    def gelu_bwd(self, da, u, dbias):
        return ops.gelu_bwd(da, u, dbias)

    def ln_modulate_bwd(self, dh, x, shift, scale, rpb, dx, dshift, dscale):
        ops.ln_modulate_bwd(dh, x, scale, rpb, dx, dshift, dscale)

    def attention_bwd(self, qkv, o, do, B, Fr, N, H, temporal):
        return ops.attention_bwd(qkv, o, do, B, Fr, N, H, temporal)

    def cross_attention(self, q, kv, B, q_rows, L, H, key_bias=None):
        """Text cross-attention: q [B*q_rows, H*hd]; kv a column window [>= B*L, 2*H*hd] of the stacked K/V of all layers."""
        return ops.cross_attention(q, kv, B, q_rows, L, H, key_bias)

    def cross_attention_bwd(self, q, kv, o, do, B, q_rows, L, H, key_bias, dkv, col0):
        """Backward of `cross_attention`: returns dq; dK | dV go to dkv[:B*L, col0:col0 + 2*H*hd] (dkv 16-bit, row-major)."""
        need = ops.workspace_bytes("b200_cross_attention_bwd_workspace_bytes", B, q_rows, L, H, q.shape[1] // H)
        ws = self._xattn_ws
        if ws is None or ws.numel() < need or ws.device != q.device:   # reused by every layer, in stream order
            ws = self._xattn_ws = torch.empty(need, dtype=torch.uint8, device=q.device)
        return ops.cross_attention_bwd(q, kv, o, do, B, q_rows, L, H, key_bias, dkv, col0, ws)

    def colsum(self, a, out):
        return ops.colsum(a, out)

    def transpose(self, a):
        assert a.dtype == self.dtype
        return ops.transpose16(a)

    def cast(self, w32):
        """A fresh 16-bit copy of a parameter."""
        return self.to_operand(w32.detach().float())

    def cast_into(self, srcs, dsts):
        """dsts[i] (16-bit, contiguous) = srcs[i] (fp32, contiguous) for all i in ONE launch; the pointer table is cached for as
        long as the tensors stay where they are (parameters are updated in place by the optimizers)."""
        assert all(b.dtype == self.dtype for b in dsts)
        ops.multi_cast(srcs, dsts)

    def to_operand(self, x32):
        x32 = x32.contiguous()
        return ops.cast16(x32, torch.empty(x32.shape, dtype=self.dtype, device=x32.device))

    # adaLN gradients, dW = dmod^T silu(c) and dsc = dmod W_ada.  Up to 8 rows (per-sample conditioning at a small local batch)
    # they are one pass each over the stacked weight (b200_ada_outer / b200_ada_dsc).  More rows (a large local batch, or one row
    # per frame in video + image training) go through the weight-gradient GEMM: dmod rounded to the operand type (what the
    # reference computes under bf16 autocast) and zero-padded to a multiple of 64 rows, fp32 reduce-add into the result.
    _ADA_ROWS = 8

    def _ada_rows16(self, dmod):
        """dmod fp32 (R, NA) -> 16-bit (R', NA), R' = R rounded up to 64 with zero rows."""
        R, NA = dmod.shape
        return ops.cast16(dmod.contiguous(), torch.zeros((R + 63) // 64 * 64, NA, dtype=self.dtype, device=dmod.device))

    def ada_outer(self, dmod, sc):
        if dmod.shape[0] > self._ADA_ROWS:
            R, D = sc.shape
            d16 = self._ada_rows16(dmod)
            sc16 = torch.zeros(d16.shape[0], D, dtype=self.dtype, device=sc.device)
            sc16[:R] = sc
            return self.wgrad(torch.zeros(dmod.shape[1], D, dtype=torch.float32, device=dmod.device), d16, sc16)
        return ops.ada_outer(dmod, sc)

    def ada_dsc(self, dmod, w):
        if dmod.shape[0] > self._ADA_ROWS:
            # dsc^T is the weight gradient of the (NA x R') operand dmod^T against W_ada: K = NA, a long-K few-tile GEMM that the
            # stream-K schedule spreads over all SMs
            d16 = self._ada_rows16(dmod)
            dsc = torch.zeros(d16.shape[0], w.shape[1], dtype=torch.float32, device=dmod.device)
            return self.wgrad(dsc, self.transpose(d16), w)[: dmod.shape[0]]
        return ops.ada_dsc(dmod, w)
