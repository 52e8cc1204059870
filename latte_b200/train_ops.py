"""Native backend of the training engines (latte_b200.training.TrainEngine, training_t2v.T2VTrainEngine): every op is one
C-ABI call into liblatte_b200.so (csrc/train.cu for the backward passes and the cross-attention, the wgmma GEMM / attention /
LayerNorm kernels of the sampling path for the rest).  CUDA only — a CPU tensor raises; the torch restatements of the same
ops live in oracle/train_ops_oracle.py and oracle/train_t2v_ops_oracle.py and are test infrastructure."""
from __future__ import annotations

import torch

from . import _lib, ops

_KIND = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}


def _s(t):
    return torch.cuda.current_stream(t.device).cuda_stream


class NativeOps:
    def __init__(self, dtype=torch.bfloat16):
        if dtype not in (torch.float16, torch.bfloat16):
            raise TypeError("NativeOps computes in float16 or bfloat16")
        self.dtype = dtype
        self.dt = _lib.BF16 if dtype == torch.bfloat16 else _lib.FP16
        self._ones = {}

    def _unit_gate(self, n, dev):
        g = self._ones.get((n, dev))
        if g is None:
            g = self._ones[(n, dev)] = torch.ones(1, n, dtype=torch.float32, device=dev)
        return g

    @staticmethod
    def _cuda(*ts):
        for t in ts:
            if t is not None and not t.is_cuda:
                raise RuntimeError("latte_b200 training ops run on CUDA (sm_90a) only; there is no CPU fallback")

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
        self._cuda(dW32, dy, x)
        rows, n_out = dy.shape
        n_in = x.shape[1]
        if rows % 64:
            pad = 64 - rows % 64
            dy, x = torch.cat((dy, dy.new_zeros(pad, n_out))), torch.cat((x, x.new_zeros(pad, n_in)))
            rows += pad
        if n_in % 128 == 0 and n_out % 8 == 0 and rows % 64 == 0:
            assert dy.is_contiguous() and x.is_contiguous() and dW32.is_contiguous() and dW32.dtype == torch.float32
            with torch.cuda.device(dy.device):
                rc = _lib.load().b200_wgrad(dy.data_ptr(), x.data_ptr(), self._unit_gate(n_in, dy.device).data_ptr(), dW32.data_ptr(),
                                            rows, n_out, n_in, self.dt, ops._sk_flags(dy.device).data_ptr(), _s(dy))
            _lib.check(rc, "b200_wgrad")
            return dW32
        return self.linear_accum(dW32, self.transpose(dy), self.transpose(x))

    def dgrad(self, dy, w):
        """dx [rows, n_in] = dy [rows, n_out] @ w [n_out, n_in] with the weight in its nn.Linear layout (MN-major W operand)."""
        self._cuda(dy, w)
        rows, n_out = dy.shape
        n_in = w.shape[1]
        if n_in % 128 == 0 and n_out % 64 == 0:
            assert dy.is_contiguous() and w.is_contiguous() and dy.dtype == w.dtype
            dx = torch.empty(rows, n_in, dtype=dy.dtype, device=dy.device)
            with torch.cuda.device(dy.device):
                rc = _lib.load().b200_dgrad(dy.data_ptr(), w.data_ptr(), dx.data_ptr(), rows, n_out, n_in, self.dt, _s(dy))
            _lib.check(rc, "b200_dgrad")
            return dx
        return self.linear(dy, self.transpose(w))

    def linear_gelu_both(self, a, w, bias):
        """(u, gelu_tanh(u)) with u = a @ w^T + bias, both from one GEMM epilogue (training-mode fc1)."""
        self._cuda(a, w, bias)
        assert a.is_contiguous() and w.is_contiguous() and a.dtype == w.dtype
        M, K = a.shape
        N = w.shape[0]
        u = torch.empty(M, N, dtype=a.dtype, device=a.device)
        act = torch.empty(M, N, dtype=a.dtype, device=a.device)
        with torch.cuda.device(a.device):
            rc = _lib.load().b200_linear_gelu_both(a.data_ptr(), w.data_ptr(), bias.data_ptr() if bias is not None else None, M, N, K, self.dt,
                                                   u.data_ptr(), act.data_ptr(), _s(a))
        _lib.check(rc, "b200_linear_gelu_both")
        return u, act

    def attention(self, qkv, B, Fr, N, H, temporal):
        return ops.attention(qkv, B, Fr, N, H, temporal)

    def gate_residual(self, x, m, gate, rpb, row_add=None, tokens=1):
        self._cuda(x, m, gate, row_add)
        assert x.dtype == torch.float32 and x.is_contiguous() and m.is_contiguous() and gate.stride(1) == 1
        out = torch.empty_like(x)
        frames = row_add.shape[0] if row_add is not None else 0
        with torch.cuda.device(x.device):
            rc = _lib.load().b200_gate_residual(x.data_ptr(), m.data_ptr(), gate.data_ptr(), gate.stride(0), rpb,
                                                row_add.data_ptr() if row_add is not None else None, tokens, frames,
                                                out.data_ptr(), x.shape[0], x.shape[1], self.dt, _s(x))
        _lib.check(rc, "b200_gate_residual")
        return out

    # ------------------------------------------------------------------ backward ops
    # Reduction outputs (dgate, dbias, dshift, dscale, column sums) ACCUMULATE into the fp32 views the engine hands in -- slices of
    # gradient buffers it zeroed once for the step -- so no pass needs a memset or a copy of its result.
    def gate_bwd(self, dx, m, gate, rpb, dgate, dbias):
        self._cuda(dx, m, gate, dgate, dbias)
        assert dx.dtype == torch.float32 and dx.is_contiguous() and m.is_contiguous() and dgate.stride(1) == 1
        T, D = dx.shape
        dm = torch.empty(T, D, dtype=self.dtype, device=dx.device)
        with torch.cuda.device(dx.device):
            rc = _lib.load().b200_gate_bwd(dx.data_ptr(), m.data_ptr(), gate.data_ptr(), gate.stride(0), rpb, dm.data_ptr(),
                                           dgate.data_ptr(), dgate.stride(0), dbias.data_ptr(), T, D, self.dt, _s(dx))
        _lib.check(rc, "b200_gate_bwd")
        return dm

    def gelu_bwd(self, da, u, dbias):
        self._cuda(da, u, dbias)
        T, D = u.shape
        du = torch.empty_like(u)
        with torch.cuda.device(u.device):
            rc = _lib.load().b200_gelu_bwd(da.data_ptr(), u.data_ptr(), du.data_ptr(), dbias.data_ptr(), T, D, self.dt, _s(u))
        _lib.check(rc, "b200_gelu_bwd")
        return du

    def ln_modulate_bwd(self, dh, x, shift, scale, rpb, dx, dshift, dscale):
        self._cuda(dh, x, scale, dx, dshift, dscale)
        assert dshift.stride(0) == dscale.stride(0) and dshift.stride(1) == 1
        T, D = x.shape
        with torch.cuda.device(x.device):
            rc = _lib.load().b200_ln_modulate_bwd(dh.data_ptr(), x.data_ptr(), scale.data_ptr(), scale.stride(0), rpb, dx.data_ptr(),
                                                  dshift.data_ptr(), dscale.data_ptr(), dshift.stride(0), T, D, self.dt, _s(x))
        _lib.check(rc, "b200_ln_modulate_bwd")

    def attention_bwd(self, qkv, o, do, B, Fr, N, H, temporal):
        self._cuda(qkv, o, do)
        D = o.shape[1]
        dqkv = torch.empty_like(qkv)
        # row statistics (lse, delta) of the two-kernel backward: spatial sequences and temporal ones longer than 16 frames;
        # the <= 16-frame temporal kernel keeps them in shared memory
        stats = None if temporal and Fr <= 16 else torch.empty(2 * B * Fr * H * N, dtype=torch.float32, device=qkv.device)
        with torch.cuda.device(qkv.device):
            rc = _lib.load().b200_attention_bwd(qkv.data_ptr(), o.data_ptr(), do.data_ptr(), dqkv.data_ptr(),
                                                stats.data_ptr() if stats is not None else None, B, Fr, N, H, D // H, self.dt,
                                                int(temporal), _s(qkv))
        _lib.check(rc, "b200_attention_bwd")
        return dqkv

    def cross_attention(self, q, kv, B, q_rows, L, H, key_bias=None):
        """Text cross-attention (b200_cross_attention): q [B*q_rows, H*hd]; kv a row-major view [>= B*L, 2*H*hd] ([k | v]
        heads, any row stride: a column window of the stacked K/V of all layers); key_bias None or fp32 [B, 128]."""
        self._cuda(q, kv, key_bias)
        assert q.is_contiguous() and kv.stride(1) == 1 and q.dtype == kv.dtype == self.dtype
        D = q.shape[1]
        out = torch.empty_like(q)
        with torch.cuda.device(q.device):
            rc = _lib.load().b200_cross_attention(q.data_ptr(), kv.data_ptr(), key_bias.data_ptr() if key_bias is not None else None,
                                                  out.data_ptr(), B, q_rows, L, q.stride(0), kv.stride(0), H, D // H, self.dt, _s(q))
        _lib.check(rc, "b200_cross_attention")
        return out

    def cross_attention_bwd(self, q, kv, o, do, B, q_rows, L, H, key_bias, dkv, col0):
        """Backward of `cross_attention`: returns dq; dK | dV go to dkv[:B*L, col0:col0 + 2*H*hd] (dkv 16-bit, row-major)."""
        self._cuda(q, kv, o, do, key_bias, dkv)
        assert q.is_contiguous() and o.is_contiguous() and do.is_contiguous() and kv.stride(1) == 1 and dkv.stride(1) == 1
        D = q.shape[1]
        lib = _lib.load()
        need = lib.b200_cross_attention_bwd_workspace_bytes(B, q_rows, L, H, D // H)
        if need == 0:
            raise RuntimeError("b200_cross_attention_bwd: unsupported shape: " + _lib.last_error())
        ws = getattr(self, "_xattn_ws", None)
        if ws is None or ws.numel() < need or ws.device != q.device:   # reused by every layer, in stream order
            ws = self._xattn_ws = torch.empty(need, dtype=torch.uint8, device=q.device)
        dq = torch.empty_like(q)
        with torch.cuda.device(q.device):
            rc = lib.b200_cross_attention_bwd(q.data_ptr(), kv.data_ptr(), key_bias.data_ptr() if key_bias is not None else None,
                                              o.data_ptr(), do.data_ptr(), dq.data_ptr(), dkv.data_ptr(), dkv.stride(0), col0, B, q_rows,
                                              L, q.stride(0), kv.stride(0), H, D // H, self.dt, ws.data_ptr(), ws.numel(), _s(q))
        _lib.check(rc, "b200_cross_attention_bwd")
        return dq

    def colsum(self, a, out):
        self._cuda(a, out)
        assert a.is_contiguous() and out.is_contiguous() and out.dtype == torch.float32
        with torch.cuda.device(a.device):
            rc = _lib.load().b200_colsum(a.data_ptr(), _KIND[a.dtype], out.data_ptr(), a.shape[0], a.shape[1], _s(a))
        _lib.check(rc, "b200_colsum")
        return out

    def transpose(self, a):
        self._cuda(a)
        assert a.is_contiguous() and a.dtype == self.dtype
        out = torch.empty(a.shape[1], a.shape[0], dtype=a.dtype, device=a.device)
        with torch.cuda.device(a.device):
            rc = _lib.load().b200_transpose16(a.data_ptr(), out.data_ptr(), a.shape[0], a.shape[1], _s(a))
        _lib.check(rc, "b200_transpose16")
        return out

    def cast(self, w32):
        """A fresh 16-bit copy of a parameter."""
        return self.to_operand(w32.detach().float())

    def cast_into(self, srcs, dsts):
        """dsts[i] (16-bit, contiguous) = srcs[i] (fp32, contiguous) for all i in ONE launch; the pointer table is cached for as
        long as the tensors stay where they are (parameters are updated in place by the optimizers)."""
        key = tuple(t.data_ptr() for t in srcs) + tuple(t.data_ptr() for t in dsts)
        st = getattr(self, "_mc", None)
        if st is None or st[0] != key:
            rows, first = [], 0
            for a, b in zip(srcs, dsts):
                self._cuda(a, b)
                assert a.dtype == torch.float32 and b.dtype == self.dtype and a.is_contiguous() and b.is_contiguous()
                assert a.numel() == b.numel() and a.numel() % 4 == 0 and a.data_ptr() % 16 == 0 and b.data_ptr() % 8 == 0
                n4 = a.numel() // 4
                rows.append([a.data_ptr(), b.data_ptr(), n4, first])
                first += (n4 + 1023) // 1024
            table = torch.tensor(rows, dtype=torch.int64).to(srcs[0].device)
            st = self._mc = (key, table, first, len(rows))
        _, table, total, n = st
        with torch.cuda.device(table.device):
            rc = _lib.load().b200_multi_cast(table.data_ptr(), n, total, self.dt, _s(table))
        _lib.check(rc, "b200_multi_cast")

    def to_operand(self, x32):
        self._cuda(x32)
        x32 = x32.contiguous()
        out = torch.empty(x32.shape, dtype=self.dtype, device=x32.device)
        with torch.cuda.device(x32.device):
            rc = _lib.load().b200_cast16(x32.data_ptr(), out.data_ptr(), x32.numel(), self.dt, _s(x32))
        _lib.check(rc, "b200_cast16")
        return out

    # adaLN gradients, dW = dmod^T silu(c) and dsc = dmod W_ada.  Up to 8 rows (per-sample conditioning at a small local batch)
    # they are one pass each over the stacked weight (b200_ada_outer / b200_ada_dsc).  More rows (a large local batch, or one row
    # per frame in video + image training) go through the weight-gradient GEMM: dmod rounded to the operand type (what the
    # reference computes under bf16 autocast) and zero-padded to a multiple of 64 rows, fp32 reduce-add into the result.
    _ADA_ROWS = 8

    def _ada_rows16(self, dmod):
        """dmod fp32 (R, NA) -> 16-bit (R', NA), R' = R rounded up to 64 with zero rows."""
        R, NA = dmod.shape
        d16 = torch.zeros((R + 63) // 64 * 64, NA, dtype=self.dtype, device=dmod.device)
        with torch.cuda.device(dmod.device):
            rc = _lib.load().b200_cast16(dmod.contiguous().data_ptr(), d16.data_ptr(), R * NA, self.dt, _s(dmod))
        _lib.check(rc, "b200_cast16")
        return d16

    def ada_outer(self, dmod, sc):
        self._cuda(dmod, sc)
        if dmod.shape[0] > self._ADA_ROWS:
            R, D = sc.shape
            d16 = self._ada_rows16(dmod)
            sc16 = torch.zeros(d16.shape[0], D, dtype=self.dtype, device=sc.device)
            sc16[:R] = sc
            return self.wgrad(torch.zeros(dmod.shape[1], D, dtype=torch.float32, device=dmod.device), d16, sc16)
        B, NA = dmod.shape
        D = sc.shape[1]
        dW = torch.empty(NA, D, dtype=torch.float32, device=dmod.device)
        with torch.cuda.device(dmod.device):
            rc = _lib.load().b200_ada_outer(dmod.data_ptr(), dmod.stride(0), sc.data_ptr(), dW.data_ptr(), B, NA, D, self.dt, _s(dmod))
        _lib.check(rc, "b200_ada_outer")
        return dW

    def ada_dsc(self, dmod, w):
        self._cuda(dmod, w)
        if dmod.shape[0] > self._ADA_ROWS:
            # dsc^T is the weight gradient of the (NA x R') operand dmod^T against W_ada: K = NA, a long-K few-tile GEMM that the
            # stream-K schedule spreads over all SMs
            d16 = self._ada_rows16(dmod)
            dsc = torch.zeros(d16.shape[0], w.shape[1], dtype=torch.float32, device=dmod.device)
            return self.wgrad(dsc, self.transpose(d16), w)[: dmod.shape[0]]
        B, NA = dmod.shape
        D = w.shape[1]
        dsc = torch.empty(B, D, dtype=torch.float32, device=dmod.device)
        with torch.cuda.device(dmod.device):
            rc = _lib.load().b200_ada_dsc(dmod.data_ptr(), dmod.stride(0), w.data_ptr(), dsc.data_ptr(), B, NA, D, self.dt, _s(dmod))
        _lib.check(rc, "b200_ada_dsc")
        return dsc
