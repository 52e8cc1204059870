"""Torch-tensor wrappers over the C ABI: the one module that calls liblatte_b200.so.  `call` runs an entry point on a
tensor's device and current stream and raises on its error code; the per-op functions below pass device pointers and
nothing else.  The modules (Latte, LatteT2V, T5, the VAE), the sampler and the training backend all go through here."""
from __future__ import annotations

from collections import OrderedDict

import torch

from . import _lib


def call(name: str, device, *args) -> None:
    """Entry point `name` of the library on `device`, with that device's current stream appended as the last argument."""
    with torch.cuda.device(device):
        rc = getattr(_lib.load(), name)(*args, torch.cuda.current_stream(device).cuda_stream)
    _lib.check(rc, name)


def workspace_bytes(name: str, *args) -> int:
    """A size query of the library (`b200_*_bytes`); 0 means it does not take the shape, which raises with its reason."""
    need = getattr(_lib.load(), name)(*args)
    if need == 0:
        raise RuntimeError(f"{name}: unsupported shape: {_lib.last_error()}")
    return need


def scratch(need: int, device) -> tuple[torch.Tensor, int]:
    """`need` bytes of device scratch on the 1024-byte boundary the library's workspaces need: (owning buffer, address)."""
    ws = torch.empty(need + 1024, dtype=torch.uint8, device=device)
    return ws, (ws.data_ptr() + 1023) // 1024 * 1024


def _dt(t: torch.Tensor) -> int:
    """The library's 16-bit operand code of `t`."""
    if t.dtype == torch.float16:
        return _lib.FP16
    if t.dtype == torch.bfloat16:
        return _lib.BF16
    raise TypeError(f"expected a float16/bfloat16 tensor, got {t.dtype}")


_KINDS = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}


def _kind(t: torch.Tensor) -> int:
    """The f32 / f16 / bf16 code of the entry points that read any of the three."""
    if t.dtype not in _KINDS:
        raise TypeError(f"expected a float32/float16/bfloat16 tensor, got {t.dtype}")
    return _KINDS[t.dtype]


def _stream(t: torch.Tensor):
    return torch.cuda.current_stream(t.device).cuda_stream


def _ptr(t: torch.Tensor | None):
    return t.data_ptr() if t is not None else None


_SK_FLAGS = {}


def _sk_flags(device):
    """Per-device stream-K ordering flags for `b200_linear` (zeroed once; every launch leaves them zero, include/latte_b200.h)."""
    buf = _SK_FLAGS.get(device)
    if buf is None:
        buf = _SK_FLAGS[device] = torch.zeros(_lib.GEMM_SK_FLAGS, dtype=torch.int64, device=device)
    return buf


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError("latte_b200.ops run on CUDA (sm_90a) only; there is no CPU fallback")


def linear(a: torch.Tensor, w: torch.Tensor, bias: torch.Tensor | None = None, gelu: bool = False,
           block_n: int = 0) -> torch.Tensor:
    """out16 = (gelu_tanh)(a @ w.T + bias); a [M,K], w [N,K] 16-bit, bias fp32."""
    _need_cuda(a, w, bias)
    assert a.dtype == w.dtype and a.is_contiguous() and w.is_contiguous()
    M, K = a.shape
    N = w.shape[0]
    out = torch.empty(M, N, dtype=a.dtype, device=a.device)
    call("b200_linear", a.device, a.data_ptr(), w.data_ptr(), _ptr(bias), M, N, K, _dt(a),
         _lib.EPI_BIAS_GELU if gelu else _lib.EPI_BIAS, out.data_ptr(), None, None, 0, 1, block_n, None)
    return out


def linear_gate_residual_(resid: torch.Tensor, a: torch.Tensor, w: torch.Tensor, bias: torch.Tensor | None,
                          gate: torch.Tensor, rows_per_batch: int, block_n: int = 0, stream_k: bool = True) -> torch.Tensor:
    """resid (fp32 [M,N], in place) += gate[row // rows_per_batch] * (a @ w.T + bias); gate fp32 [B, N].
    stream_k=False withholds the flag buffer, which keeps the data-parallel schedule (one add per element)."""
    _need_cuda(resid, a, w, bias, gate)
    assert resid.dtype == torch.float32 and gate.dtype == torch.float32 and resid.is_contiguous()
    assert gate.stride(-1) == 1
    M, K = a.shape
    N = w.shape[0]
    call("b200_linear", a.device, a.data_ptr(), w.data_ptr(), _ptr(bias), M, N, K, _dt(a), _lib.EPI_GATE_RESIDUAL, None,
         resid.data_ptr(), gate.data_ptr(), gate.stride(0), rows_per_batch, block_n,
         _sk_flags(a.device).data_ptr() if stream_k else None)
    return resid


def attention(qkv: torch.Tensor, batch: int, frames: int, tokens: int, heads: int, temporal: bool) -> torch.Tensor:
    """qkv [batch*frames*tokens, 3*heads*hd] 16-bit -> out [T, heads*hd] 16-bit."""
    _need_cuda(qkv)
    assert qkv.is_contiguous() and qkv.shape[0] == batch * frames * tokens
    D = qkv.shape[1] // 3
    out = torch.empty(qkv.shape[0], D, dtype=qkv.dtype, device=qkv.device)
    call("b200_attention", qkv.device, qkv.data_ptr(), out.data_ptr(), batch, frames, tokens, heads, D // heads, _dt(qkv),
         int(temporal))
    return out


def spatial_attention_any(qkv: torch.Tensor, batch: int, frames: int, tokens: int, heads: int) -> torch.Tensor:
    """Spatial attention at any number of tokens per frame (b200_spatial_attention_any): qkv [batch*frames*tokens,
    3*heads*hd] 16-bit -> out [T, heads*hd] 16-bit."""
    _need_cuda(qkv)
    assert qkv.is_contiguous() and qkv.shape[0] == batch * frames * tokens
    D = qkv.shape[1] // 3
    out = torch.empty(qkv.shape[0], D, dtype=qkv.dtype, device=qkv.device)
    call("b200_spatial_attention_any", qkv.device, qkv.data_ptr(), out.data_ptr(), batch, frames, tokens, heads, D // heads,
         _dt(qkv))
    return out


def ln_modulate(x: torch.Tensor, shift: torch.Tensor, scale: torch.Tensor, rows_per_batch: int,
                dtype: torch.dtype = torch.float16) -> torch.Tensor:
    """x fp32 [rows, D]; shift/scale fp32 [B, D] (row stride arbitrary) -> 16-bit [rows, D]."""
    _need_cuda(x, shift, scale)
    assert x.dtype == torch.float32 and x.is_contiguous() and shift.stride(0) == scale.stride(0)
    out = torch.empty(x.shape, dtype=dtype, device=x.device)
    call("b200_ln_modulate", x.device, x.data_ptr(), shift.data_ptr(), scale.data_ptr(), shift.stride(0), rows_per_batch,
         out.data_ptr(), x.shape[0], x.shape[1], _dt(out))
    return out


def quantize_rows_e4m3(w: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """w fp32 [rows, cols] -> (q [rows, cols] float8_e4m3fn, scales fp32 [rows]): s = amax(|row|) / 448 (1 for a zero row),
    q = e4m3_rn_satfinite(row / s) (b200_quantize_rows_e4m3)."""
    _need_cuda(w)
    assert w.dtype == torch.float32 and w.dim() == 2 and w.is_contiguous()
    q = torch.empty(w.shape, dtype=torch.uint8, device=w.device)
    s = torch.empty(w.shape[0], dtype=torch.float32, device=w.device)
    call("b200_quantize_rows_e4m3", w.device, w.data_ptr(), w.shape[0], w.shape[1], q.data_ptr(), s.data_ptr())
    return q.view(torch.float8_e4m3fn), s


def ln_modulate_e4m3(x: torch.Tensor, shift: torch.Tensor, scale: torch.Tensor,
                     rows_per_batch: int) -> tuple[torch.Tensor, torch.Tensor]:
    """ln_modulate quantized per row: x fp32 [rows, D] -> (q [rows, D] float8_e4m3fn, row scales fp32 [rows])."""
    _need_cuda(x, shift, scale)
    assert x.dtype == torch.float32 and x.is_contiguous() and shift.stride(0) == scale.stride(0)
    q = torch.empty(x.shape, dtype=torch.uint8, device=x.device)
    s = torch.empty(x.shape[0], dtype=torch.float32, device=x.device)
    call("b200_ln_modulate_e4m3", x.device, x.data_ptr(), shift.data_ptr(), scale.data_ptr(), shift.stride(0), rows_per_batch,
         q.data_ptr(), s.data_ptr(), x.shape[0], x.shape[1])
    return q.view(torch.float8_e4m3fn), s


def linear_e4m3(a8: torch.Tensor, a_scale: torch.Tensor, w8: torch.Tensor, w_scale: torch.Tensor,
                bias: torch.Tensor | None = None, gelu: bool = False, dtype: torch.dtype = torch.float16) -> torch.Tensor:
    """out16 = (gelu_tanh)(a_scale[:, None] * w_scale[None, :] * (a8 @ w8.T) + bias) in `dtype`; a8 [M, K], w8 [N, K] e4m3
    (float8_e4m3fn or its uint8 bytes), scales and bias fp32 (b200_linear_e4m3)."""
    _need_cuda(a8, a_scale, w8, w_scale, bias)
    assert a8.element_size() == 1 and w8.element_size() == 1 and a8.is_contiguous() and w8.is_contiguous()
    assert a_scale.dtype == w_scale.dtype == torch.float32 and a_scale.is_contiguous() and w_scale.is_contiguous()
    M, K = a8.shape
    N = w8.shape[0]
    out = torch.empty(M, N, dtype=dtype, device=a8.device)
    call("b200_linear_e4m3", a8.device, a8.data_ptr(), a_scale.data_ptr(), w8.data_ptr(), w_scale.data_ptr(), _ptr(bias),
         M, N, K, _dt(out), _lib.EPI_BIAS_GELU if gelu else _lib.EPI_BIAS, out.data_ptr())
    return out


def cross_attention(q: torch.Tensor, kv: torch.Tensor, batch: int, q_rows_per_batch: int, kv_len: int, heads: int,
                    key_bias: torch.Tensor | None = None) -> torch.Tensor:
    """q [batch*q_rows, heads*hd] 16-bit; kv a row-major view [>= batch*kv_len, 2*heads*hd] 16-bit ([k | v] heads, any row
    stride: a contiguous kv, or a column window of the stacked K/V of all layers); kv_len <= 128 -> out like q.
    key_bias: optional fp32 [batch, 128] additive score bias per key (columns >= kv_len ignored)."""
    _need_cuda(q, kv, key_bias)
    assert q.is_contiguous() and kv.stride(1) == 1 and q.dtype == kv.dtype
    if key_bias is not None:
        assert key_bias.dtype == torch.float32 and key_bias.is_contiguous() and tuple(key_bias.shape) == (batch, 128)
    D = q.shape[1]
    out = torch.empty_like(q)
    call("b200_cross_attention", q.device, q.data_ptr(), kv.data_ptr(), _ptr(key_bias), out.data_ptr(), batch,
         q_rows_per_batch, kv_len, q.stride(0), kv.stride(0), heads, D // heads, _dt(q))
    return out


_VAE_CONV_KINDS = {"3x3": _lib.VAE_CONV3X3, "t3": _lib.VAE_CONV_T3, "down2": _lib.VAE_CONV_DOWN2}


def vae_conv(x: torch.Tensor, w16: torch.Tensor, bias: torch.Tensor | None, kind: str = "3x3",
             add16: torch.Tensor | None = None) -> torch.Tensor:
    """One VAE convolution (b200_vae_conv).  x [n, h, w, cin] 16-bit NHWC; w16 the packed 2-D weight (vae.pack_conv3x3 /
    pack_conv_t3 / pack_down2, cast to x's dtype); bias fp32 [cout]; add16 like the output.  kind "3x3": Conv2d padding 1;
    "t3": Conv3d (3,1,1) over the n frames of one clip; "down2": pad (0,1,0,1) + stride-2 Conv2d -> [n, h/2, w/2, cout]."""
    _need_cuda(x, w16, bias, add16)
    assert x.dim() == 4 and x.is_contiguous() and w16.is_contiguous() and w16.dtype == x.dtype
    n, h, w, cin = x.shape
    cout = w16.shape[0]
    ho, wo = (h // 2, w // 2) if kind == "down2" else (h, w)
    out = torch.empty(n, ho, wo, cout, dtype=x.dtype, device=x.device)
    if add16 is not None:
        assert add16.shape == out.shape and add16.dtype == x.dtype and add16.is_contiguous()
    scratch = torch.empty(n, ho, wo, 4 * cin, dtype=x.dtype, device=x.device) if kind == "down2" else None
    call("b200_vae_conv", x.device, x.data_ptr(), w16.data_ptr(), _ptr(bias), _ptr(add16), out.data_ptr(), _ptr(scratch),
         n, h, w, cin, cout, _VAE_CONV_KINDS[kind], _dt(x))
    return out


def group_norm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, groups: int, eps: float, silu: bool = False) -> torch.Tensor:
    """GroupNorm (+ SiLU) of the VAE (b200_group_norm) over each image of x [n, ..., C] 16-bit channels-last; gamma, beta fp32 [C]."""
    _need_cuda(x, gamma, beta)
    assert x.is_contiguous() and gamma.dtype == beta.dtype == torch.float32
    n, C = x.shape[0], x.shape[-1]
    out = torch.empty_like(x)
    part = torch.empty(n, groups, 2, dtype=torch.float32, device=x.device)
    call("b200_group_norm", x.device, x.data_ptr(), out.data_ptr(), gamma.data_ptr(), beta.data_ptr(), part.data_ptr(), n,
         x.numel() // (n * C), C, groups, eps, int(silu), _dt(x))
    return out


def vae_mid_attention(x: torch.Tensor, gn_g: torch.Tensor, gn_b: torch.Tensor, q_w16: torch.Tensor, q_b: torch.Tensor,
                      k_w16: torch.Tensor, k_b: torch.Tensor, v_w16: torch.Tensor, o_w16: torch.Tensor, o_b: torch.Tensor,
                      groups: int, eps: float = 1e-6) -> torch.Tensor:
    """Mid-block attention of the VAE (b200_vae_mid_attention): x [n, h, w, C] 16-bit NHWC -> x + to_out(softmax(q k^T / sqrt(C)) v),
    q/k/v of GroupNorm(x).  *_w16 [C, C] in x's dtype; biases fp32, o_b with the v bias folded in (vae.fold_v_bias)."""
    _need_cuda(x, q_w16, k_w16, v_w16, o_w16)
    assert x.dim() == 4 and x.is_contiguous() and all(t.is_contiguous() and t.dtype == x.dtype for t in (q_w16, k_w16, v_w16, o_w16))
    n, h, w, C = x.shape
    need = workspace_bytes("b200_vae_mid_attention_workspace_bytes", n, h, w, C, groups)
    ws, base = scratch(need, x.device)
    out = torch.empty_like(x)
    call("b200_vae_mid_attention", x.device, x.data_ptr(), out.data_ptr(), gn_g.data_ptr(), gn_b.data_ptr(), q_w16.data_ptr(),
         q_b.data_ptr(), k_w16.data_ptr(), k_b.data_ptr(), v_w16.data_ptr(), o_w16.data_ptr(), o_b.data_ptr(),
         n, h, w, C, groups, eps, _dt(x), base, need)
    return out


def frames_to_uint8(video: torch.Tensor, mode: str = "pipeline") -> torch.Tensor:
    """Decoded frames [n, c, h, w] in [-1, 1] -> uint8 [n, h, w, c] on the device, byte-identical to the reference expression:
    mode "pipeline" = pipeline_latte.py:775,796 (truncating), mode "sample" = sample.py:122 / sample_ddp.py:172 (+0.5 rounding)."""
    _need_cuda(video)
    assert video.dim() == 4 and video.is_contiguous()
    n, c, h, w = video.shape
    out = torch.empty(n, h, w, c, dtype=torch.uint8, device=video.device)
    call("b200_frames_to_uint8", video.device, video.data_ptr(), _kind(video), n, c, h, w, {"pipeline": 0, "sample": 1}[mode],
         out.data_ptr())
    return out


# ---------------------------------------------------------------------------------------------------- training-step passes
def wgrad(dW32: torch.Tensor, dy: torch.Tensor, x: torch.Tensor, col_scale: torch.Tensor) -> torch.Tensor:
    """dW32 [n_out, n_in] (fp32, in place) += col_scale[n_in] * dy [rows, n_out]^T @ x [rows, n_in] (b200_wgrad: both
    activations read untransposed; rows % 64 == 0, n_out % 8 == 0, n_in % 128 == 0)."""
    _need_cuda(dW32, dy, x, col_scale)
    assert dy.is_contiguous() and x.is_contiguous() and dW32.is_contiguous() and dW32.dtype == torch.float32
    rows, n_out = dy.shape
    n_in = x.shape[1]
    call("b200_wgrad", dy.device, dy.data_ptr(), x.data_ptr(), col_scale.data_ptr(), dW32.data_ptr(), rows, n_out, n_in, _dt(dy),
         _sk_flags(dy.device).data_ptr())
    return dW32


def dgrad(dy: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """dx [rows, n_in] = dy [rows, n_out] @ w [n_out, n_in] with the weight in its nn.Linear layout (b200_dgrad: MN-major W
    operand; n_out % 64 == 0, n_in % 128 == 0)."""
    _need_cuda(dy, w)
    assert dy.is_contiguous() and w.is_contiguous() and dy.dtype == w.dtype
    rows, n_out = dy.shape
    n_in = w.shape[1]
    dx = torch.empty(rows, n_in, dtype=dy.dtype, device=dy.device)
    call("b200_dgrad", dy.device, dy.data_ptr(), w.data_ptr(), dx.data_ptr(), rows, n_out, n_in, _dt(dy))
    return dx


def linear_gelu_both(a: torch.Tensor, w: torch.Tensor, bias: torch.Tensor | None) -> tuple[torch.Tensor, torch.Tensor]:
    """(u, gelu_tanh(u)) with u = a @ w^T + bias, both from one GEMM epilogue (training-mode fc1)."""
    _need_cuda(a, w, bias)
    assert a.is_contiguous() and w.is_contiguous() and a.dtype == w.dtype
    M, K = a.shape
    N = w.shape[0]
    u = torch.empty(M, N, dtype=a.dtype, device=a.device)
    act = torch.empty(M, N, dtype=a.dtype, device=a.device)
    call("b200_linear_gelu_both", a.device, a.data_ptr(), w.data_ptr(), _ptr(bias), M, N, K, _dt(a), u.data_ptr(), act.data_ptr())
    return u, act


def gate_residual(x: torch.Tensor, m: torch.Tensor, gate: torch.Tensor, rows_per_batch: int, row_add: torch.Tensor | None = None,
                  tokens: int = 1) -> torch.Tensor:
    """x fp32 [rows, D] + gate[row // rows_per_batch] * m (16-bit), + row_add[(row // tokens) % frames] when given."""
    _need_cuda(x, m, gate, row_add)
    assert x.dtype == torch.float32 and x.is_contiguous() and m.is_contiguous() and gate.stride(1) == 1
    out = torch.empty_like(x)
    frames = row_add.shape[0] if row_add is not None else 0
    call("b200_gate_residual", x.device, x.data_ptr(), m.data_ptr(), gate.data_ptr(), gate.stride(0), rows_per_batch,
         _ptr(row_add), tokens, frames, out.data_ptr(), x.shape[0], x.shape[1], _dt(m))
    return out


def gate_bwd(dx: torch.Tensor, m: torch.Tensor, gate: torch.Tensor, rows_per_batch: int, dgate: torch.Tensor,
             dbias: torch.Tensor) -> torch.Tensor:
    """Backward of gate_residual: returns dm = dx * gate (like m); dgate and dbias accumulate."""
    _need_cuda(dx, m, gate, dgate, dbias)
    assert dx.dtype == torch.float32 and dx.is_contiguous() and m.is_contiguous() and dgate.stride(1) == 1
    T, D = dx.shape
    dm = torch.empty(T, D, dtype=m.dtype, device=dx.device)
    call("b200_gate_bwd", dx.device, dx.data_ptr(), m.data_ptr(), gate.data_ptr(), gate.stride(0), rows_per_batch, dm.data_ptr(),
         dgate.data_ptr(), dgate.stride(0), dbias.data_ptr(), T, D, _dt(m))
    return dm


def gelu_bwd(da: torch.Tensor, u: torch.Tensor, dbias: torch.Tensor) -> torch.Tensor:
    """du = da * gelu_tanh'(u) (16-bit); dbias accumulates its column sums."""
    _need_cuda(da, u, dbias)
    T, D = u.shape
    du = torch.empty_like(u)
    call("b200_gelu_bwd", u.device, da.data_ptr(), u.data_ptr(), du.data_ptr(), dbias.data_ptr(), T, D, _dt(u))
    return du


def ln_modulate_bwd(dh: torch.Tensor, x: torch.Tensor, scale: torch.Tensor, rows_per_batch: int, dx: torch.Tensor,
                    dshift: torch.Tensor, dscale: torch.Tensor) -> None:
    """Backward of ln_modulate: dx (fp32), dshift and dscale accumulate."""
    _need_cuda(dh, x, scale, dx, dshift, dscale)
    assert dshift.stride(0) == dscale.stride(0) and dshift.stride(1) == 1
    T, D = x.shape
    call("b200_ln_modulate_bwd", x.device, dh.data_ptr(), x.data_ptr(), scale.data_ptr(), scale.stride(0), rows_per_batch,
         dx.data_ptr(), dshift.data_ptr(), dscale.data_ptr(), dshift.stride(0), T, D, _dt(dh))


def attention_bwd(qkv: torch.Tensor, o: torch.Tensor, do: torch.Tensor, batch: int, frames: int, tokens: int, heads: int,
                  temporal: bool) -> torch.Tensor:
    """Backward of `attention`: dqkv like qkv."""
    _need_cuda(qkv, o, do)
    D = o.shape[1]
    dqkv = torch.empty_like(qkv)
    # row statistics (lse, delta) of the two-kernel backward: spatial sequences and temporal ones longer than 16 frames;
    # the <= 16-frame temporal kernel keeps them in shared memory
    stats = None if temporal and frames <= 16 else torch.empty(2 * batch * frames * heads * tokens, dtype=torch.float32,
                                                               device=qkv.device)
    call("b200_attention_bwd", qkv.device, qkv.data_ptr(), o.data_ptr(), do.data_ptr(), dqkv.data_ptr(), _ptr(stats), batch,
         frames, tokens, heads, D // heads, _dt(qkv), int(temporal))
    return dqkv


def cross_attention_bwd(q: torch.Tensor, kv: torch.Tensor, o: torch.Tensor, do: torch.Tensor, batch: int, q_rows_per_batch: int,
                        kv_len: int, heads: int, key_bias: torch.Tensor | None, dkv: torch.Tensor, col0: int,
                        workspace: torch.Tensor) -> torch.Tensor:
    """Backward of `cross_attention`: returns dq; dK | dV go to dkv[:batch*kv_len, col0:col0 + 2*heads*hd] (dkv 16-bit,
    row-major).  workspace: >= b200_cross_attention_bwd_workspace_bytes(...) bytes on q's device."""
    _need_cuda(q, kv, o, do, key_bias, dkv, workspace)
    assert q.is_contiguous() and o.is_contiguous() and do.is_contiguous() and kv.stride(1) == 1 and dkv.stride(1) == 1
    D = q.shape[1]
    dq = torch.empty_like(q)
    call("b200_cross_attention_bwd", q.device, q.data_ptr(), kv.data_ptr(), _ptr(key_bias), o.data_ptr(), do.data_ptr(),
         dq.data_ptr(), dkv.data_ptr(), dkv.stride(0), col0, batch, q_rows_per_batch, kv_len, q.stride(0), kv.stride(0), heads,
         D // heads, _dt(q), workspace.data_ptr(), workspace.numel())
    return dq


def colsum(a: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """out fp32 [dim] += column sums of a [rows, dim] (fp32 or 16-bit)."""
    _need_cuda(a, out)
    assert a.is_contiguous() and out.is_contiguous() and out.dtype == torch.float32
    call("b200_colsum", a.device, a.data_ptr(), _kind(a), out.data_ptr(), a.shape[0], a.shape[1])
    return out


def transpose16(a: torch.Tensor) -> torch.Tensor:
    """a [rows, cols] 16-bit -> a^T [cols, rows], contiguous."""
    _need_cuda(a)
    assert a.is_contiguous() and a.element_size() == 2
    out = torch.empty(a.shape[1], a.shape[0], dtype=a.dtype, device=a.device)
    call("b200_transpose16", a.device, a.data_ptr(), out.data_ptr(), a.shape[0], a.shape[1])
    return out


def cast16(x32: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """The first x32.numel() elements of out (16-bit) = x32 (fp32, contiguous)."""
    _need_cuda(x32, out)
    assert x32.dtype == torch.float32 and x32.is_contiguous() and out.is_contiguous() and out.numel() >= x32.numel()
    call("b200_cast16", x32.device, x32.data_ptr(), out.data_ptr(), x32.numel(), _dt(out))
    return out


def ada_outer(dmod: torch.Tensor, sc: torch.Tensor) -> torch.Tensor:
    """dW fp32 [NA, D] = dmod fp32 [B, NA]^T @ sc 16-bit [B, D] for B <= 8 rows."""
    _need_cuda(dmod, sc)
    B, NA = dmod.shape
    D = sc.shape[1]
    dW = torch.empty(NA, D, dtype=torch.float32, device=dmod.device)
    call("b200_ada_outer", dmod.device, dmod.data_ptr(), dmod.stride(0), sc.data_ptr(), dW.data_ptr(), B, NA, D, _dt(sc))
    return dW


def ada_dsc(dmod: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """dsc fp32 [B, D] = dmod fp32 [B, NA] @ w 16-bit [NA, D] for B <= 8 rows."""
    _need_cuda(dmod, w)
    B, NA = dmod.shape
    D = w.shape[1]
    dsc = torch.empty(B, D, dtype=torch.float32, device=dmod.device)
    call("b200_ada_dsc", dmod.device, dmod.data_ptr(), dmod.stride(0), w.data_ptr(), dsc.data_ptr(), B, NA, D, _dt(w))
    return dsc


# ---------------------------------------------------------------------------------------------------- multi-tensor passes
_TABLE_CHUNK = 4096     # floats per chunk of both multi-tensor kernels (MT_CHUNK elements, MC_CHUNK float4s)
_tables: "OrderedDict[tuple, tuple]" = OrderedDict()


def _table(srcs, dsts, dst_dtype, unit):
    """Device table of {src, dst, count, first_chunk} records (None = an unused side) for one launch over many tensors;
    counts are in units of `unit` elements.  Cached (LRU of 8) on the pointers and sizes: it is rebuilt only when a tensor
    moves or changes size."""
    key = (unit,) + tuple(t.data_ptr() if t is not None else 0 for t in srcs) + \
        tuple(t.data_ptr() if t is not None else 0 for t in dsts) + tuple(t.numel() for t in (srcs if srcs[0] is not None else dsts))
    hit = _tables.get(key)
    if hit is not None:
        _tables.move_to_end(key)
        return hit
    rows, first, dev, chunk = [], 0, None, _TABLE_CHUNK // unit
    for a, b in zip(srcs, dsts):
        _need_cuda(a, b)
        t = a if a is not None else b
        for s, dtype in ((a, torch.float32), (b, dst_dtype)):
            if s is not None and (s.dtype != dtype or not s.is_contiguous() or s.shape != t.shape):
                raise TypeError(f"latte_b200: contiguous float32 sources and {dst_dtype} destinations of matching shapes expected")
            # a record counts whole units: a multiple of `unit` elements starting on a unit boundary
            if s is not None and (s.numel() % unit or s.data_ptr() % (unit * s.element_size())):
                raise ValueError(f"latte_b200: {unit}-element aligned tensors of a multiple of {unit} elements expected")
        dev = t.device
        n = t.numel() // unit
        rows.append([a.data_ptr() if a is not None else 0, b.data_ptr() if b is not None else 0, n, first])
        first += (n + chunk - 1) // chunk
    host = torch.tensor(rows, dtype=torch.int64).pin_memory()        # async upload: building a table never stalls the host on the GPU
    out = (host.to(dev, non_blocking=True), len(rows), first, dev, host)
    _tables[key] = out
    while len(_tables) > 8:
        _tables.popitem(last=False)
    return out


def multi_tensor(op: int, srcs, dsts, a: float = 0.0, b: float = 0.0, scalar: torch.Tensor | None = None,
                 accum: torch.Tensor | None = None) -> None:
    """One b200_multi_tensor launch (`op` = utils.MT_*) over fp32 tensors srcs[i] / dsts[i]; None stands for an unused side."""
    table, n, total, dev, _ = _table(srcs, dsts, torch.float32, 1)
    call("b200_multi_tensor", dev, table.data_ptr(), n, total, op, float(a), float(b), _ptr(scalar), _ptr(accum))


def multi_cast(srcs, dsts) -> None:
    """dsts[i] (16-bit, contiguous) = srcs[i] (fp32, contiguous) for all i in one launch (b200_multi_cast)."""
    table, n, total, dev, _ = _table(srcs, dsts, dsts[0].dtype, 4)
    call("b200_multi_cast", dev, table.data_ptr(), n, total, _dt(dsts[0]))
