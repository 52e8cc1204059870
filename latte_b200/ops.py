"""Thin torch-tensor wrappers over the per-op C-ABI entry points (used by the parity tests and by
anyone who wants a single fused op).  Device pointers + current stream in, nothing else."""
from __future__ import annotations

import torch

from . import _lib


def _dt(t: torch.Tensor) -> int:
    if t.dtype == torch.float16:
        return _lib.FP16
    if t.dtype == torch.bfloat16:
        return _lib.BF16
    raise TypeError(f"expected a float16/bfloat16 tensor, got {t.dtype}")


def _stream(t: torch.Tensor):
    return torch.cuda.current_stream(t.device).cuda_stream


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
    with torch.cuda.device(a.device):
        rc = _lib.load().b200_linear(a.data_ptr(), w.data_ptr(), bias.data_ptr() if bias is not None else None, M, N, K,
                                     _dt(a), _lib.EPI_BIAS_GELU if gelu else _lib.EPI_BIAS, out.data_ptr(), None, None,
                                     0, 1, block_n, None, _stream(a))
    _lib.check(rc, "b200_linear")
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
    with torch.cuda.device(a.device):
        rc = _lib.load().b200_linear(a.data_ptr(), w.data_ptr(), bias.data_ptr() if bias is not None else None, M, N, K,
                                     _dt(a), _lib.EPI_GATE_RESIDUAL, None, resid.data_ptr(), gate.data_ptr(),
                                     gate.stride(0), rows_per_batch, block_n,
                                     _sk_flags(a.device).data_ptr() if stream_k else None, _stream(a))
    _lib.check(rc, "b200_linear")
    return resid


def attention(qkv: torch.Tensor, batch: int, frames: int, tokens: int, heads: int, temporal: bool) -> torch.Tensor:
    """qkv [batch*frames*tokens, 3*heads*hd] 16-bit -> out [T, heads*hd] 16-bit."""
    _need_cuda(qkv)
    assert qkv.is_contiguous() and qkv.shape[0] == batch * frames * tokens
    D = qkv.shape[1] // 3
    out = torch.empty(qkv.shape[0], D, dtype=qkv.dtype, device=qkv.device)
    with torch.cuda.device(qkv.device):
        rc = _lib.load().b200_attention(qkv.data_ptr(), out.data_ptr(), batch, frames, tokens, heads, D // heads,
                                        _dt(qkv), int(temporal), _stream(qkv))
    _lib.check(rc, "b200_attention")
    return out


def ln_modulate(x: torch.Tensor, shift: torch.Tensor, scale: torch.Tensor, rows_per_batch: int,
                dtype: torch.dtype = torch.float16) -> torch.Tensor:
    """x fp32 [rows, D]; shift/scale fp32 [B, D] (row stride arbitrary) -> 16-bit [rows, D]."""
    _need_cuda(x, shift, scale)
    assert x.dtype == torch.float32 and x.is_contiguous() and shift.stride(0) == scale.stride(0)
    out = torch.empty(x.shape, dtype=dtype, device=x.device)
    with torch.cuda.device(x.device):
        rc = _lib.load().b200_ln_modulate(x.data_ptr(), shift.data_ptr(), scale.data_ptr(), shift.stride(0),
                                          rows_per_batch, out.data_ptr(), x.shape[0], x.shape[1], _dt(out), _stream(x))
    _lib.check(rc, "b200_ln_modulate")
    return out


def quantize_rows_e4m3(w: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """w fp32 [rows, cols] -> (q [rows, cols] float8_e4m3fn, scales fp32 [rows]): s = amax(|row|) / 448 (1 for a zero row),
    q = e4m3_rn_satfinite(row / s) (b200_quantize_rows_e4m3)."""
    _need_cuda(w)
    assert w.dtype == torch.float32 and w.dim() == 2 and w.is_contiguous()
    q = torch.empty(w.shape, dtype=torch.uint8, device=w.device)
    s = torch.empty(w.shape[0], dtype=torch.float32, device=w.device)
    with torch.cuda.device(w.device):
        rc = _lib.load().b200_quantize_rows_e4m3(w.data_ptr(), w.shape[0], w.shape[1], q.data_ptr(), s.data_ptr(), _stream(w))
    _lib.check(rc, "b200_quantize_rows_e4m3")
    return q.view(torch.float8_e4m3fn), s


def ln_modulate_e4m3(x: torch.Tensor, shift: torch.Tensor, scale: torch.Tensor,
                     rows_per_batch: int) -> tuple[torch.Tensor, torch.Tensor]:
    """ln_modulate quantized per row: x fp32 [rows, D] -> (q [rows, D] float8_e4m3fn, row scales fp32 [rows])."""
    _need_cuda(x, shift, scale)
    assert x.dtype == torch.float32 and x.is_contiguous() and shift.stride(0) == scale.stride(0)
    q = torch.empty(x.shape, dtype=torch.uint8, device=x.device)
    s = torch.empty(x.shape[0], dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        rc = _lib.load().b200_ln_modulate_e4m3(x.data_ptr(), shift.data_ptr(), scale.data_ptr(), shift.stride(0), rows_per_batch,
                                               q.data_ptr(), s.data_ptr(), x.shape[0], x.shape[1], _stream(x))
    _lib.check(rc, "b200_ln_modulate_e4m3")
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
    with torch.cuda.device(a8.device):
        rc = _lib.load().b200_linear_e4m3(a8.data_ptr(), a_scale.data_ptr(), w8.data_ptr(), w_scale.data_ptr(),
                                          bias.data_ptr() if bias is not None else None, M, N, K, _dt(out),
                                          _lib.EPI_BIAS_GELU if gelu else _lib.EPI_BIAS, out.data_ptr(), _stream(a8))
    _lib.check(rc, "b200_linear_e4m3")
    return out


def cross_attention(q: torch.Tensor, kv: torch.Tensor, batch: int, q_rows_per_batch: int, kv_len: int, heads: int,
                    key_bias: torch.Tensor | None = None) -> torch.Tensor:
    """q [batch*q_rows, heads*hd] 16-bit; kv [batch*kv_len, 2*heads*hd] 16-bit ([k | v]); kv_len <= 128 -> out like q.
    key_bias: optional fp32 [batch, 128] additive score bias per key (columns >= kv_len ignored)."""
    _need_cuda(q, kv, key_bias)
    assert q.is_contiguous() and kv.is_contiguous() and q.dtype == kv.dtype
    if key_bias is not None:
        assert key_bias.dtype == torch.float32 and key_bias.is_contiguous() and tuple(key_bias.shape) == (batch, 128)
    D = q.shape[1]
    out = torch.empty_like(q)
    with torch.cuda.device(q.device):
        rc = _lib.load().b200_cross_attention(q.data_ptr(), kv.data_ptr(), key_bias.data_ptr() if key_bias is not None else None,
                                              out.data_ptr(), batch, q_rows_per_batch, kv_len,
                                              q.shape[1], kv.shape[1], heads, D // heads, _dt(q), _stream(q))
    _lib.check(rc, "b200_cross_attention")
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
    with torch.cuda.device(x.device):
        rc = _lib.load().b200_vae_conv(x.data_ptr(), w16.data_ptr(), bias.data_ptr() if bias is not None else None,
                                       add16.data_ptr() if add16 is not None else None, out.data_ptr(),
                                       scratch.data_ptr() if scratch is not None else None, n, h, w, cin, cout,
                                       _VAE_CONV_KINDS[kind], _dt(x), _stream(x))
    _lib.check(rc, "b200_vae_conv")
    return out


def group_norm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, groups: int, eps: float, silu: bool = False) -> torch.Tensor:
    """GroupNorm (+ SiLU) of the VAE (b200_group_norm) over each image of x [n, ..., C] 16-bit channels-last; gamma, beta fp32 [C]."""
    _need_cuda(x, gamma, beta)
    assert x.is_contiguous() and gamma.dtype == beta.dtype == torch.float32
    n, C = x.shape[0], x.shape[-1]
    out = torch.empty_like(x)
    part = torch.empty(n, groups, 2, dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        rc = _lib.load().b200_group_norm(x.data_ptr(), out.data_ptr(), gamma.data_ptr(), beta.data_ptr(), part.data_ptr(), n,
                                         x.numel() // (n * C), C, groups, eps, int(silu), _dt(x), _stream(x))
    _lib.check(rc, "b200_group_norm")
    return out


def vae_mid_attention(x: torch.Tensor, gn_g: torch.Tensor, gn_b: torch.Tensor, q_w16: torch.Tensor, q_b: torch.Tensor,
                      k_w16: torch.Tensor, k_b: torch.Tensor, v_w16: torch.Tensor, o_w16: torch.Tensor, o_b: torch.Tensor,
                      groups: int, eps: float = 1e-6) -> torch.Tensor:
    """Mid-block attention of the VAE (b200_vae_mid_attention): x [n, h, w, C] 16-bit NHWC -> x + to_out(softmax(q k^T / sqrt(C)) v),
    q/k/v of GroupNorm(x).  *_w16 [C, C] in x's dtype; biases fp32, o_b with the v bias folded in (vae.fold_v_bias)."""
    _need_cuda(x, q_w16, k_w16, v_w16, o_w16)
    assert x.dim() == 4 and x.is_contiguous() and all(t.is_contiguous() and t.dtype == x.dtype for t in (q_w16, k_w16, v_w16, o_w16))
    n, h, w, C = x.shape
    lib = _lib.load()
    need = lib.b200_vae_mid_attention_workspace_bytes(n, h, w, C, groups)
    if need == 0:
        raise RuntimeError("b200_vae_mid_attention: unsupported shape: " + _lib.last_error())
    ws = torch.empty(need + 1024, dtype=torch.uint8, device=x.device)
    base = (ws.data_ptr() + 1023) // 1024 * 1024
    out = torch.empty_like(x)
    with torch.cuda.device(x.device):
        rc = lib.b200_vae_mid_attention(x.data_ptr(), out.data_ptr(), gn_g.data_ptr(), gn_b.data_ptr(), q_w16.data_ptr(), q_b.data_ptr(),
                                        k_w16.data_ptr(), k_b.data_ptr(), v_w16.data_ptr(), o_w16.data_ptr(), o_b.data_ptr(),
                                        n, h, w, C, groups, eps, _dt(x), base, need, _stream(x))
    _lib.check(rc, "b200_vae_mid_attention")
    return out


_U8_DT = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}


def frames_to_uint8(video: torch.Tensor, mode: str = "pipeline") -> torch.Tensor:
    """Decoded frames [n, c, h, w] in [-1, 1] -> uint8 [n, h, w, c] on the device, byte-identical to the reference expression:
    mode "pipeline" = pipeline_latte.py:775,796 (truncating), mode "sample" = sample.py:122 / sample_ddp.py:172 (+0.5 rounding)."""
    _need_cuda(video)
    assert video.dim() == 4 and video.is_contiguous() and video.dtype in _U8_DT
    n, c, h, w = video.shape
    out = torch.empty(n, h, w, c, dtype=torch.uint8, device=video.device)
    with torch.cuda.device(video.device):
        rc = _lib.load().b200_frames_to_uint8(video.data_ptr(), _U8_DT[video.dtype], n, c, h, w, {"pipeline": 0, "sample": 1}[mode],
                                              out.data_ptr(), _stream(video))
    _lib.check(rc, "b200_frames_to_uint8")
    return out
