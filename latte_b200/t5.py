"""`T5EncoderModel` — the text encoder surface the reference's pipeline calls (`sample/pipeline_latte.py:214`:
`self.text_encoder(input_ids, attention_mask=mask)[0]`, transformers' T5EncoderModel for t5-v1_1-xxl), backed by the same
sm_90a kernels as the denoiser through ONE C-ABI call (`b200_t5_encode`): wgmma GEMMs (q|k|v in one, gated-GELU
feed-forward with the multiply in the second GEMM's epilogue, fp32 residual adds in the GEMM epilogue), the attention
kernel with T5's relative-position bias and the prompt mask as additive score biases, RMSNorm and the embedding gather.

Parameter names follow transformers' state dict (`shared.weight`, `encoder.block.N.layer.0.SelfAttention.q.weight`, ...),
so a `T5EncoderModel` checkpoint loads with `load_state_dict`.  Built for the T5 v1.1 family: gated-GELU feed-forward,
d_kv = 64, no biases, bidirectional relative attention buckets, sequences of up to 128 tokens (the pipeline uses 120).
No CPU path.  The tokenizer (sentencepiece) is host code and out of scope.
"""
from __future__ import annotations

import ctypes as C
import math
from types import SimpleNamespace

import torch
import torch.nn as nn

from . import _lib, ops
from ._cache import DeviceCacheMixin

MAX_LEN = 128


class _Attn(nn.Module):
    def __init__(self, d_model, inner, heads, has_bias_table, buckets):
        super().__init__()
        self.q = nn.Linear(d_model, inner, bias=False)
        self.k = nn.Linear(d_model, inner, bias=False)
        self.v = nn.Linear(d_model, inner, bias=False)
        self.o = nn.Linear(inner, d_model, bias=False)
        if has_bias_table:
            self.relative_attention_bias = nn.Embedding(buckets, heads)


class _Norm(nn.Module):
    def __init__(self, d_model):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(d_model))


class _AttnLayer(nn.Module):
    def __init__(self, d_model, inner, heads, first, buckets):
        super().__init__()
        self.SelfAttention = _Attn(d_model, inner, heads, first, buckets)
        self.layer_norm = _Norm(d_model)


class _Dense(nn.Module):
    def __init__(self, d_model, d_ff):
        super().__init__()
        self.wi_0 = nn.Linear(d_model, d_ff, bias=False)
        self.wi_1 = nn.Linear(d_model, d_ff, bias=False)
        self.wo = nn.Linear(d_ff, d_model, bias=False)


class _FFLayer(nn.Module):
    def __init__(self, d_model, d_ff):
        super().__init__()
        self.DenseReluDense = _Dense(d_model, d_ff)
        self.layer_norm = _Norm(d_model)


class _Block(nn.Module):
    def __init__(self, d_model, inner, heads, d_ff, first, buckets):
        super().__init__()
        self.layer = nn.ModuleList([_AttnLayer(d_model, inner, heads, first, buckets), _FFLayer(d_model, d_ff)])


class _Stack(nn.Module):
    def __init__(self, shared, cfg):
        super().__init__()
        self.embed_tokens = shared                      # tied to `shared`, as in transformers
        inner = cfg.num_heads * cfg.d_kv
        self.block = nn.ModuleList([_Block(cfg.d_model, inner, cfg.num_heads, cfg.d_ff, i == 0, cfg.relative_attention_num_buckets)
                                    for i in range(cfg.num_layers)])
        self.final_layer_norm = _Norm(cfg.d_model)


class EncoderOutput(tuple):
    """`out[0]` / `out.last_hidden_state`, like transformers' BaseModelOutput."""

    @property
    def last_hidden_state(self):
        return self[0]


def relative_position_buckets(length: int, num_buckets: int = 32, max_distance: int = 128) -> torch.Tensor:
    """Bucket index of (key position j - query position i) for the bidirectional encoder (transformers
    T5Attention._relative_position_bucket): half of the buckets per sign; within a sign the first half are exact offsets and
    the rest grow logarithmically up to `max_distance`.  Returns int64 [length, length], entry [i, j]."""
    pos = torch.arange(length)
    rel = pos[None, :] - pos[:, None]
    half = num_buckets // 2
    out = (rel > 0).long() * half
    dist = rel.abs()
    exact = half // 2
    log_bucket = exact + (torch.log(dist.float().clamp(min=1) / exact) / math.log(max_distance / exact) * (half - exact)).long()
    log_bucket = log_bucket.clamp(max=half - 1)
    return out + torch.where(dist < exact, dist, log_bucket)


def mask_text_embeddings(emb: torch.Tensor, mask: torch.Tensor):
    """`LattePipeline.mask_text_embeddings` (sample/pipeline_latte.py:118-124): a single prompt is TRIMMED to its kept tokens
    (emb (1, 1, L, D) -> (1, 1, keep, D)); a batch keeps the padding and zeroes the masked rows.  Returns (emb, keep)."""
    if emb.shape[0] == 1:
        keep = int(mask.sum().item())
        return emb[:, :, :keep, :], keep
    return emb * mask[:, None, :, None], emb.shape[2]


class T5EncoderModel(DeviceCacheMixin, nn.Module):
    def __init__(self, vocab_size=32128, d_model=4096, d_kv=64, d_ff=10240, num_layers=24, num_heads=64,
                 relative_attention_num_buckets=32, relative_attention_max_distance=128, layer_norm_epsilon=1e-6,
                 feed_forward_proj="gated-gelu", **unused):
        super().__init__()
        if feed_forward_proj != "gated-gelu" or d_kv != 64:
            raise NotImplementedError("latte_b200.T5EncoderModel is built for the T5 v1.1 family (gated-gelu, d_kv = 64)")
        self.config = SimpleNamespace(vocab_size=vocab_size, d_model=d_model, d_kv=d_kv, d_ff=d_ff, num_layers=num_layers,
                                      num_heads=num_heads, relative_attention_num_buckets=relative_attention_num_buckets,
                                      relative_attention_max_distance=relative_attention_max_distance,
                                      layer_norm_epsilon=layer_norm_epsilon, feed_forward_proj=feed_forward_proj)
        self.shared = nn.Embedding(vocab_size, d_model)
        self.encoder = _Stack(self.shared, self.config)
        self.compute_dtype = torch.float16
        self._packed = None
        self._packed_key = None
        self._workspace = None

    @property
    def dtype(self):
        return self.shared.weight.dtype

    def _operand_dtype(self):
        pd = self.shared.weight.dtype
        return pd if pd in (torch.float16, torch.bfloat16) else self.compute_dtype

    def repack(self):
        self._packed = None
        self._packed_key = None

    @torch.no_grad()
    def _pack(self):
        ver = sum(p._version for p in self.parameters())
        w0 = self.shared.weight
        key = (ver, w0.data_ptr(), w0.device, w0.dtype, self.compute_dtype)
        if self._packed is not None and key == self._packed_key:
            return self._packed
        dev, od, c = w0.device, self._operand_dtype(), self.config
        f32 = lambda t: t.detach().to(device=dev, dtype=torch.float32).contiguous()   # noqa: E731
        h16 = lambda t: t.detach().to(device=dev, dtype=od).contiguous()              # noqa: E731
        blocks = list(self.encoder.block)
        att = [b.layer[0].SelfAttention for b in blocks]
        ff = [b.layer[1].DenseReluDense for b in blocks]
        T = {
            "embed16": h16(self.shared.weight),
            "qkv_w16": h16(torch.stack([torch.cat([a.q.weight.detach(), a.k.weight.detach(), a.v.weight.detach()]) for a in att])),
            "o_w16": h16(torch.stack([a.o.weight.detach() for a in att])),
            "ln0_w": f32(torch.stack([b.layer[0].layer_norm.weight.detach() for b in blocks])),
            "wi0_w16": h16(torch.stack([f.wi_0.weight.detach() for f in ff])),
            "wi1_w16": h16(torch.stack([f.wi_1.weight.detach() for f in ff])),
            "wo_w16": h16(torch.stack([f.wo.weight.detach() for f in ff])),
            "ln1_w": f32(torch.stack([b.layer[1].layer_norm.weight.detach() for b in blocks])),
            "final_w": f32(self.encoder.final_layer_norm.weight),
        }
        # position bias [heads, 128, 128]: relative_attention_bias[bucket(j - i)][h] -- depends on the weights only
        buckets = relative_position_buckets(MAX_LEN, c.relative_attention_num_buckets, c.relative_attention_max_distance).to(dev)
        table = f32(att[0].relative_attention_bias.weight)                     # [buckets, heads]
        pos = table[buckets].permute(2, 0, 1).contiguous()                     # [heads, 128, 128]
        w = _lib.T5Weights()
        for name in _lib.T5_WEIGHT_FIELDS:
            setattr(w, name, T[name].data_ptr())
        shape = _lib.T5Shape(layers=c.num_layers, d_model=c.d_model, heads=c.num_heads, d_ff=c.d_ff, vocab=c.vocab_size,
                             dtype=_lib.BF16 if od == torch.bfloat16 else _lib.FP16, eps=float(c.layer_norm_epsilon))
        self._packed, self._packed_key = (shape, w, T, pos), key
        return self._packed

    def forward(self, input_ids=None, attention_mask=None, return_dict=True, **unused):
        """input_ids (B, L <= 128) int64, attention_mask (B, L) 1 = keep -> last_hidden_state (B, L, d_model)."""
        if input_ids is None or not input_ids.is_cuda:
            raise RuntimeError("latte_b200.T5EncoderModel runs on CUDA (sm_90a) only; there is no CPU fallback")
        B, L = input_ids.shape
        if L > MAX_LEN:
            raise NotImplementedError(f"sequences longer than {MAX_LEN} tokens are not built (the pipeline uses 120)")
        dev = input_ids.device
        with torch.cuda.device(dev):
            shape, w, _, pos = self._pack()
            ids = torch.zeros(B, MAX_LEN, dtype=torch.int64, device=dev)
            ids[:, :L] = input_ids
            bias = torch.full((B, MAX_LEN), -1e30, dtype=torch.float32, device=dev)     # padding columns: never attended
            keep = torch.ones(B, L, device=dev) if attention_mask is None else attention_mask.to(device=dev, dtype=torch.float32)
            bias[:, :L] = (1.0 - keep) * -1e30                                         # the extended attention mask
            out = torch.empty(B, MAX_LEN, self.config.d_model, dtype=torch.float32, device=dev)
            need = ops.workspace_bytes("b200_t5_workspace_bytes", C.byref(shape), B)
            ops.call("b200_t5_encode", dev, C.byref(shape), C.byref(w), ids.data_ptr(), bias.data_ptr(), pos.data_ptr(), B,
                     out.data_ptr(), self._aligned_workspace(need, dev), need)
        pd = self.dtype
        res = out[:, :L].contiguous()
        res = res if pd == torch.float32 else res.to(pd)
        return EncoderOutput((res,))
