"""Row-by-row budget of the sampling forward against fp64, shared by test_gpu_sample_fp64.py (the native forward at the
geometries and precisions the models sample at) and test_sample_forward_bounds.py (the same machinery on the CPU).

A row is one (sample, frame, patch token) of the model output, with its eps half and its variance half as separate rows:
p p C values each (16 at p = 2).  The halves are measured apart because guidance touches eps only and because their
scales differ.  Every row r of each half (R rows) must satisfy the budget of tests/step_fp64.py without its Z0 term:

    |o_nat[r] - o64[r]| <= K a[r] + A u |o64[r]| + Z |o64|_F / sqrt(R)
    a[r] = max(|o_ac[r] - o64[r]|, rho max(|o64[r]|, |o64|_F / sqrt(R))),  rho = |o_ac - o64|_F / |o64|_F

o64 is the functional oracle in fp64 on the module's own weights and inputs, o_ac the same oracle under the recipe's
yardstick, u the unit roundoff of the output's type:
  * fp16 / bf16: fp32 parameters with that compute_dtype; o_ac the oracle in fp32 under that autocast.
  * half: `model.half()` (fp16 parameters, fp16 output); o64 and o_ac on the fp16 parameter values, o_ac under fp16 autocast.
  * fp8: `use_fp8` with fp16 operands; o_ac the fp64 oracle with an e4m3 quantize-dequantize on both operands of every
    QKV and fc1 (`fp8_recipe`): a per-token activation scale amax / 448 and a per-output-channel weight scale, values
    through torch's float8_e4m3fn cast, as test_gpu_fp8.py quantizes.

The oracle edits (`edits`) restate the oracles' attention and feed-forward with hooks, to build the fp8 recipe and the
wrong results the budget must reject: swapped heads, keys dropped, the text K/V of another layer.  With no hook set they
compute exactly what the oracles compute (test_sample_forward_bounds.py checks that bit for bit)."""
import contextlib
import re

import torch
import torch.nn.functional as F

import step_fp64 as SB
from oracle import latte_oracle as O
from oracle import t2v_oracle as T
from oracle import t2v_res_oracle as R

# (K, A, Z, Z0) per recipe, set from a run of tests/test_gpu_sample_fp64.py on an NVIDIA H100 80GB HBM3 at a 700 W power
# limit; the figures it printed are in that file's docstring
BUDGET = {"fp16": (4.0, 1.0, 2.0 ** -10, 0.0), "bf16": (4.0, 1.0, 2.0 ** -10, 0.0), "half": (4.0, 1.0, 2.0 ** -10, 0.0),
          "fp8": (4.0, 1.0, 2.0 ** -10, 0.0)}
E4M3_MAX = 448.0


# ------------------------------------------------------------------------------------------------------------ rows
def out_rows(o, p, channels_first=False):
    """Model output (B, F, 2C, H, W), or LatteT2V's (B, 2C, F, H, W) with channels_first -> {"eps": (R, C p p),
    "var": (R, C p p)}, one row per (sample, frame, patch token) in the output's own dtype."""
    if channels_first:
        o = o.transpose(1, 2)
    B, Fr, C2, H, W = o.shape
    r = o.reshape(B, Fr, 2, C2 // 2, H // p, p, W // p, p).permute(2, 0, 1, 4, 6, 3, 5, 7)
    r = r.reshape(2, B * Fr * (H // p) * (W // p), -1)
    return {"eps": r[0], "var": r[1]}


def check(got, o64, oac, budget, p, channels_first=False):
    """{"eps": Row, "var": Row}: step_fp64.ratio on each half's rows."""
    g, r64, rac = (out_rows(v, p, channels_first) for v in (got, o64, oac))
    return {h: SB.ratio(g[h], r64[h], rac[h], budget, 0.0) for h in g}


def rejected(got, o64, oac, wrong, base, budget, p, channels_first=False):
    """The worst ratio of the wrong result got + (wrong - base) (base: o64, or the recipe oracle the defect modifies)."""
    bad = (got.double() + (wrong.double() - base.double())).to(got.dtype)
    return max(check(bad, o64, oac, budget, p, channels_first).values(), key=lambda w: w.ratio)


# ------------------------------------------------------------------------------------------------------------ oracle edits
def _core(q, k, v, bias):
    s = q @ k.transpose(-1, -2) * q.shape[-1] ** -0.5
    if bias is not None:
        s = s + bias.to(s.dtype)[:, None, None, :]
    return torch.softmax(s, dim=-1) @ v


@contextlib.contextmanager
def edits(core=None, lin=None, kv_prefix=None):
    """Within the block, the oracles' attention and feed-forward run restated with hooks:
    core(prefix, q, k, v, bias) -> per-head attention output (B, heads, S, hd), or None for the plain one;
    lin(name, x, weight, bias) -> F.linear for QKV and fc1, or None for the plain one (name: "blocks.0.attn.qkv",
    "transformer_blocks.0.attn1.to_q", ..., "blocks.0.mlp.fc1", "temporal_transformer_blocks.0.ff.net.0.proj");
    kv_prefix(prefix) -> the attention prefix whose to_k / to_v project the context, or None for the prefix itself."""
    def attn_out(prefix, q, k, v, bias):
        o = core(prefix, q, k, v, bias) if core is not None else None
        return _core(q, k, v, bias) if o is None else o

    def qkv_lin(name, x, w, b):
        out = lin(name, x, w, b) if lin is not None else None
        return F.linear(x, w, b) if out is None else out

    def attention_math(sd, prefix, x, num_heads):
        Bs, S, C = x.shape
        hd, dt = C // num_heads, x.dtype
        qkv = qkv_lin(prefix + "qkv", x, sd[prefix + "qkv.weight"].to(dt), sd[prefix + "qkv.bias"].to(dt))
        q, k, v = qkv.reshape(Bs, S, 3, num_heads, hd).permute(2, 0, 3, 1, 4)
        o = attn_out(prefix, q, k, v, None).transpose(1, 2).reshape(Bs, S, C)
        return F.linear(o, sd[prefix + "proj.weight"].to(dt), sd[prefix + "proj.bias"].to(dt))

    def mlp(sd, prefix, x):
        dt = x.dtype
        h = F.gelu(qkv_lin(prefix + "fc1", x, sd[prefix + "fc1.weight"].to(dt), sd[prefix + "fc1.bias"].to(dt)), approximate="tanh")
        return F.linear(h, sd[prefix + "fc2.weight"].to(dt), sd[prefix + "fc2.bias"].to(dt))

    def attention(sd, prefix, x, ctx, heads, key_bias=None):
        B, S, D = x.shape
        hd, dt = D // heads, x.dtype
        self_attn = ".attn1" in prefix                     # QKV of the self-attentions only, not the cross-attention

        def proj(n, z):
            w, b = sd[n + ".weight"].to(dt), sd[n + ".bias"].to(dt)
            return qkv_lin(n, z, w, b) if self_attn else F.linear(z, w, b)
        kvp = (kv_prefix(prefix) if kv_prefix is not None else None) or prefix
        q = proj(prefix + ".to_q", x).reshape(B, S, heads, hd).transpose(1, 2)
        k = proj(kvp + ".to_k", ctx).reshape(B, -1, heads, hd).transpose(1, 2)
        v = proj(kvp + ".to_v", ctx).reshape(B, -1, heads, hd).transpose(1, 2)
        o = attn_out(prefix, q, k, v, key_bias).transpose(1, 2).reshape(B, S, D)
        return T._lin(sd, prefix + ".to_out.0", o)

    def feed_forward(sd, prefix, x):
        n = prefix + ".net.0.proj"
        h = F.gelu(qkv_lin(n, x, sd[n + ".weight"].to(x.dtype), sd[n + ".bias"].to(x.dtype)), approximate="tanh")
        return T._lin(sd, prefix + ".net.2", h)

    saved = [(O, "attention_math", attention_math), (O, "mlp", mlp), (T, "attention", attention), (T, "feed_forward", feed_forward)]
    old = [getattr(m, n) for m, n, _ in saved]
    for m, n, f in saved:
        setattr(m, n, f)
    try:
        yield
    finally:
        for (m, n, _), f in zip(saved, old):
            setattr(m, n, f)


@contextlib.contextmanager
def pos_table(fn):
    """t2v_res_oracle's position table replaced by fn(cfg, grid_h, grid_w)."""
    old = R.pos_embed_table
    R.pos_embed_table = fn
    try:
        yield
    finally:
        R.pos_embed_table = old


def _block(prefix):
    return int(re.match(r"(?:blocks|transformer_blocks|temporal_transformer_blocks)\.(\d+)", prefix).group(1))


def is_temporal(prefix):
    """Latte's odd blocks, LatteT2V's temporal blocks."""
    return prefix.startswith("temporal_transformer_blocks.") or (prefix.startswith("blocks.") and _block(prefix) % 2 == 1)


def is_spatial_self(prefix):
    return (prefix.startswith("blocks.") and _block(prefix) % 2 == 0) or re.match(r"transformer_blocks\.\d+\.attn1", prefix) is not None


def swap_heads(target):
    """Heads 0 and 1 of the attention at `target` exchange their outputs."""
    def core(prefix, q, k, v, bias):
        if prefix != target:
            return None
        o = _core(q, k, v, bias)
        return o[:, [1, 0] + list(range(2, o.shape[1]))]
    return core


def drop_last_key(where):
    """The last key (and value) of every sequence of the attentions `where(prefix)` selects is left out."""
    def core(prefix, q, k, v, bias):
        if not where(prefix):
            return None
        return _core(q, k[..., :-1, :], v[..., :-1, :], None if bias is None else bias[:, :-1])
    return core


def previous_layer_text_kv(prefix):
    """Layer l's cross-attention projects the caption with layer l - 1's to_k / to_v (layer 0 keeps its own)."""
    m = re.match(r"transformer_blocks\.(\d+)\.attn2$", prefix)
    if m is None or int(m.group(1)) == 0:
        return None
    return f"transformer_blocks.{int(m.group(1)) - 1}.attn2"


# ------------------------------------------------------------------------------------------------------------ e4m3
def qdq_rows(x, next_scale=False, drop_scale=0):
    """e4m3 quantize-dequantize of a matrix, one scale per row: s = amax / 448 (1 for an all-zero row),
    q = e4m3(x / s) (satfinite) -> q s in x's dtype.  next_scale: each row's q comes back with the next row's scale (the
    last row keeps its own), as a GEMM reading its neighbour's activation scale would give it.  drop_scale: the last
    `drop_scale` rows come back as q, without their scale."""
    amax = x.abs().amax(-1, keepdim=True)
    s = torch.where(amax > 0, amax / E4M3_MAX, torch.ones_like(amax))
    q = (x / s).float().clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn).to(x.dtype)
    if next_scale:
        s = torch.cat([s[1:], s[-1:]])
    out = q * s
    if drop_scale:
        out[..., -drop_scale:, :] = q[..., -drop_scale:, :]
    return out


def _last_output_rows(name):
    """The native QKV stacks q, k, v by output channel, so its last output channels are to_v's (or qkv's) last rows."""
    return name.endswith(("qkv", ".to_v", "fc1", ".net.0.proj"))


def fp8_recipe(defect=None):
    """lin hook for `edits`: both operands of every QKV and fc1 e4m3 quantize-dequantized, the product in x's precision.
    The weight is quantized from its fp32 values, as the module packs it.  defect: None, "token" (every token's
    activations scaled back with the next token's scale) or "w_scale" (the weight scale dropped on the last 32 output
    channels).  A single token scaled back with its neighbour's scale is no defect this budget can see: neighbouring
    tokens' scales differ by a few percent, inside the recipe's own error (at the CPU rehearsal's shapes that wrong result
    needs K = 2.5 to 3.8); test_gpu_fp8.py holds the GEMM to its dequantized operands element by element."""
    def lin(name, x, w, b):
        xq = qdq_rows(x.reshape(-1, x.shape[-1]), next_scale=defect == "token").reshape(x.shape)
        w32 = w.float()
        wq = qdq_rows(w32, drop_scale=32 if defect == "w_scale" and _last_output_rows(name) else 0).to(x.dtype)
        return F.linear(xq, wq, b)
    return lin


# ------------------------------------------------------------------------------------------------------------ forwards
def latte_out(sd, cfg, x, t, y, dtype, cfg_scale=None, guided=None):
    """O.latte_forward, or O.latte_forward_with_cfg with cfg_scale; guided: the number of leading channels guidance is
    applied to, when it is not the reference's in_channels."""
    if cfg_scale is None:
        return O.latte_forward(sd, cfg, x, t, y, dtype)
    if guided is None:
        return O.latte_forward_with_cfg(sd, cfg, x, t, y, cfg_scale, dtype)
    half = x[: len(x) // 2]
    out = O.latte_forward(sd, cfg, torch.cat([half, half]), t, y, dtype)
    c, u = out[:, :, :guided].chunk(2)
    g = u + cfg_scale * (c - u)
    return torch.cat([torch.cat([g, g]), out[:, :, guided:]], dim=2)


def t2v_out(sd, cfg, x, t, text, mask, dtype):
    """t2v_oracle.t2v_forward on the configured square latent, t2v_res_oracle.t2v_forward on any other."""
    if tuple(x.shape[-2:]) == (cfg.sample_size, cfg.sample_size):
        return T.t2v_forward(sd, cfg, x, t, text, dtype, True, mask)
    return R.t2v_forward(sd, cfg, x, t, text, dtype, True, mask)


def square_table(cfg, gh, gw):
    """The table of a gw x gw grid (the configured one when gw = sample_size / patch), its first gh gw rows."""
    return _table(cfg, gw, gw, cfg.sample_size // cfg.patch_size)[: gh * gw]


def other_base_table(cfg, gh, gw):
    """The grid's table interpolated to base_size = grid_h instead of sample_size / patch."""
    return _table(cfg, gh, gw, gh)


def _table(cfg, gh, gw, base):
    return torch.from_numpy(R.get_2d_sincos_pos_embed(cfg.inner_dim, (gh, gw), base, max(cfg.sample_size // 64, 1))).float()
