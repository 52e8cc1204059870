"""CPU restatement of Pyramid Attention Broadcast on LatteT2V -- test infrastructure, not product code.

`forward` is `oracle/t2v_res_oracle.t2v_forward` (any latent height x width) with one more argument, `attn`: each kind of
attention's output before its gate -- spatial `attn1` (gated by gate_msa), temporal `attn1` (its own gate_msa) and cross
`attn2` (no gate) -- is returned per layer, or, where `attn` holds it, taken from there instead of computed.  Both are
[layers, T, D] in the library's row order (b, f, n).  `schedule` restates the rule `LatteT2V.enable_cache` documents, and
`trajectory` runs a sequence of calls that reuses its own outputs under it."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle import latte_oracle as LO
from oracle import t2v_oracle as T
from oracle import t2v_res_oracle as R

KINDS = ("spatial", "temporal", "cross")
COMPUTE, STORE, REUSE = 0, 1, 2


def schedule(taus, ranges, windows):
    """Modes of each call of one trajectory at timesteps `taus` (descending): ranges {kind: r or None}, windows {kind:
    (lo, hi)}.  A kind is computed and stored when its cache is empty, the timestep lies outside (lo, hi), r == 1 or its
    call count is a multiple of r; else reused.  A timestep not below the previous one starts over."""
    out, prev = [], None
    count = {k: 0 for k in KINDS}
    have = {k: False for k in KINDS}
    for tau in taus:
        if prev is not None and tau >= prev:
            count = {k: 0 for k in KINDS}
            have = {k: False for k in KINDS}
        prev = tau
        modes = {}
        for k in KINDS:
            r = ranges.get(k)
            if r is None:
                modes[k] = COMPUTE
                continue
            lo, hi = windows[k]
            reuse = have[k] and lo < tau < hi and r > 1 and count[k] % r != 0
            modes[k] = REUSE if reuse else STORE
            have[k] = True
            count[k] += 1
        out.append(modes)
    return out


def _seq_rows(a, B, Fr, N):
    """[T, D] rows (b, f, n) -> (B*N, F, D), the temporal block's sequences."""
    return a.reshape(B, Fr, N, -1).permute(0, 2, 1, 3).reshape(B * N, Fr, -1)


def _lib_rows(a, B, Fr, N):
    """(B*N, F, D) -> [T, D] rows (b, f, n)."""
    return a.reshape(B, N, Fr, -1).permute(0, 2, 1, 3).reshape(B * Fr * N, -1)


def forward(sd, cfg: T.T2VConfig, x, t, text, dtype=torch.float32, enable_temporal=True, text_mask=None, attn=None):
    """-> (out (B, out_channels, F, H, W), {kind: [layers, T, D] pre-gate outputs used}).  attn: None or {kind: [layers, T, D]
    or None}; a given kind is not computed but read from there (a reused cache)."""
    attn = attn or {}
    B, C, Fr, Hh, Ww = x.shape
    D, p, heads = cfg.inner_dim, cfg.patch_size, cfg.num_attention_heads
    gh, gw = Hh // p, Ww // p
    N = gh * gw
    xf = x.permute(0, 2, 1, 3, 4).reshape(B * Fr, C, Hh, Ww).to(dtype)
    patches = xf.reshape(B * Fr, C, gh, p, gw, p).permute(0, 2, 4, 1, 3, 5).reshape(B * Fr, N, C * p * p)
    h = patches @ sd["pos_embed.proj.weight"].to(dtype).reshape(D, -1).t() + sd["pos_embed.proj.bias"].to(dtype)
    h = h + R.pos_embed_table(cfg, gh, gw).to(dtype)
    ts, emb = T.adaln_single(sd, t, dtype)
    txt = T._lin(sd, "caption_projection.linear_2", F.gelu(T._lin(sd, "caption_projection.linear_1", text.to(dtype)), approximate="tanh"))
    txt_sp = txt.repeat_interleave(Fr, dim=0)
    bias_sp = None if text_mask is None else ((1 - text_mask.to(dtype)) * -10000.0).repeat_interleave(Fr, dim=0)
    ts_sp = ts.repeat_interleave(Fr, dim=0)
    ts_tm = ts.repeat_interleave(N, dim=0)
    used = {k: [] for k in KINDS}

    def given(kind, i):
        a = attn.get(kind)
        return None if a is None else a[i].to(dtype)

    for i in range(cfg.num_layers):
        # spatial block (t2v_oracle.spatial_block) with its two attention outputs exposed
        pre = f"transformer_blocks.{i}"
        sh1, sc1, g1, sh2, sc2, g2 = (sd[pre + ".scale_shift_table"].to(dtype)[None] + ts_sp.reshape(B * Fr, 6, -1)).chunk(6, dim=1)
        a = given("spatial", i)
        if a is None:
            m = LO.layer_norm(h) * (1 + sc1) + sh1
            a = T.attention(sd, pre + ".attn1", m, m, heads).reshape(-1, D)
        used["spatial"].append(a)
        h = h + g1 * a.reshape(B * Fr, N, D)
        a = given("cross", i)
        if a is None:
            a = T.attention(sd, pre + ".attn2", h, txt_sp, heads, bias_sp).reshape(-1, D)
        used["cross"].append(a)
        h = h + a.reshape(B * Fr, N, D)
        m = LO.layer_norm(h) * (1 + sc2) + sh2
        h = h + g2 * T.feed_forward(sd, pre + ".ff", m)
        if not enable_temporal:
            continue
        # temporal block (t2v_oracle.temporal_block) on sequences over frames
        h = _seq_rows(h, B, Fr, N)
        if i == 0 and Fr > 1:
            h = h + T.temp_pos_embed_table(cfg).to(dtype)
        pre = f"temporal_transformer_blocks.{i}"
        sh1, sc1, g1, sh2, sc2, g2 = (sd[pre + ".scale_shift_table"].to(dtype)[None] + ts_tm.reshape(B * N, 6, -1)).chunk(6, dim=1)
        a = given("temporal", i)
        if a is None:
            m = LO.layer_norm(h) * (1 + sc1) + sh1
            a = _lib_rows(T.attention(sd, pre + ".attn1", m, m, heads), B, Fr, N)
        used["temporal"].append(a)
        h = h + g1 * _seq_rows(a, B, Fr, N)
        m = LO.layer_norm(h) * (1 + sc2) + sh2
        h = h + g2 * T.feed_forward(sd, pre + ".ff", m)
        h = _lib_rows(h, B, Fr, N).reshape(B * Fr, N, D)
    shift, scale = (sd["scale_shift_table"].to(dtype)[None] + emb.repeat_interleave(Fr, dim=0)[:, None]).chunk(2, dim=1)
    h = LO.layer_norm(h) * (1 + scale) + shift
    h = T._lin(sd, "proj_out", h)
    h = h.reshape(B * Fr, gh, gw, p, p, cfg.out_channels)
    h = torch.einsum("nhwpqc->nchpwq", h).reshape(B * Fr, cfg.out_channels, Hh, Ww)
    out = h.reshape(B, Fr, cfg.out_channels, Hh, Ww).permute(0, 2, 1, 3, 4).contiguous()
    return out, {k: torch.stack(v) if v else None for k, v in used.items()}


def trajectory(sd, cfg, xs, taus, text, ranges, windows, **kw):
    """One call per (x, tau) under `schedule`, each reusing this oracle's own cached outputs -> the list of outputs."""
    cache, outs = {}, []
    for x, tau, modes in zip(xs, taus, schedule(taus, ranges, windows)):
        t = torch.full((x.shape[0],), int(tau), dtype=torch.int64)
        out, used = forward(sd, cfg, x, t, text, attn={k: cache[k] for k in KINDS if modes[k] == REUSE}, **kw)
        cache.update({k: used[k] for k in KINDS if modes[k] == STORE})
        outs.append(out)
    return outs
