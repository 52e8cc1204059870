"""GPU: the stages only LatteT2V runs (`b200_t2v_forward`) against fp64, one op at a time -- the timestep embedder and the
adaLN-single gemv, `t2v_mod_kernel`, the caption projection and the all-layers K/V GEMM, the cross-attention reading one
layer's K/V out of the all-layers buffer, the channels-first patch embedding with temp_pos_embed, and the output head.

Each case calls `b200_t2v_forward` with the module's packed weights (`LatteT2V._pack`) and the test's own workspace
(tests/text_workspace.py), filled with NaN bytes before each call, and reads every stage's input and output from it.  The
references take the weights from the module's parameters (cast to the 16-bit type where the kernel reads 16 bits), not
from the packed copies, so the packing is checked too.  Latte-1 width (D 1152, 16 heads x 72, caption_channels 4096);
distinct timesteps per sample (0, 1, 500, 999 among them), so a mixed-up sample index changes the result.
  * Call A, all weights random: tfreq, th, emb, ts, mod, text16, cap_h, cap_o, kv_all, the head's LayerNorm-modulated rows
    (h), the head output (head, fp32 [T, 32]) and out.
  * Call B, zero gates: the gate_msa / gate_mlp chunks (2 and 5) of adaln_single.linear and rows 2 and 5 of every
    scale_shift_table, and attn2.to_out, are zero, so every block adds exactly 0 and the workspace x after the blocks is
    patch_embed(x as (b c f h w)) + pos_embed (+ temp_pos_embed exactly when enable_temporal and F > 1), temporal on and off.
  * Strided cross-attention: b200_cross_attention on call A's kv_all at layer l (kv + 2 l D, kv_row_stride 2 L D), l = 0 and
    L - 1, with the module's -10000 text bias from an encoder_attention_mask (one prompt masked down to one token).
  * Call C, call B's zero gates with attn2.to_out nonzero in the last layer only, temporal blocks off: every other layer adds
    0, so the forward's own cross-attention of the last layer reads call B's x; its q GEMM output is left in the qkv buffer,
    and x = x + to_out(softmax(q k^T / sqrt(hd) + text bias) v) with that layer's K/V from kv_all.  This pins the layer
    offset the forward itself uses into the all-layers buffer.

Bounds (tests/fp64_bounds.py, A = 2, B = 4, F = 3): |got - ref| <= A u_out |ref| + B u_op mag + floor.  Each stage's
reference is evaluated on the exact workspace tensor the kernel read, so no error is carried between stages.
  * Sinusoid (tfreq): 2^-24 (|t freq| + 1): the fp32 argument (the reference also forms it in fp32; the kernel's expf
    frequency may differ by an ulp) and cosf / sinf, as test_gpu_forward_ops_fp64.test_conditioning.
  * gemv (th = SiLU(Linear(256, D)), emb = Linear(D, D), ts = Linear(SiLU(emb)) on 16-bit weights): sqrt(K) 2^-24
    (|W| |in| + |bias|); SiLU (fp64_bounds.silu_err) on the output of th and on the input of ts (__expf, CUDA C
    Programming Guide: 2 + 1.173 |x| ulp).
  * mod: tables + ts and final_table + emb are single fp32 adds: bit for bit.  text16 and out are a cast and a permutation:
    bit for bit.
  * GEMMs (cap_h with the GELU epilogue at K = caption_channels = 4096, cap_o, kv_all at N = 2 L D): as the forward file,
    mag = |a| |w|^T + |bias|, u_op = ACC sqrt(K) 2^-24, ACC = 1 (held to that at K = 4096 and 10240 by
    test_gpu_t5_fp64.test_accumulation_at_text_k); GELU by fp64_bounds.gelu_fwd_terms, which cannot tell GELU-tanh from
    GELU-erf.
  * Head: LayerNorm + modulate as test_gpu_forward_ops_fp64.test_ln_modulate (fp32 statistics sqrt(D) 2^-24 (rstd mean|x| +
    |xh|), three roundings of xh, one of 1 + scale and of the fma); the N = 32 head GEMM through the gated-residual epilogue
    into a zeroed fp32 buffer: A 2^-24 |ref| + B sqrt(D) 2^-24 (|h| |w| + |bias|).
  * Patch embedding (call B): the fp32 fma chain over K = C p p = 16 plus the pos and temp adds, sqrt(K + 2) 2^-24 of
    |x| |w| + |bias| + |pos| + |temp|.
  * Cross-attention: fp64_bounds.softmax_fwd_terms (max|s| over keys with nonzero probability; the fp16 subnormal floor).
    In call C its whole bound (with the 16-bit rounding of the output) goes through |Wout|, and the to_out GEMM adds
    sqrt(D) 2^-24 (|att| |Wout| + |bias|) and the residual add 2^-24 |x|.  The attention output itself is overwritten
    later in the forward, so this worst-case sum through |Wout| is loose (the largest err / bound is about 0.01); it still
    rejects another layer's K/V by a factor of 6 and more.

Latte-1 layers: L = 2 for most cases; one case runs L = 28, so the K/V GEMM runs at N = 64512, on a 16 x 16 latent video.
Text lengths 1, 9 (a single trimmed prompt) and 120 at batch 2 (a CFG pair).  Every case runs in fp16 and bf16.  The
checks reject a plausible wrong result: the neighbouring sample's ts in mod, the spatial and temporal tables swapped, sin
and cos swapped, GELU before the caption bias, K and V swapped, layer l + 1's K/V (in the strided call and in the forward's
own cross-attention), shift and scale swapped in the head,
c and f swapped in the channels-first read and write, temp_pos_embed at F = 1 or shifted by one frame.  The worst err /
bound per op and dtype is printed at the end (pytest -s)."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as Fn

import text_workspace as TW
from fp64_bounds import A, ACC, B, DTS, SUB, U16, U32, Checker, gelu_fwd_terms, report_worst, silu_err, softmax_fwd_terms

pytestmark = pytest.mark.gpu

D, HEADS, CAP, PATCH, C_IN, C_OUT = 1152, 16, 4096, 2, 4, 8
_WORST = {}
_NETS = {}


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def _module_state():
    yield
    _NETS.clear()
    report_worst(_WORST)


def _rejects(dt, op, got, ref, bound):
    m = Checker(dt)
    m.add(op, "wrong result", got, ref, bound, lambda i: str(i))
    assert m.bad, f"{op}: the bound accepts a wrong result"


def _rc(idx):
    return f"row {idx[0]}, column {idx[1]}"


def _net(dev, L, size, frames, seed):
    """A LatteT2V with fp32 parameters drawn on the device with oracle/t2v_oracle.make_weights' magnitudes (built once per
    geometry: the 28-layer model is large)."""
    from latte_b200 import LatteT2V
    key = (L, size, frames)
    if key in _NETS:
        return _NETS[key]
    _NETS.clear()
    with torch.device(dev):
        net = LatteT2V(num_attention_heads=HEADS, attention_head_dim=D // HEADS, num_layers=L, sample_size=size,
                       video_length=frames, caption_channels=CAP)
    g = torch.Generator(device=dev).manual_seed(seed)
    with torch.no_grad():
        for name, p in net.named_parameters():
            r = torch.randn(p.shape, device=dev, generator=g)
            if name.endswith(".bias"):
                r *= 0.05
            elif name.endswith("scale_shift_table"):
                r *= 4.0 / math.sqrt(p.shape[-1])
            elif name == "pos_embed.proj.weight":
                r *= 0.25
            elif name == "adaln_single.linear.weight":
                r *= 0.5 / math.sqrt(p.shape[1])
            else:
                r *= 1.0 / math.sqrt(p.shape[-1])
            p.copy_(r)
    net.eval()
    _NETS[key] = net
    return net


def _weights(T):
    from latte_b200 import _lib
    w = _lib.T2VWeights()
    for name in _lib.T2V_WEIGHT_FIELDS:
        setattr(w, name, T[name].data_ptr() if T[name] is not None else None)
    return w


def _forward(shape, T, x, t, text, bias, temporal, ws, out):
    from latte_b200 import _lib
    w = _weights(T)
    ws.poison()
    out.fill_(float("nan"))
    rc = _lib.load().b200_t2v_forward(C.byref(shape), C.byref(w), x.data_ptr(), t.data_ptr(), text.data_ptr(),
                                      bias.data_ptr() if bias is not None else None, x.shape[0], text.shape[1], int(temporal),
                                      out.data_ptr(), ws.ptr, ws.nbytes, torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, "b200_t2v_forward")
    torch.cuda.synchronize()


def _gemm(a, w, b):
    a64, w64, b64 = a.double(), w.double(), b.double()
    return a64 @ w64.t() + b64, a64.abs() @ w64.abs().t() + b64.abs()


CASES = {  # layers, latent size, video_length, timesteps, text_len, kept text tokens per sample (None: no mask)
    "L2-f4-b2-txt120-cfg": (2, 16, 4, (999, 0), 120, (120, 1)),
    "L2-f1-b1-txt9": (2, 32, 1, (500,), 9, None),
    "L2-f16-b2-txt1": (2, 16, 16, (1, 500), 1, None),
    "L28-f4-b2-txt120-cfg": (28, 16, 4, (0, 999), 120, (77, 1)),
}


@pytest.mark.parametrize("case,dt", [(c, d) for c in CASES for d in DTS], ids=lambda v: str(v).replace("torch.", ""))
def test_t2v_glue(dev, case, dt):
    from latte_b200 import _lib
    from oracle import latte_oracle as LO
    from oracle import t2v_oracle as TO
    L, size, Fr, ts_, Lt, keeps = CASES[case]
    Bn = len(ts_)
    grid = size // PATCH
    N = grid * grid
    T = Bn * Fr * N
    R = Bn * Lt
    net = _net(dev, L, size, Fr, L * 1000 + size + Fr)
    net.compute_dtype = dt
    shape, _, Tw = net._pack()
    sd = {k: v.detach() for k, v in net.state_dict().items()}
    chk = Checker(dt, _WORST)
    tag = case
    g = torch.Generator(device=dev).manual_seed(Fr * 31 + Lt)
    x = torch.randn(Bn, C_IN, Fr, size, size, device=dev, generator=g)
    t = torch.tensor(ts_, dtype=torch.int64, device=dev)
    text = torch.randn(Bn, Lt, CAP, device=dev, generator=g) * 0.5
    bias = None
    if keeps is not None:      # the module's (1 - mask) * -10000 over 128 columns
        mask = (torch.arange(Lt, device=dev)[None] < torch.tensor(keeps, device=dev)[:, None]).float()
        bias = torch.zeros(Bn, 128, device=dev)
        bias[:, :Lt] = (1.0 - mask) * -10000.0
    ws = TW.Workspace(TW.t2v_layout(L, D, 4 * D, PATCH, C_OUT, size, Fr, CAP, Bn, Lt, dt), dev)
    out = torch.empty(Bn, C_OUT, Fr, size, size, device=dev)

    # ================================================================ call A
    _forward(shape, Tw, x, t, text, bias, True, ws, out)

    # ---- timestep embedder: tfreq, th, emb
    freqs = torch.exp(-math.log(10000) * torch.arange(0, 128, dtype=torch.float32, device=dev) / 128)
    arg = (t[:, None].float() * freqs[None]).double()
    ref = torch.cat([torch.cos(arg), torch.sin(arg)], 1)
    bnd = A * U32 * ref.abs() + B * U32 * (torch.cat([arg, arg], 1).abs() + 1)
    chk.add("tfreq sinusoid", tag, ws["tfreq"], ref, bnd, _rc)
    _rejects(dt, "tfreq: sin and cos swapped", ref.roll(128, 1), ref, bnd)
    assert torch.allclose(ref, LO.timestep_embedding(t.cpu()).double().to(dev), atol=1e-4)
    pre = "adaln_single.emb.timestep_embedder."
    h1, mag = _gemm(ws["tfreq"], sd[pre + "linear_1.weight"], sd[pre + "linear_1.bias"])
    ref = Fn.silu(h1)
    chk.add("gemv Linear(256, D) + SiLU (th)", tag, ws["th"], ref,
            A * U32 * ref.abs() + B * silu_err(h1, math.sqrt(256) * U32 * mag), _rc)
    ref, mag = _gemm(ws["th"], sd[pre + "linear_2.weight"], sd[pre + "linear_2.bias"])
    chk.add("gemv Linear(D, D) (emb)", tag, ws["emb"], ref, A * U32 * ref.abs() + B * math.sqrt(D) * U32 * mag, _rc)

    # ---- ts = Linear(SiLU(emb)) on the 16-bit adaLN weight
    e64 = ws["emb"].double()
    w16 = sd["adaln_single.linear.weight"].to(dt).double()
    sc = Fn.silu(e64)
    ref = sc @ w16.t() + sd["adaln_single.linear.bias"].double()
    e = silu_err(e64, torch.zeros_like(e64)) @ w16.abs().t() + \
        math.sqrt(D) * U32 * (sc.abs() @ w16.abs().t() + sd["adaln_single.linear.bias"].double().abs())
    chk.add("gemv adaLN-single, 16-bit weight (ts)", tag, ws["ts"], ref, A * U32 * ref.abs() + B * e, _rc)

    # ---- mod = tables + ts (blocks interleaved spatial, temporal), then final_table + emb: fp32 adds, bit for bit
    spat = [sd[f"transformer_blocks.{i}.scale_shift_table"] for i in range(L)]
    temp = [sd[f"temporal_transformer_blocks.{i}.scale_shift_table"] for i in range(L)]

    def mod_of(tables, tsr, emb):
        blocks = torch.stack(tables).reshape(2 * L, 6 * D)[None] + tsr[:, None, :]
        fin = sd["scale_shift_table"][None] + emb[:, None, :]
        return torch.cat([blocks.reshape(Bn, -1), fin.reshape(Bn, -1)], 1)
    inter = [tb for pair in zip(spat, temp) for tb in pair]
    want = mod_of(inter, ws["ts"], ws["emb"])
    assert torch.equal(ws["mod"], want), f"{tag}: mod != tables + ts ({int((ws['mod'] != want).sum())} elements)"
    swapped = [tb for pair in zip(temp, spat) for tb in pair]
    assert not torch.equal(ws["mod"], mod_of(swapped, ws["ts"], ws["emb"])), "mod check accepts swapped tables"
    if Bn > 1:
        assert not torch.equal(ws["mod"], mod_of(inter, ws["ts"].roll(1, 0), ws["emb"])), "mod check accepts a neighbour's ts"

    # ---- caption projection and the all-layers K/V GEMM
    assert torch.equal(ws["text16"], text.reshape(R, CAP).to(dt)), f"{tag}: text16 != text.to({dt})"
    cw1, cb1 = sd["caption_projection.linear_1.weight"].to(dt), sd["caption_projection.linear_1.bias"]
    pre1, mag = _gemm(ws["text16"], cw1, cb1)
    ref, term = gelu_fwd_terms(pre1, ACC * math.sqrt(CAP) * U32, mag)
    bnd = A * U16[dt] * ref.abs() + term + SUB[dt]
    chk.add(f"caption fc1 + GELU K={CAP}", tag, ws["cap_h"], ref, bnd, _rc)
    late, _ = gelu_fwd_terms(pre1 - cb1.double(), 0.0, mag)
    _rejects(dt, "caption fc1: GELU before the bias", (ws["cap_h"].double() + late + cb1.double() - ref).to(dt), ref, bnd)
    del pre1, mag, term, late

    ref, mag = _gemm(ws["cap_h"], sd["caption_projection.linear_2.weight"].to(dt), sd["caption_projection.linear_2.bias"])
    chk.add(f"caption fc2 K={D}", tag, ws["cap_o"], ref,
            A * U16[dt] * ref.abs() + B * ACC * math.sqrt(D) * U32 * mag + SUB[dt], _rc)
    kvw = torch.cat([torch.cat([sd[f"transformer_blocks.{i}.attn2.to_k.weight"], sd[f"transformer_blocks.{i}.attn2.to_v.weight"]])
                     for i in range(L)]).to(dt)
    kvb = torch.cat([torch.cat([sd[f"transformer_blocks.{i}.attn2.to_k.bias"], sd[f"transformer_blocks.{i}.attn2.to_v.bias"]])
                     for i in range(L)])
    ref, mag = _gemm(ws["cap_o"], kvw, kvb)
    bnd = A * U16[dt] * ref.abs() + B * ACC * math.sqrt(D) * U32 * mag + SUB[dt]
    del kvw, mag
    chk.add(f"K/V of all layers N={2 * L * D}", tag, ws["kv_all"], ref, bnd, _rc)
    kv_swapped = ws["kv_all"].reshape(R, L, 2, D).flip(2).reshape(R, 2 * L * D)
    _rejects(dt, "kv_all: K and V swapped", kv_swapped, ref, bnd)
    del ref, bnd, kv_swapped

    # ---- output head: LN + modulate from the final slot of mod, the N = 32 GEMM, unpatchify to (b c f h w)
    fin = ws["mod"][:, 2 * L * 6 * D:].double()
    bidx = torch.arange(T, device=dev) // (Fr * N)
    shift, scale = fin[bidx, :D], fin[bidx, D:]
    x64 = ws["x"].double()
    mean = x64.mean(1, keepdim=True)
    rstd = (((x64 - mean) ** 2).mean(1, keepdim=True) + 1e-6).rsqrt()
    xh = (x64 - mean) * rstd
    ref = xh * (1 + scale) + shift
    c1 = (1 + scale).abs()
    e_xh = U32 * (math.sqrt(D) * (rstd * x64.abs().mean(1, keepdim=True) + xh.abs()) + 3 * xh.abs())
    bnd = A * U16[dt] * ref.abs() + B * (c1 * e_xh + U32 * (2 * xh.abs() * c1 + shift.abs())) + SUB[dt]
    chk.add("head LayerNorm + modulate", tag, ws["h"], ref, bnd, _rc)
    _rejects(dt, "head: shift and scale swapped", (ws["h"].double() + xh * (1 + shift) + scale - ref).to(dt), ref, bnd)
    del x64, mean, xh, e_xh, c1, shift, scale, ref, bnd

    n_out = PATCH * PATCH * C_OUT
    head = ws["head"][:T * n_out].reshape(T, n_out)
    assert torch.equal(ws["head"][T * n_out:(T + 1) * n_out], torch.ones(n_out, device=dev))
    ref, mag = _gemm(ws["h"], sd["proj_out.weight"].to(dt), sd["proj_out.bias"])
    chk.add(f"head GEMM N={n_out} K={D}", tag, head, ref, A * U32 * ref.abs() + B * math.sqrt(D) * U32 * mag, _rc)
    want = head.reshape(Bn, Fr, grid, grid, PATCH, PATCH, C_OUT).permute(0, 6, 1, 2, 4, 3, 5).reshape(out.shape)
    assert torch.equal(out, want), f"{tag}: out is not the (b c f h w) unpatchify of head"
    if Fr > 1:
        assert not torch.equal(out, want.transpose(1, 2).contiguous().reshape(out.shape)), "out check accepts c and f swapped"

    # ---- cross-attention on layer l's K/V in the all-layers buffer (kv_row_stride = 2 L D)
    hd = D // HEADS
    kb = bias if bias is not None else torch.zeros(Bn, 128, device=dev)
    q = torch.randn(Bn * 256, D, device=dev, generator=g)
    q[::7] *= 4                                                       # logits up to ~+-30
    q = q.to(dt)
    kv5 = ws["kv_all"].double().reshape(Bn, Lt, L, 2, HEADS, hd)
    q4 = q.double().reshape(Bn, 256, HEADS, hd).transpose(1, 2)
    for lay in sorted({0, L - 1}):
        got = torch.empty_like(q)
        kv_ptr = ws["kv_all"].data_ptr() + 2 * lay * D * ws["kv_all"].element_size()
        rc = _lib.load().b200_cross_attention(q.data_ptr(), kv_ptr, kb.data_ptr(), got.data_ptr(), Bn, 256, Lt, D, 2 * L * D,
                                              HEADS, hd, _lib.BF16 if dt == torch.bfloat16 else _lib.FP16,
                                              torch.cuda.current_stream().cuda_stream)
        _lib.check(rc, "b200_cross_attention")
        torch.cuda.synchronize()
        got4 = got.reshape(Bn, 256, HEADS, hd).transpose(1, 2)
        for b in range(Bn):
            k4, v4 = kv5[b, :, lay, 0].transpose(0, 1), kv5[b, :, lay, 1].transpose(0, 1)        # [H, Lt, hd]
            kbb = kb[b, :Lt].double()[None, None, :]
            ref, term, _ = softmax_fwd_terms(q4[b], k4, v4, kbb, dt)
            bnd = A * U16[dt] * ref.abs() + term

            def where(i, b=b, lay=lay):
                return f"layer {lay}, sample {b}, head {i[0]}, query {i[1]}, dim {i[2]}"
            chk.add("cross-attention, layer K/V strided in kv_all", tag, got4[b], ref, bnd, where)
            other = lay + 1 if lay + 1 < L else lay - 1
            alt, _, _ = softmax_fwd_terms(q4[b], kv5[b, :, other, 0].transpose(0, 1), kv5[b, :, other, 1].transpose(0, 1), kbb, dt)
            _rejects(dt, f"cross-attention: layer {other}'s K/V for layer {lay}", (got4[b].double() + alt - ref).to(dt), ref, bnd)
            alt, _, _ = softmax_fwd_terms(q4[b], v4, k4, kbb, dt)
            _rejects(dt, "cross-attention: K and V swapped", (got4[b].double() + alt - ref).to(dt), ref, bnd)
    del kv5, q4, kb

    # ================================================================ call B: zero gates, every block adds exactly 0
    Tb = dict(Tw)
    ada_w, ada_b = Tw["ada_w16"].clone(), Tw["ada_b"].clone()
    tables = Tw["tables"].clone()
    for c in (2, 5):
        ada_w[c * D:(c + 1) * D] = 0
        ada_b[c * D:(c + 1) * D] = 0
        tables[:, c] = 0
    Tb.update(ada_w16=ada_w, ada_b=ada_b, tables=tables, c_out_w16=torch.zeros_like(Tw["c_out_w16"]),
              c_out_b=torch.zeros_like(Tw["c_out_b"]))
    cfg = TO.T2VConfig(num_attention_heads=HEADS, attention_head_dim=hd, num_layers=L, sample_size=size, video_length=Fr,
                       caption_channels=CAP)
    pos = TO.pos_embed_table(cfg).to(dev).double()                                 # [N, D]
    tmp = TO.temp_pos_embed_table(cfg).to(dev).double()                            # [F, D]
    wp = sd["pos_embed.proj.weight"].double().reshape(D, -1)
    bp = sd["pos_embed.proj.bias"].double()
    K = wp.shape[1]

    def embed(xin):        # xin (b f c h w) -> [(b f n), D] patch_embed + pos, and its magnitude
        xp = xin.double().reshape(Bn * Fr, C_IN, grid, PATCH, grid, PATCH).permute(0, 2, 4, 1, 3, 5).reshape(Bn * Fr, N, K)
        return (xp @ wp.t() + bp + pos).reshape(T, D), (xp.abs() @ wp.abs().t() + bp.abs() + pos.abs()).reshape(T, D)
    base, mag = embed(x.permute(0, 2, 1, 3, 4))
    frame = (torch.arange(T, device=dev) // N) % Fr
    for temporal in (True, False):
        _forward(shape, Tb, x, t, text, bias, temporal, ws, out)
        if not temporal:
            x_emb = ws["x"].clone()
        with_temp = temporal and Fr > 1
        ref = base + tmp[frame] if with_temp else base
        bnd = A * U32 * ref.abs() + B * math.sqrt(K + 2) * U32 * (mag + (tmp[frame].abs() if with_temp else 0))
        name = f"patch embed + pos{' + temp' if with_temp else ''} (zero-gate blocks)"
        chk.add(name, f"{tag} temporal={temporal}", ws["x"], ref, bnd, _rc)
        if Fr > 1:
            wrong, _ = embed(x.reshape(Bn, Fr, C_IN, size, size))
            _rejects(dt, "patch embed: c and f swapped in the read", wrong + (ref - base), ref, bnd)
        if with_temp:
            _rejects(dt, "temp_pos_embed shifted by one frame", base + tmp[(frame + 1) % Fr], ref, bnd)
        elif temporal:
            _rejects(dt, "temp_pos_embed added at F = 1", base + tmp[frame], ref, bnd)
    del base, mag, ref, bnd

    # ================================================================ call C: call B with attn2.to_out of the last layer only
    # Every layer but the last adds 0, so the last layer's cross-attention reads x_emb (call B's x without temporal
    # blocks, bit for bit the same computation), its q is left in the qkv buffer, and x = x_emb + to_out(cross-attention).
    lc = L - 1
    pre = f"transformer_blocks.{lc}.attn2."
    c_out_w, c_out_b = torch.zeros_like(Tw["c_out_w16"]), torch.zeros_like(Tw["c_out_b"])
    c_out_w[lc] = sd[pre + "to_out.0.weight"].to(dt)
    c_out_b[lc * D:(lc + 1) * D] = sd[pre + "to_out.0.bias"]
    _forward(shape, dict(Tb, c_out_w16=c_out_w, c_out_b=c_out_b), x, t, text, bias, False, ws, out)
    q16 = ws["qkv"].reshape(-1)[:T * D].reshape(T, D)
    ref, mag = _gemm(x_emb.to(dt), sd[pre + "to_q.weight"].to(dt), sd[pre + "to_q.bias"])
    chk.add(f"cross-attention q GEMM K={D}", tag, q16, ref, A * U16[dt] * ref.abs() + B * math.sqrt(D) * U32 * mag + SUB[dt], _rc)
    kv5 = ws["kv_all"].double().reshape(Bn, Lt, L, 2, HEADS, hd)
    q4 = q16.double().reshape(Bn, Fr * N, HEADS, hd).transpose(1, 2)
    kbias = bias if bias is not None else torch.zeros(Bn, 128, device=dev)
    wo = sd[pre + "to_out.0.weight"].to(dt).double()
    bo = sd[pre + "to_out.0.bias"].double()

    def rows(a):                         # [Bn, H, F N, hd] -> [T, D]
        return a.transpose(1, 2).reshape(T, D)

    def attend(layer):
        outs = [softmax_fwd_terms(q4[b], kv5[b, :, layer, 0].transpose(0, 1), kv5[b, :, layer, 1].transpose(0, 1),
                                  kbias[b, :Lt].double()[None, None, :], dt)[:2] for b in range(Bn)]
        return rows(torch.stack([o[0] for o in outs])), rows(torch.stack([o[1] for o in outs]))
    att, term = attend(lc)
    ref = x_emb.double() + att @ wo.t() + bo
    e_att = A * U16[dt] * att.abs() + term
    bnd = A * U32 * ref.abs() + e_att @ wo.abs().t() + B * U32 * (math.sqrt(D) * (att.abs() @ wo.abs().t() + bo.abs()) + x_emb.double().abs())
    chk.add(f"forward cross-attention, layer {lc} of {L} + to_out", tag, ws["x"], ref, bnd, _rc)
    if L > 1:
        other, _ = attend((lc + 1) % L)
        _rejects(dt, "forward cross-attention: another layer's K/V", ws["x"].double() + (other - att) @ wo.t(), ref, bnd)
    chk.done()
