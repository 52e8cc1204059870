"""GPU: the T5 encoder (`b200_t5_encode`) against fp64, one op at a time -- the embedding gather, RMSNorm with 16-bit and
fp32 output, the QKV GEMM, the unscaled attention with T5's position bias and the padding mask, the gated-GELU feed-forward
(GELU epilogue, then the MUL16 epilogue) and the two gated-residual GEMMs into the fp32 stream.

Each case runs a one-layer encoder twice with the module's packed weights (`T5EncoderModel._pack`) and the test's own
workspace (tests/text_workspace.py), filled with NaN bytes before each call.  After a call the workspace still holds x (the
fp32 residual after the layer), h (the second RMSNorm's output), qkv, att, g0 and g, and each is compared with its op in
fp64 evaluated on the exact tensors the kernel read.
  * Call 1 isolates the QKV input: o = 0, wo = 0 and ln1's weight equal to ln0's, so the residual is the embedding
    throughout (x += 1 * 0 is exact) and h, the ln1 output, is bit for bit the ln0 output the QKV GEMM read.  It pins the
    embedding (x == table[ids], bit for bit), RMSNorm -> 16 bits (h), the QKV GEMM (qkv) and RMSNorm -> fp32 (out).
  * Call 2, all weights random, pins the attention (att), gelu(h wi_0^T) (g0), the MUL16 product (g), RMSNorm of the
    non-trivial residual embed + att Wo^T (h), the two residual GEMMs (x) and the final norm (out).

Bounds (tests/fp64_bounds.py, A = 2, B = 4, F = 3): |got - ref| <= A u_out |ref| + B u_op mag + floor.
  * RMSNorm y = x rsqrt(mean x^2 + eps) w: the fp32 sum of D squares is off by at most sqrt(D) 2^-24 relative (the squares
    are positive; each lane sums D / 128 float4 groups before a 5-step butterfly, so even the worst case, (D / 128 + 6)
    roundings, stays below sqrt(D)), the division by D and the eps add one rounding each; rsqrtf halves that relative error and
    adds its own 2 ulp (CUDA C Programming Guide: rsqrtf is not correctly rounded; 2 ulp <= 4 * 2^-24 relative); x r w two
    products: u_op = 2^-24 (sqrt(D) / 2 + 8), mag = |y|.  An input error e (the o-GEMM's, on the non-trivial residual) moves y
    by |w| r (e + |xh| mean(|xh| e)), xh = x r.  One token of every sample has its embedding row scaled by 1e-3, so its mean
    square is near eps and an eps of 1e-5 instead of 1e-6 moves its output by half.
  * GEMM (QKV, K = d_model): mag = |a| |w|^T, u_op = ACC sqrt(K) 2^-24 with ACC = 1, as in test_gpu_forward_ops_fp64.py.
    That file measured ACC up to K = 4608; `test_accumulation_at_text_k` extends the table to the encoder's K = 4096
    (t5-v1_1-xxl qkv / wi and o, caption_channels) and 10240 (wo), same inputs and schedule (M = 8192, N = 1152, three
    +-60 outliers per row), on an H100 80GB HBM3 at a 700 W power limit:

        K                                4096    10240
        fp16 err / (2^-24 mag)           20.9    22.6     / sqrt(K): 0.33  0.22
        bf16 err / (2^-24 mag)           17.9    20.8     / sqrt(K): 0.28  0.21

    The ratio to sqrt(K) keeps falling past K = 4608, so ACC = 1 and the sqrt(K) form hold at the text path's K with
    room to spare; the test holds the accumulation to B sqrt(K) on every run.
  * Gated GELU.  g0 = gelu_tanh(h wi_0^T) through the GELU epilogue: fp64_bounds.gelu_fwd_terms (tanh.approx.f32, the
    fp32 argument, the accumulation through |gelu'|); that bound cannot tell GELU-tanh from GELU-erf (the tanh.approx term
    is as large as their difference).  g = round16(round16(h wi_1^T) g0): the MUL16 epilogue rounds twice by design, as
    transformers' fp16 product of two 16-bit tensors does; the first factor's rounding and accumulation are carried through
    |g0| (A u16 |pre1| + B u_acc mag1 + a 2^-24 fp16 subnormal floor), the product's rounding is A u16 |g|.
  * Residual GEMMs.  x = embed + att Wo^T (K = inner) + g Wwo^T (K = d_ff), each through the gated-residual epilogue with
    gate 1 into fp32: B 2^-24 (sqrt(inner) |att| |Wo| + sqrt(d_ff) |g| |Wwo| + |embed| + |embed + att Wo^T|) -- the two
    accumulations, plus the two fp32 adds (and stream-K's segment adds, fewer than sqrt(K)).
  * Attention (scale 1, the position bias of head h and the -1e30 padding mask added to the scores):
    fp64_bounds.softmax_fwd_terms.  The fp32 exp2 argument term uses max|s| over keys with nonzero probability only; the
    padding keys get exactly 0 in fp64 and in the kernel (ex2 of about -1.4e30), and with them in max|s| the bound would be
    ~1e23.  fp16 adds the subnormal floor of the rounded probabilities (sqfloor).

Shapes: a tiny encoder (d_model 256, 4 heads, d_ff 512) at batch 1, 2 and 3, and one t5-v1_1-xxl layer (d_model 4096, 64
heads x 64, d_ff 10240, vocab 512) at batch 2; kept prompt lengths 1, 9, 120 and 128 (no padding row), padding ids 0,
ids 0 and vocab - 1 present; logits up to about +-30 (the query rows of a quarter of the heads scaled by 6), position biases
up to +-10.  The position bias is rebuilt here from the oracle's bucket function, not taken from the module.  Every case runs
in fp16 and bf16.  Each op's bound rejects a plausible wrong result: a neighbour's embedding row, eps 1e-5, the position
bias transposed, the scores scaled by 1/8 (both on samples with more than one kept token: with one, the output is v_0
whatever the scores), the padding mask ignored, GELU on the wi_1 factor, ln0's weight in ln1, one 64-wide K segment of the
d_ff residual GEMM dropped.  The worst err / bound per op and dtype is printed at the end
(pytest -s)."""
import ctypes as C
import math

import pytest
import torch

import text_workspace as TW
from fp64_bounds import A, ACC, B, DTS, SUB, U16, U32, Checker, dtn, gelu_fwd_terms, report_worst, softmax_fwd_terms

pytestmark = pytest.mark.gpu

EPS = 1e-6
_WORST = {}
_ACC_TABLE = {}


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    if _ACC_TABLE:
        print("\nfp32 tensor-core accumulation at the encoder's K: worst err / (2^-24 mag), and that / sqrt(K):")
        for (dt, K), r in sorted(_ACC_TABLE.items()):
            print(f"  {dt:<9} K = {K:5d}   {r:8.3g}   {r / math.sqrt(K):8.3g}")
    report_worst(_WORST)


def _rejects(dt, op, got, ref, bound):
    m = Checker(dt)
    m.add(op, "wrong result", got, ref, bound, lambda i: str(i))
    assert m.bad, f"{op}: the bound accepts a wrong result"


def _rc(idx):
    return f"row {idx[0]} (sample {idx[0] // 128}, position {idx[0] % 128}), column {idx[1]}"


def _rms_ref(x64, w64, eps=EPS):
    r = ((x64 * x64).mean(-1, keepdim=True) + eps).rsqrt()
    return x64 * r * w64, r


def _rms_bound(ref, D, dt_out):
    """A u_out |y| + B 2^-24 (sqrt(D) / 2 + 8) |y| (+ the fp16 floor for a 16-bit output)."""
    u_out = U32 if dt_out is None else U16[dt_out]
    return A * u_out * ref.abs() + B * U32 * (math.sqrt(D) / 2 + 8) * ref.abs() + (SUB[dt_out] if dt_out is not None else 0.0)


def _gemm_ref(a, w):
    a64, w64 = a.double(), w.double()
    return a64 @ w64.t(), a64.abs() @ w64.abs().t()


def _pos_bias(table):
    """[H, 128, 128]: relative_attention_bias[bucket(j - i)][h], bucketed by the oracle."""
    from oracle import t5_oracle as T
    pos = torch.arange(128)
    bk = T.relative_position_bucket(pos[None, :] - pos[:, None], 32, 128).to(table.device)
    return table[bk].permute(2, 0, 1).contiguous()


CASES = {  # d_model, heads, d_ff, vocab, kept tokens per sample
    "tiny-b1-keep128": (256, 4, 512, 100, [128]),
    "tiny-b2-keep9-120": (256, 4, 512, 100, [9, 120]),
    "tiny-b3-keep1-9-128": (256, 4, 512, 100, [1, 9, 128]),
    "xxl-b2-keep120-1": (4096, 64, 10240, 512, [120, 1]),
}


def _setup(dev, dt, d_model, heads, d_ff, vocab, keeps, seed):
    from latte_b200 import T5EncoderModel
    from oracle import t5_oracle as T
    cfg = T.T5Cfg(vocab_size=vocab, d_model=d_model, d_ff=d_ff, num_layers=1, num_heads=heads)
    sd = T.make_weights(cfg, seed)
    g = torch.Generator().manual_seed(seed + 1)
    sd["encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"] = \
        (torch.randn(32, heads, generator=g) * 4).clamp(-10, 10)
    sd["encoder.block.0.layer.0.SelfAttention.q.weight"][: heads // 4 * 64] *= 6.0        # logits up to ~+-30
    sd["shared.weight"][1] *= 1e-3                                                         # mean square near eps
    with torch.device(dev):
        net = T5EncoderModel(vocab_size=vocab, d_model=d_model, d_ff=d_ff, num_layers=1, num_heads=heads)
    net.load_state_dict(sd, strict=True)
    net.eval().compute_dtype = dt                       # fp32 parameters, 16-bit GEMM operands
    shape, _, Tw, pos = net._pack()
    Bn = len(keeps)
    ids = torch.zeros(Bn, 128, dtype=torch.int64)
    bias = torch.full((Bn, 128), -1e30)                  # the module's extended attention mask on 128 padded columns
    L = max(keeps)
    for b, keep in enumerate(keeps):
        ids[b, :keep] = torch.randint(2, vocab, (keep,), generator=g)
        bias[b, :L] = torch.where(torch.arange(L) < keep, 0.0, -1e30)
        ids[b, 1] = 1                                    # the 1e-3 row
    ids[0, 2] = vocab - 1
    ids[-1, 0] = 0
    assert int(ids.min()) >= 0 and int(ids.max()) < vocab       # embed_kernel traps on an out-of-range id
    table = sd["encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"].to(dev)
    pos_ref = _pos_bias(table)
    assert torch.equal(pos, pos_ref), "the module's position bias is not relative_attention_bias[bucket(j - i)]"
    return shape, Tw, pos, ids.to(dev), bias.to(dev)


def _encode(shape, Tw, ids, bias, pos, ws, out):
    from latte_b200 import _lib
    w = _lib.T5Weights()
    for name in _lib.T5_WEIGHT_FIELDS:
        setattr(w, name, Tw[name].data_ptr())
    ws.poison()
    out.fill_(float("nan"))
    rc = _lib.load().b200_t5_encode(C.byref(shape), C.byref(w), ids.data_ptr(), bias.data_ptr(), pos.data_ptr(), ids.shape[0],
                                    out.data_ptr(), ws.ptr, ws.nbytes, torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, "b200_t5_encode")
    torch.cuda.synchronize()


@pytest.mark.parametrize("case,dt", [(c, d) for c in CASES for d in DTS], ids=lambda v: str(v).replace("torch.", ""))
def test_t5_layer_ops(dev, case, dt):
    d_model, heads, d_ff, vocab, keeps = CASES[case]
    D, H, I, FF, Bn = d_model, heads, heads * 64, d_ff, len(keeps)
    R = Bn * 128
    shape, Tw, pos, ids, bias = _setup(dev, dt, d_model, heads, d_ff, vocab, keeps, sum(keeps) + d_model)
    assert float(shape.eps) == pytest.approx(EPS)
    ws = TW.Workspace(TW.t5_layout(D, H, FF, Bn, dt), dev)
    out = torch.empty(Bn, 128, D, device=dev)
    chk = Checker(dt, _WORST)
    tag = f"{case}"
    emb16 = Tw["embed16"][ids.reshape(-1)]
    emb64 = emb16.double()

    # ---------------------------------------------------------------- call 1: o = 0, wo = 0, ln1 = ln0
    T1 = dict(Tw, o_w16=torch.zeros_like(Tw["o_w16"]), wo_w16=torch.zeros_like(Tw["wo_w16"]), ln1_w=Tw["ln0_w"].clone())
    _encode(shape, T1, ids, bias, pos, ws, out)
    x = ws["x"]
    assert torch.equal(x, emb16.float()), f"{tag}: embedding != table[ids] ({int((x != emb16.float()).sum())} elements)"
    wrong = emb16.float().clone()
    wrong[1] = Tw["embed16"][(ids.reshape(-1)[1] + 1) % vocab].float()
    assert not torch.equal(x, wrong), "the embedding check accepts a neighbour's row"

    w0 = Tw["ln0_w"][0].double()
    ref_h, _ = _rms_ref(emb64, w0)
    bnd_h = _rms_bound(ref_h, D, dt)
    chk.add("rms_norm -> 16-bit", tag, ws["h"], ref_h, bnd_h, _rc)
    eps5, _ = _rms_ref(emb64, w0, 1e-5)
    _rejects(dt, "rms_norm: eps 1e-5", (ws["h"].double() + eps5 - ref_h).to(dt), ref_h, bnd_h)

    ref_q, mag_q = _gemm_ref(ws["h"], Tw["qkv_w16"][0])
    bnd_q = A * U16[dt] * ref_q.abs() + B * ACC * math.sqrt(D) * U32 * mag_q + SUB[dt]
    chk.add(f"qkv GEMM K={D}", tag, ws["qkv"], ref_q, bnd_q, _rc)
    del ref_q, mag_q, bnd_q

    wf = Tw["final_w"].double()
    ref_o, _ = _rms_ref(emb64, wf)
    bnd_o = _rms_bound(ref_o, D, None)
    chk.add("rms_norm -> fp32 (final)", tag, out.reshape(R, D), ref_o, bnd_o, _rc)
    eps5, _ = _rms_ref(emb64, wf, 1e-5)
    _rejects(dt, "final rms_norm: eps 1e-5", out.reshape(R, D).double() + eps5 - ref_o, ref_o, bnd_o)
    del ref_o, bnd_o, eps5

    # ---------------------------------------------------------------- call 2: every weight random
    _encode(shape, Tw, ids, bias, pos, ws, out)
    qkv = ws["qkv"].double().reshape(Bn, 128, 3, H, 64).permute(2, 0, 3, 1, 4)      # [3, B, H, S, 64]
    att = ws["att"].reshape(Bn, 128, H, 64).transpose(1, 2)
    pos64 = pos.double()
    for b in range(Bn):
        q, k, v = qkv[0, b], qkv[1, b], qkv[2, b]
        kb = bias[b].double()[None, None, :]
        ref, term, _ = softmax_fwd_terms(q, k, v, pos64 + kb, dt, scale=1.0)
        bnd = A * U16[dt] * ref.abs() + term

        def where(i, b=b):
            return f"sample {b}, head {i[0]}, query {i[1]}, dim {i[2]}"
        chk.add("attention pos_bias + mask, scale 1", tag, att[b], ref, bnd, where)
        got = att[b].double()
        for name, wb, sc in (("position bias transposed", pos64.transpose(-1, -2) + kb, 1.0),
                             ("scores scaled by 1/8", pos64 + kb, 0.125),
                             ("padding mask ignored", pos64, 1.0)):
            if keeps[b] == 1 and name != "padding mask ignored":
                continue          # one key: the output is v_0 whatever the scores are
            if name == "padding mask ignored" and keeps[b] == 128:
                continue
            alt, _, _ = softmax_fwd_terms(q, k, v, wb, dt, scale=sc)
            _rejects(dt, f"attention: {name}", (got + alt - ref).to(dt), ref, bnd)
        del ref, term, bnd
    del qkv, att

    h2 = ws["h"]
    # ln1 input: x1 = embed + att Wo^T, with the o-GEMM's error carried through the norm
    o_ref, o_mag = _gemm_ref(ws["att"], Tw["o_w16"][0])
    x1 = emb64 + o_ref
    e_x1 = U32 * (math.sqrt(I) * o_mag + x1.abs())
    w1 = Tw["ln1_w"][0].double()
    ref_h, r = _rms_ref(x1, w1)
    xh = x1 * r
    e_y = w1.abs() * r * (e_x1 + xh.abs() * (xh.abs() * e_x1).mean(-1, keepdim=True))
    bnd_h = _rms_bound(ref_h, D, dt) + B * e_y
    chk.add("rms_norm -> 16-bit, residual after attention", tag, h2, ref_h, bnd_h, _rc)
    wrong_ln, _ = _rms_ref(x1, w0)
    _rejects(dt, "rms_norm: ln0's weight in ln1", (h2.double() + wrong_ln - ref_h).to(dt), ref_h, bnd_h)
    del ref_h, bnd_h, e_y, xh, wrong_ln

    uacc = ACC * math.sqrt(D) * U32
    pre0, mag0 = _gemm_ref(h2, Tw["wi0_w16"][0])
    ref_g0, term = gelu_fwd_terms(pre0, uacc, mag0)
    bnd_g0 = A * U16[dt] * ref_g0.abs() + term + SUB[dt]
    chk.add(f"wi_0 GEMM + GELU K={D}", tag, ws["g0"], ref_g0, bnd_g0, _rc)
    del term, bnd_g0, mag0

    pre1, mag1 = _gemm_ref(h2, Tw["wi1_w16"][0])
    g0 = ws["g0"].double()
    ref_g = pre1 * g0
    bnd_g = A * U16[dt] * ref_g.abs() + g0.abs() * (A * U16[dt] * pre1.abs() + B * uacc * mag1 + SUB[dt]) + SUB[dt]
    chk.add(f"wi_1 GEMM * g0 (MUL16) K={D}", tag, ws["g"], ref_g, bnd_g, _rc)
    gelu1, _ = gelu_fwd_terms(pre1, uacc, mag1)
    _rejects(dt, "gated GELU: GELU on the wi_1 factor", (ws["g"].double() + gelu1 * pre0 - ref_g).to(dt), ref_g, bnd_g)
    del pre0, pre1, mag1, g0, ref_g, bnd_g, gelu1, ref_g0

    f_ref, f_mag = _gemm_ref(ws["g"], Tw["wo_w16"][0])
    ref_x = x1 + f_ref
    bnd_x = A * U32 * ref_x.abs() + B * U32 * (math.sqrt(I) * o_mag + math.sqrt(FF) * f_mag + emb64.abs() + x1.abs())
    chk.add(f"o (K={I}) + wo (K={FF}) residual GEMMs", tag, ws["x"], ref_x, bnd_x, _rc)
    seg = slice(FF - 64, FF)
    drop = ws["g"][:, seg].double() @ Tw["wo_w16"][0][:, seg].double().t()
    _rejects(dt, "residual GEMM: last K segment of d_ff dropped", ws["x"].double() - drop, ref_x, bnd_x)
    del f_ref, f_mag, o_ref, o_mag, x1, e_x1, bnd_x, drop

    xf = ws["x"].double()
    ref_o, _ = _rms_ref(xf, wf)
    chk.add("rms_norm -> fp32 (final)", tag, out.reshape(R, D), ref_o, _rms_bound(ref_o, D, None), _rc)
    chk.done()


def _outliers(M, K, g, dev):
    x = torch.randn(M, K, device=dev, generator=g)
    cols = torch.randint(0, K, (M, 3), device=dev, generator=g)
    sign = torch.randint(0, 2, (M, 3), device=dev, generator=g).float() * 2 - 1
    return x.scatter_(1, cols, 60.0 * sign)


@pytest.mark.parametrize("dt", DTS)
def test_accumulation_at_text_k(dev, dt):
    """The forward GEMM's fp32 accumulation alone at the text path's K, as test_gpu_forward_ops_fp64.test_gemm_accumulation
    measures it up to K = 4608: x = 0 + 1 * (a w^T) through the gated-residual epilogue on the data-parallel schedule,
    M = 8192, N = 1152, three +-60 outliers per row of a, at K = 4096 and 10240.  Records worst err / (2^-24 mag) per K and
    holds it to B * ACC * sqrt(K)."""
    from latte_b200 import ops
    chk = Checker(dt, _WORST)
    M, N = 8192, 1152
    for K in (4096, 10240):
        g = torch.Generator(device=dev).manual_seed(K)
        a = _outliers(M, K, g, dev).to(dt)
        lim = math.sqrt(6.0 / (K + N))
        w = ((torch.rand(N, K, device=dev, generator=g) * 2 - 1) * lim).to(dt)
        x = torch.zeros(M, N, device=dev)
        ops.linear_gate_residual_(x, a, w, None, torch.ones(1, N, device=dev), M, stream_k=False)
        ref, mag = _gemm_ref(a, w)
        r = float(((x.double() - ref).abs() / (U32 * mag).clamp_min(1e-300)).max())
        _ACC_TABLE[(dtn(dt), K)] = r
        chk.add("gemm fp32 accumulation", f"K={K}", x, ref, A * U32 * ref.abs() + B * ACC * math.sqrt(K) * U32 * mag,
                lambda i: f"row {i[0]}, column {i[1]}")
        del a, w, x, ref, mag
    chk.done()
