"""GPU: the FP8 (e4m3) sampling path -- weight quantization, the e4m3 LayerNorm + modulate, the e4m3 GEMM, and `Latte` with
`use_fp8` set.

Quantization formula (both operands, row by row): s = amax(|row|) / 448 (1 for an all-zero row), q = e4m3_rn_satfinite(row / s)
with the division correctly rounded in fp32 -- so torch's CPU `float8_e4m3fn` cast of `row / s` reproduces the weight bytes.

Bounds, element by element against fp64 (tests/fp64_bounds.py conventions):
  * ln_modulate_e4m3, dequantized (q * s): the 16-bit test's LayerNorm bound on y, plus half an e4m3 ulp of y (2^-4 |y| for
    normal values, 2^-10 s below 2^-6 s: half the subnormal spacing) -- the division's own rounding is far below both.
  * GEMM: the reference is fp64 on the DEQUANTIZED operands, a_scale[row] * w_scale[col] * (A8 . W8^T) + bias.  The
    output rounding A * u16 |ref|, the epilogue's three fp32 roundings, and the accumulation: the kernel adds each 128-wide
    k-block's partial sum into an fp32 total, but inside a k-block the e4m3 wgmma accumulates with fewer bits than fp32.
    With mag = sum_k |a_k w_k| (scaled), the bound allows ACC8 * mag for the in-k-block sums (ACC8 = 2^-13: the
    accumulator width the DeepSeek-V3 report gives for Hopper FP8, ~14 bits, with one bit of slack) plus the fp32 term
    sqrt(K) 2^-24 mag of the total.  GELU adds its slope (<= 1.13) times that and the tanh.approx error.
    The test also prints the measured accumulation error in units of fp32 accumulation (2^-24 sqrt(K) mag) at K = 1152.
  * Whole model: max-abs against the fp32 goldens, in units of the reference's own bf16-autocast deviation on the same
    weights and inputs (ref_bf16_maxabs, stored in each golden), so one factor serves models whose outputs differ in
    size.  Measured on an H100 (fp16 / bf16 for the 16-bit operands): tiny64 1.9 / 1.9, tiny72 2.3 / 2.1, S/2 4.0 / 3.8,
    XL/2 4.1 / 3.7 of those units.  The tolerance is FP8_TOL_FACTOR = 6 units: the worst measured value plus ~45 %
    for rounding that differs between GPUs (the residual GEMMs' stream-K splits follow the SM count).  The element-wise
    fp64 tests above carry the kernels' correctness; this one catches errors in how the model uses them."""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest
import torch

from fp64_bounds import A, B, SUB, TANH_U, U16, U32, Checker, report_worst  # noqa: E402
from golden_sample import as_stored  # noqa: E402

pytestmark = pytest.mark.gpu

E4M3_HALF_ULP = 2.0 ** -4
E4M3_SUB_HALF = 2.0 ** -10      # half the e4m3 subnormal spacing 2^-9, in units of the row scale
ACC8 = 2.0 ** -13
FP8_TOL_FACTOR = 6.0
GELU_K0, GELU_K1 = 0.7978845608028654, 0.044715

_WORST = {}
_ACC = {}


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if _ACC:
        print("\ne4m3 GEMM accumulation: worst error beyond the 16-bit output rounding, in units of 2^-24 sqrt(K) mag:")
        for k, r in sorted(_ACC.items()):
            print(f"  {k}: {r:.3g}")
    report_worst(_WORST)


def _rc(idx):
    return f"row {idx[0]}, column {idx[1]}"


def _quantize_cpu(w):
    amax = w.abs().amax(1)
    s = torch.where(amax > 0, amax / 448.0, torch.ones_like(amax))
    return (w / s[:, None]).to(torch.float8_e4m3fn), s


# ------------------------------------------------------------------------------------------------ weight quantization
@pytest.mark.parametrize("rows,cols", [(3456, 1152), (4608, 1152), (37, 576), (5, 16), (64, 4608)])
def test_quantize_rows_matches_torch_cast(dev, rows, cols):
    from latte_b200 import ops
    g = torch.Generator().manual_seed(rows + cols)
    w = torch.randn(rows, cols, generator=g) * 0.03
    w[0] = 0.0                                                     # an all-zero row: scale 1, bytes 0
    w[1] *= 1e-6                                                   # values deep in the e4m3 subnormal range of their row
    w[2, 3] = 7.5                                                  # one outlier: the rest of its row goes subnormal
    w[3] = torch.linspace(-1, 1, cols)                             # exact ties between e4m3 values
    q, s = ops.quantize_rows_e4m3(w.to(dev))
    q_ref, s_ref = _quantize_cpu(w)
    assert torch.equal(s.cpu().view(torch.int32), s_ref.view(torch.int32)), "scales differ"
    assert s.cpu()[0].item() == 1.0
    assert torch.equal(q.cpu().view(torch.uint8), q_ref.view(torch.uint8)), "e4m3 bytes differ from torch's cast"


# ------------------------------------------------------------------------------------------------ LayerNorm + modulate
@pytest.mark.parametrize("D", [384, 576, 1152, 1536])
def test_ln_modulate_e4m3(dev, D):
    from latte_b200 import ops
    chk = Checker(torch.float16, _WORST)
    g = torch.Generator(device=dev).manual_seed(D + 7)
    for Bb, rpb, short in [(3, 37, 5), (3, 4095, 1000)]:
        T = Bb * rpb - short
        x = torch.randn(T, D, device=dev, generator=g) * 3 + 1
        x[::3] = 8 + 0.05 * torch.randn(x[::3].shape, device=dev, generator=g)
        mod = torch.randn(Bb, 6 * D, device=dev, generator=g) * 0.5
        shift, scale = mod[:, 3 * D:4 * D], mod[:, 4 * D:5 * D]
        q, s = ops.ln_modulate_e4m3(x, shift, scale, rpb)
        bidx = torch.arange(T, device=dev) // rpb
        x64 = x.double()
        mean = x64.mean(1, keepdim=True)
        rstd = (((x64 - mean) ** 2).mean(1, keepdim=True) + 1e-6).rsqrt()
        xh = (x64 - mean) * rstd
        ref = xh * (1 + scale.double()[bidx]) + shift.double()[bidx]
        c1 = (1 + scale.double()[bidx]).abs()
        e_xh = U32 * (math.sqrt(D) * (rstd * x64.abs().mean(1, keepdim=True) + xh.abs()) + 3 * xh.abs())
        e_y = B * (c1 * e_xh + U32 * (2 * xh.abs() * c1 + shift.double()[bidx].abs()))
        s64 = s.double()[:, None]
        got = q.double() * s64
        bnd = E4M3_HALF_ULP * (1 + 2 * U32) * (ref.abs() + e_y) + E4M3_SUB_HALF * s64 + e_y + 2 * U32 * got.abs()
        chk.add("ln_modulate_e4m3", f"B={Bb} rpb={rpb}", got, ref, bnd, _rc)
        # the scale is the row's amax / 448: every row reaches +-448 exactly, and s matches the fp64 amax
        assert torch.equal(q.float().abs().amax(1), torch.full((T,), 448.0, device=dev))
        amax = ref.abs().amax(1)
        assert ((s.double() * 448 - amax).abs() <= e_y.amax(1) + 4 * U32 * amax).all()
    chk.done()


# ------------------------------------------------------------------------------------------------ e4m3 GEMM
def _gelu64(v):
    return 0.5 * v * (1 + torch.tanh(GELU_K0 * (v + GELU_K1 * v ** 3)))


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("M,N,K,gelu", [(8192, 3456, 1152, False), (8192, 4608, 1152, True), (1000, 1728, 576, False),
                                        (1000, 2304, 576, True), (300, 96, 80, False)])
def test_linear_e4m3_against_fp64(dev, dt, M, N, K, gelu):
    """XL/2 QKV and fc1 (T = 16 frames x 256 tokens x CFG pair), tiny72's (K = 576: the last k-block is half past K), and a
    narrow one (N = 96, K = 80) whose single tile and k-block are both partial.  The kernel has one tile width (128)."""
    from latte_b200 import ops
    chk = Checker(dt, _WORST)
    g = torch.Generator(device=dev).manual_seed(M + N + K)
    a = torch.randn(M, K, device=dev, generator=g)
    a[:, :: 97] *= 20                                              # outlier channels, as after modulate
    w = torch.randn(N, K, device=dev, generator=g) * 0.03
    bias = torch.randn(N, device=dev, generator=g) * 0.1
    a8, sa = ops.quantize_rows_e4m3(a)
    w8, sw = ops.quantize_rows_e4m3(w)
    for use_bias in (True, False):
        bb = bias if use_bias else None
        got = ops.linear_e4m3(a8, sa, w8, sw, bb, gelu=gelu, dtype=dt)
        A64, W64 = a8.double(), w8.double()
        sc = sa.double()[:, None] * sw.double()[None, :]
        acc = A64 @ W64.T
        mag = (A64.abs() @ W64.abs().T) * sc
        v = acc * sc + (bb.double()[None, :] if use_bias else 0.0)
        e_v = ACC8 * mag + U32 * (math.sqrt(K) * mag + 3 * v.abs())
        if gelu:
            ref = _gelu64(v)
            e = 1.13 * e_v + TANH_U * 0.5 * v.abs() + 4 * U32 * v.abs()
        else:
            ref = v
            e = e_v
            if not use_bias:
                # the measurement: error beyond the output rounding (half a 16-bit ulp), in fp32-accumulation units
                excess = ((got.double() - ref).abs() - U16[dt] * ref.abs()).clamp_min(0)
                r = (excess / (U32 * math.sqrt(K) * mag).clamp_min(1e-300)).amax().item()
                _ACC[f"{str(dt)[6:]} M={M} N={N} K={K}"] = r
        bnd = A * U16[dt] * ref.abs() + B * e + SUB[dt]
        chk.add("linear_e4m3" + ("_gelu" if gelu else ""), f"M={M} N={N} K={K} bias={use_bias}", got, ref, bnd, _rc)
        # a dropped per-channel weight scale on the last tile is rejected
        wrong = got.double().clone()
        wrong[:, -32:] = (acc * sa.double()[:, None])[:, -32:]
        m = Checker(dt)
        m.add("wrong", "w_scale dropped", wrong, ref, bnd, _rc)
        assert m.bad
    chk.done()


# ------------------------------------------------------------------------------------------------ whole model
def _build(golden_dir, fname):
    from latte_b200 import Latte
    from oracle import latte_oracle as O
    g = np.load(os.path.join(golden_dir, fname))
    m = re.match(r"(\S+) batch=(\d+) wseed=(\d+) iseed=(\d+) extras=(\d+) frames=(\d+) input=(\d+)", str(g["meta"]))
    name, batch, wseed, iseed, extras, frames, inp = m.group(1), *map(int, m.groups()[1:])
    cfg = O.make_config(name, extras=extras, num_frames=frames, input_size=inp)
    sd = O.make_weights(cfg, wseed)
    x, t, y = O.make_inputs(cfg, batch, iseed)
    net = Latte(input_size=cfg.input_size, hidden_size=cfg.hidden_size, depth=cfg.depth, num_heads=cfg.num_heads,
                num_frames=cfg.num_frames, num_classes=cfg.num_classes, learn_sigma=True, extras=cfg.extras)
    net.load_state_dict(sd, strict=True)
    dev = torch.device("cuda:0")
    return g, net.to(dev).eval(), (x.to(dev), t.to(dev), y.to(dev) if extras == 2 else None)


@pytest.mark.parametrize("fname", ["latte_tiny64_2_b2.npz", "latte_tiny72_2_b2.npz", "latte_s_2_b2.npz", "latte_xl_2_b2.npz"])
def test_fp8_forward_matches_golden(golden_dir, fname):
    g, net, (x, t, y) = _build(golden_dir, fname)
    ref = torch.from_numpy(g["out"])
    tol = FP8_TOL_FACTOR * float(g["ref_bf16_maxabs"])
    net.use_fp8 = True
    with torch.no_grad():
        for dt in (torch.float16, torch.bfloat16):
            net.compute_dtype = dt
            out = net(x, t, y=y).cpu()
            err = (as_stored(out, g, "out") - ref).abs().max().item()
            print(f"\n{fname} fp8 + {dt}: max-abs {err:.3e} (tolerance {tol:.3e}, output absmax {ref.abs().max().item():.2f})")
            assert err < tol, f"{fname} fp8 + {dt}: max-abs {err:.3e} >= {tol:.3e}"


def test_fp8_eager_graph_and_trajectory_are_bit_identical(golden_dir):
    g, net, (x, t, y) = _build(golden_dir, "latte_tiny72_2_b2.npz")
    net.use_fp8 = True
    with torch.no_grad():
        net.use_cuda_graphs = False
        eager = net.forward_with_cfg(x, t, y=y, cfg_scale=4.0)
        net.use_cuda_graphs = True
        outs = [net.forward_with_cfg(x, t, y=y, cfg_scale=4.0) for _ in range(3)]      # eager, capture, replay
        assert net._graphs and all(st["graph"] is not None for st in net._graphs.values())
        net.precompute_conditioning(t.view(1, -1), y)
        traj = net.forward_with_cfg(x, t, y=y, cfg_scale=4.0, trajectory_step=0)
        net.clear_conditioning()
    for o in outs + [traj]:
        assert torch.equal(o, eager)


def test_fp8_toggle_restores_the_16bit_output(golden_dir):
    g, net, (x, t, y) = _build(golden_dir, "latte_tiny64_2_b2.npz")
    _, fresh, _ = _build(golden_dir, "latte_tiny64_2_b2.npz")
    with torch.no_grad():
        net.use_fp8 = True
        o8 = net(x, t, y=y)
        net.use_fp8 = False
        o16 = [net(x, t, y=y) for _ in range(3)]
        want = fresh(x, t, y=y)
    assert not torch.equal(o8, want)
    for o in o16:
        assert torch.equal(o, want)


def test_fp8_forward_rejects_bad_e4m3_pointers(golden_dir):
    """b200_latte_forward checks the e4m3 fields of the QKV and fc1 stacks before any launch: a stack with e4m3 bytes but
    no scales, or with neither copy, is B200_ERR_SHAPE (the check b200_t2v_forward runs on each of its four stacks)."""
    from latte_b200 import _lib
    g, net, (x, t, y) = _build(golden_dir, "latte_tiny64_2_b2.npz")
    net.use_fp8 = True
    with torch.no_grad():
        good = net(x, t, y=y)
    shape, w, _, _ = net._packed
    dev = good.device
    out = torch.zeros_like(good)
    lib = _lib.load()
    B = x.shape[0]
    need = lib.b200_latte_workspace_bytes(C.byref(shape), B)
    ws = torch.empty(need + 1024, dtype=torch.uint8, device=dev)
    base = (ws.data_ptr() + 1023) // 1024 * 1024
    xf = x.float().contiguous()
    for name in ("qkv", "fc1"):
        for broken in (name + "_ws", name + "_w8"):
            bad = _lib.LatteWeights.from_buffer_copy(w)
            setattr(bad, broken, None)
            rc = lib.b200_latte_forward(C.byref(shape), C.byref(bad), xf.data_ptr(), t.data_ptr(),
                                        y.data_ptr(), B, 0, 0.0, out.data_ptr(), base, need,
                                        torch.cuda.current_stream(dev).cuda_stream)
            assert rc == -1, f"{broken} = NULL: rc {rc}"
    torch.cuda.synchronize()
    assert not out.any(), "a rejected call launched"


def test_fp8_training_raises(golden_dir):
    g, net, (x, t, y) = _build(golden_dir, "latte_tiny64_2_b2.npz")
    net.train()
    net.use_fp8 = True
    with pytest.raises(NotImplementedError, match="FP8 is a sampling path"):
        net(x, t, y=y)


def test_fp8_toggle_inside_a_trajectory(golden_dir):
    """Between precompute_conditioning and clear_conditioning the packing is frozen; toggling use_fp8 there repacks in the
    new mode (no 16-bit QKV / fc1 copies in FP8 mode), and every call gives what a model in that mode gives eagerly."""
    g, net, (x, t, y) = _build(golden_dir, "latte_tiny72_2_b2.npz")
    _, ref8, _ = _build(golden_dir, "latte_tiny72_2_b2.npz")
    _, ref16, _ = _build(golden_dir, "latte_tiny72_2_b2.npz")
    ref8.use_fp8 = True
    ref8.use_cuda_graphs = ref16.use_cuda_graphs = False
    call = lambda m, **kw: m.forward_with_cfg(x, t, y=y, cfg_scale=4.0, **kw)
    with torch.no_grad():
        want8, want16 = call(ref8), call(ref16)
        net.precompute_conditioning(t.view(1, -1), y)
        a16 = [call(net, trajectory_step=0) for _ in range(3)]           # eager, capture, replay
        net.use_fp8 = True
        a8 = [call(net, trajectory_step=0) for _ in range(3)]
        T = net._frozen[2]
        assert T["qkv_w8"] is not None and T["qkv_w16"] is None and T["fc1_w16"] is None
        net.use_fp8 = False
        b16 = [call(net, trajectory_step=0) for _ in range(3)]
        net.clear_conditioning()
    assert not torch.equal(want8, want16)
    for o in a8:
        assert torch.equal(o, want8)
    for o in a16 + b16:
        assert torch.equal(o, want16)


def test_fp8_latte_img_with_images_raises():
    """LatteIMG's frames-with-images forward (training and eval) runs the 16-bit training engine: with use_fp8 set it
    raises instead of ignoring the flag; its video-only training forward raises through Latte's."""
    from latte_b200 import LatteIMG
    dev = torch.device("cuda:0")
    F, I, B = 4, 2, 2
    net = LatteIMG(input_size=16, hidden_size=128, depth=2, num_heads=2, num_frames=F, num_classes=5, extras=2).to(dev)
    net.use_fp8 = True
    x = torch.randn(B, F + I, 4, 16, 16, device=dev)
    t = torch.tensor([3, 500], device=dev)
    y = torch.tensor([1, 2], device=dev)
    yi = torch.tensor([[0, 1], [2, 3]], device=dev)
    net.train()
    with pytest.raises(NotImplementedError, match="use_image_num > 0"):
        net(x, t, y=y, y_image=yi, use_image_num=I)
    with pytest.raises(NotImplementedError, match="FP8 is a sampling path"):
        net(x[:, :F].contiguous(), t, y=y)
    net.eval()
    with torch.no_grad(), pytest.raises(NotImplementedError, match="use_image_num > 0"):
        net(x, t, y=y, y_image=yi, use_image_num=I)
