"""GPU: `LatteT2V` with `use_fp8` set -- QKV and fc1 of every spatial and temporal block on e4m3 tensor cores.

Bounds follow tests/test_gpu_fp8.py's docstring:
  * The e4m3 GEMM at Latte-1's CFG-pair row count (M = 2 x 16 frames x 1024 tokens = 32768, K = D = 1152, N = 3D and 4D),
    element by element against fp64 on the dequantized operands, with that file's bound: A * u16 |ref| + B * e + floor,
    e = ACC8 * mag + 2^-24 (sqrt(K) mag + 3 |v|) (GELU: times its slope 1.13, plus the tanh.approx term).
  * Whole model: max-abs against the reference goldens of every case below, fp16 and bf16 operands, in units of the
    reference's own bf16-autocast deviation on the same weights and inputs (tests/golden/t2v_ref_bf16.npz, written by
    oracle/make_golden_t2v_bf16.py), within FP8_TOL_FACTOR = 6 units as for `Latte`.  Each measured ratio is printed.
The packing is checked byte for byte against torch's CPU float8_e4m3fn cast, and the output bit for bit across calls and
against a model that never had the flag set."""
import ast
import copy
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

from fp64_bounds import A, B, SUB, TANH_U, U16, U32, Checker, report_worst  # noqa: E402
from golden_sample import as_stored  # noqa: E402

pytestmark = pytest.mark.gpu

ACC8 = 2.0 ** -13
FP8_TOL_FACTOR = 6.0
GELU_K0, GELU_K1 = 0.7978845608028654, 0.044715
FP8_STACKS = ("s_qkv", "s_fc1", "t_qkv", "t_fc1")

CASES = [
    "tiny_b2_l20",                 # D = 128: one k-block
    "tiny_b2_l20_notemporal",      # temporal blocks off
    "hd72_b2_l120_masked",         # D = 576: partial last k-block; padded prompt
    "f12_b1_l20",                  # head_dim 80, D = 320
    "f1_b2_l20",                   # text-to-image
    "f1_latte1_b2_l120",           # Latte-1: 28 layer pairs, 512^2 text-to-image, CFG-pair batch, padded prompt
    "latte1_b1_l120",              # Latte-1: 16 x 512^2
]

_WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    report_worst(_WORST)


def _case(golden_dir, tag):
    from latte_b200 import LatteT2V
    from oracle import t2v_oracle as T
    g = np.load(os.path.join(golden_dir, f"t2v_{tag}.npz"))
    kw = ast.literal_eval(str(g["cfg"]))
    cfg = T.T2VConfig(**kw)
    sd = T.make_weights(cfg, int(g["wseed"]))
    x, t, text = T.make_inputs(cfg, int(g["batch"]), int(g["text_len"]), int(g["iseed"]))
    mask = torch.from_numpy(g["mask"]) if "mask" in g else None
    net = LatteT2V(**kw)
    net.load_state_dict(sd, strict=True)
    del sd
    dev = torch.device("cuda:0")
    net = net.to(dev).eval()
    kwargs = dict(encoder_hidden_states=text.to(dev), encoder_attention_mask=mask.to(dev) if mask is not None else None,
                  enable_temporal_attentions=bool(int(g["temporal"])), return_dict=False)
    run = lambda m: m(x.to(dev), t.to(dev), **kwargs)[0]
    return g, net, run


# ------------------------------------------------------------------------------------------------ e4m3 GEMM, Latte-1 M
def _gelu64(v):
    return 0.5 * v * (1 + torch.tanh(GELU_K0 * (v + GELU_K1 * v ** 3)))


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("N,gelu", [(3456, False), (4608, True)])
def test_linear_e4m3_latte1_cfg_pair_against_fp64(dt, N, gelu):
    """Latte-1's QKV (N = 3D) and fc1 (N = 4D, bias+GELU) over a CFG pair of 16 x 512^2: M = 32768, K = 1152."""
    from latte_b200 import ops
    dev = torch.device("cuda:0")
    M, K = 32768, 1152
    chk = Checker(dt, _WORST)
    g = torch.Generator(device=dev).manual_seed(N + 11)
    a = torch.randn(M, K, device=dev, generator=g)
    a[:, ::97] *= 20                                               # outlier channels, as after modulate
    w = torch.randn(N, K, device=dev, generator=g) * 0.03
    bias = torch.randn(N, device=dev, generator=g) * 0.1
    a8, sa = ops.quantize_rows_e4m3(a)
    w8, sw = ops.quantize_rows_e4m3(w)
    del a, w
    got = ops.linear_e4m3(a8, sa, w8, sw, bias, gelu=gelu, dtype=dt)
    A64, W64 = a8.double(), w8.double()
    sc = sa.double()[:, None] * sw.double()[None, :]
    mag = (A64.abs() @ W64.abs().T) * sc
    v = (A64 @ W64.T) * sc + bias.double()[None, :]
    del A64, W64, sc
    e = ACC8 * mag + U32 * (math.sqrt(K) * mag + 3 * v.abs())
    del mag
    if gelu:
        ref = _gelu64(v)
        e = 1.13 * e + TANH_U * 0.5 * v.abs() + 4 * U32 * v.abs()
    else:
        ref = v
    bnd = A * U16[dt] * ref.abs() + B * e + SUB[dt]
    chk.add("linear_e4m3" + ("_gelu" if gelu else ""), f"M={M} N={N} K={K}", got, ref, bnd,
            lambda idx: f"row {idx[0]}, column {idx[1]}")
    chk.done()


# ------------------------------------------------------------------------------------------------ whole model
@pytest.mark.parametrize("tag", CASES)
def test_fp8_forward_matches_golden(golden_dir, tag):
    g, net, run = _case(golden_dir, tag)
    unit = float(np.load(os.path.join(golden_dir, "t2v_ref_bf16.npz"))[tag])
    ref = torch.from_numpy(g["out"])
    net.use_fp8 = True
    with torch.no_grad():
        for dt in (torch.float16, torch.bfloat16):
            net.compute_dtype = dt
            out = run(net).cpu()
            err = (as_stored(out, g, "out") - ref).abs().max().item()
            print(f"\nt2v_{tag} fp8 + {str(dt)[6:]}: max-abs {err:.3e} = {err / unit:.2f} x the reference's bf16 deviation "
                  f"{unit:.3e} (tolerance {FP8_TOL_FACTOR:g}; output absmax {ref.abs().max().item():.2f})")
            assert err < FP8_TOL_FACTOR * unit, f"t2v_{tag} fp8 + {dt}: max-abs {err:.3e} >= {FP8_TOL_FACTOR} x {unit:.3e}"


def _quantize_cpu(w):
    amax = w.abs().amax(1)
    s = torch.where(amax > 0, amax / 448.0, torch.ones_like(amax))
    return (w / s[:, None]).to(torch.float8_e4m3fn), s


def _stack_fp32(net, name):
    """The fp32 weight stack [layers * N, D] the packing quantizes for `name`."""
    blocks = net.transformer_blocks if name.startswith("s_") else net.temporal_transformer_blocks
    if name.endswith("qkv"):
        ws = [w for b in blocks for w in (b.attn1.to_q.weight, b.attn1.to_k.weight, b.attn1.to_v.weight)]
    else:
        ws = [b.ff.net[0].proj.weight for b in blocks]
    return torch.cat([w.detach().float().cpu() for w in ws])


@pytest.mark.parametrize("tag", ["tiny_b2_l20", "f12_b1_l20"])
def test_fp8_packing_holds_e4m3_stacks_only(golden_dir, tag):
    g, net, run = _case(golden_dir, tag)
    net.use_fp8 = True
    with torch.no_grad():
        run(net)
    T = net._packed[2]
    for name in FP8_STACKS:
        assert T[name + "_w16"] is None, f"{name}: FP8 packing holds a 16-bit copy"
        q_ref, s_ref = _quantize_cpu(_stack_fp32(net, name))
        assert torch.equal(T[name + "_ws"].cpu().view(torch.int32), s_ref.view(torch.int32)), f"{name}: scales differ"
        assert torch.equal(T[name + "_w8"].cpu(), q_ref.view(torch.uint8)), f"{name}: e4m3 bytes differ from torch's cast"
    for name in ("s_out_w16", "c_q_w16", "c_kv_w16", "c_out_w16", "s_fc2_w16", "t_out_w16", "t_fc2_w16", "final_w16"):
        assert T[name] is not None and T[name].dtype == torch.float16


def test_fp8_bit_exact_and_toggle_restores_the_16bit_output(golden_dir):
    g, net, run = _case(golden_dir, "hd72_b2_l120_masked")
    _, fresh, _ = _case(golden_dir, "hd72_b2_l120_masked")
    with torch.no_grad():
        want16 = run(fresh)
        net.use_fp8 = True
        o8 = [run(net) for _ in range(2)]
        twin = copy.deepcopy(net)                      # the packing is a cache: the copy repacks and gives the same output
        o8_copy = run(twin)
        net.use_fp8 = False
        o16 = [run(net) for _ in range(2)]
    assert torch.equal(o8[0], o8[1])
    assert torch.equal(o8_copy, o8[0]) and twin.use_fp8
    assert not torch.equal(o8[0], want16)
    for o in o16:
        assert torch.equal(o, want16)
    assert net.state_dict().keys() == fresh.state_dict().keys()


def test_fp8_forward_rejects_bad_e4m3_pointers(golden_dir):
    """b200_t2v_forward checks the e4m3 fields before any launch: a stack with e4m3 bytes but no scales, or with neither
    copy, is B200_ERR_SHAPE."""
    from latte_b200 import _lib
    g, net, run = _case(golden_dir, "tiny_b2_l20")
    net.use_fp8 = True
    with torch.no_grad():
        good = run(net)
    shape, w, _ = net._packed
    dev = good.device
    x = torch.zeros(2, 4, net.config.video_length, net.config.sample_size, net.config.sample_size, device=dev)
    t = torch.zeros(2, dtype=torch.int64, device=dev)
    text = torch.zeros(2, 20, net.config.caption_channels, device=dev)
    out = torch.zeros_like(good)
    lib = _lib.load()
    need = lib.b200_t2v_workspace_bytes(C.byref(shape), 2, 20)
    ws = torch.empty(need + 1024, dtype=torch.uint8, device=dev)
    base = (ws.data_ptr() + 1023) // 1024 * 1024
    for name in FP8_STACKS:
        for broken in (name + "_ws", name + "_w8"):
            bad = _lib.T2VWeights.from_buffer_copy(w)
            setattr(bad, broken, None)
            rc = lib.b200_t2v_forward(C.byref(shape), C.byref(bad), x.data_ptr(), t.data_ptr(), text.data_ptr(), None, 2, 20, 1,
                                      out.data_ptr(), base, need, torch.cuda.current_stream(dev).cuda_stream)
            assert rc == -1, f"{broken} = NULL: rc {rc}"
    torch.cuda.synchronize()
    assert not out.any(), "a rejected call launched"


# ------------------------------------------------------------------------------------------------ training raises
def _train_model():
    from latte_b200 import LatteT2V
    net = LatteT2V(num_attention_heads=2, attention_head_dim=64, num_layers=2, sample_size=16, video_length=8,
                   caption_channels=256).cuda().train()
    net.use_fp8 = True
    return net


@pytest.mark.parametrize("mode", ["plain", "checkpointing", "images"])
def test_fp8_training_raises(mode):
    net = _train_model()
    I = 2 if mode == "images" else 0
    if mode == "checkpointing":
        net.enable_gradient_checkpointing()
    x = torch.randn(2, 4, 8 + I, 16, 16, device="cuda")
    t = torch.tensor([3, 500], device="cuda")
    text = torch.randn(2, *((1 + I,) if I else ()), 20, 256, device="cuda")
    with pytest.raises(NotImplementedError, match="FP8 is a sampling path"):
        net(x, t, encoder_hidden_states=text, use_image_num=I)
    assert net._packed is None and net._train_backend is None
