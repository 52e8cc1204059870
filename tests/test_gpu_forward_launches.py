"""GPU: the sampling forwards' launch sequence, counted per kernel class by the library's event profiler
(b200_profile_enable / b200_profile_collect; while it is on the modules launch eagerly instead of replaying a CUDA graph).

The expected counts are written from the block structure, so an added or dropped launch fails here:
  * every block: attention half = LN + modulate, QKV GEMM, self-attention, gated out-projection GEMM; MLP half = LN +
    modulate, fc1 GEMM, gated fc2 GEMM.  FP8 swaps the LN and GEMM kernels of QKV and fc1 one for one.
  * Latte: depth such blocks.  Other: conditioning (timestep features, two t-MLP GEMVs, the stacked adaLN GEMV; none with
    precomputed conditioning rows), patch embedding, and the CFG combine.  The head is LN + modulate, one GEMM, a fill of
    its gate and the unpatchify when p*p*out_channels == 32 and a 16-bit weight copy exists, else one fp32 CUDA-core kernel.
  * LatteT2V: per layer a spatial block (plus the cross-attention step: a cast of the stream, the query GEMM, cross-attention
    and the output GEMM) and, with temporal attention on, a temporal block.  GEMMs before the blocks: the two caption
    projections and the K/V of every layer.  Other: conditioning (timestep features, two t-MLP GEMVs, the 6D GEMV, the
    modulation tables), a fill of the ones vector, the caption cast and patch embedding.  The head as for Latte."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu


def _launches(fn):
    """Per-class launch counts [GEMM, attention, LN, other] of everything `fn` enqueues."""
    from latte_b200 import _lib
    lib = _lib.load()
    torch.cuda.synchronize()
    _lib.profile_enable(True)
    try:
        with torch.no_grad():
            fn()
        torch.cuda.synchronize()
    finally:
        ms, n = (C.c_double * 4)(), (C.c_int * 4)()
        rc = lib.b200_profile_collect(ms, n, 4)
        _lib.profile_enable(False)
    _lib.check(rc, "b200_profile_collect")
    return list(n)


def latte_launches(depth, cfg, tensor_head, precomputed):
    return [4 * depth + tensor_head,
            depth,
            2 * depth + tensor_head,
            (0 if precomputed else 4) + 1 + (2 if tensor_head else 1) + cfg]


def t2v_launches(layers, temporal):
    return [3 + layers * (6 + 4 * temporal) + 1,
            layers * (2 + temporal),
            layers * (2 + 2 * temporal) + 1,
            6 + 1 + 1 + layers + 2]


LATTE_CASES = {
    "fp16": dict(),
    "bf16": dict(dtype=torch.bfloat16),
    "cfg": dict(cfg=True),
    "cfg_bf16": dict(cfg=True, dtype=torch.bfloat16),
    "precomputed": dict(precomputed=True),
    "precomputed_cfg": dict(cfg=True, precomputed=True),
    "fp8": dict(fp8=True),
    "fp8_cfg": dict(cfg=True, fp8=True),
    "fp32_head": dict(learn_sigma=False),
    "fp32_head_cfg": dict(cfg=True, learn_sigma=False),
    "depth28_cfg": dict(cfg=True, depth=28),
}


@pytest.mark.parametrize("case", list(LATTE_CASES))
def test_latte_launch_counts(case):
    from latte_b200 import Latte
    kw = dict(cfg=False, precomputed=False, fp8=False, learn_sigma=True, depth=4, dtype=torch.float16)
    kw.update(LATTE_CASES[case])
    dev = torch.device("cuda:0")
    net = Latte(input_size=16, hidden_size=128, depth=kw["depth"], num_heads=2, num_frames=8, num_classes=10,
                learn_sigma=kw["learn_sigma"], extras=2).to(dev).eval()
    net.compute_dtype = kw["dtype"]
    net.use_fp8 = kw["fp8"]
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 8, 4, 16, 16, generator=g).to(dev)
    t = torch.tensor([3, 500], device=dev)
    y = torch.tensor([1, 10], device=dev)
    step = None
    if kw["precomputed"]:
        with torch.no_grad():
            net.precompute_conditioning(t.view(1, 2), y)
        step = 0
    run = (lambda: net.forward_with_cfg(x, t, y=y, cfg_scale=4.0, trajectory_step=step)) if kw["cfg"] else \
        (lambda: net(x, t, y=y, trajectory_step=step))
    tensor_head = kw["learn_sigma"]          # p*p*out_channels = 32 with learned sigma, 16 without
    want = latte_launches(kw["depth"], kw["cfg"], tensor_head, kw["precomputed"])
    assert _launches(run) == want, f"{case}: [GEMM, attention, LN, other]"
    if case == "depth28_cfg":
        assert sum(want) == 206                  # Latte-XL/2's forward_with_cfg


T2V_CASES = {
    "temporal": dict(),
    "no_temporal": dict(temporal=False),
    "video_length_1": dict(video_length=1, sample_size=32),
    "fp8": dict(fp8=True),
    "fp8_no_temporal": dict(fp8=True, temporal=False),
    "bf16": dict(dtype=torch.bfloat16),
}


@pytest.mark.parametrize("case", list(T2V_CASES))
def test_t2v_launch_counts(case):
    from latte_b200 import LatteT2V
    kw = dict(temporal=True, fp8=False, video_length=8, sample_size=16, dtype=torch.float16)
    kw.update(T2V_CASES[case])
    dev = torch.device("cuda:0")
    layers, F, S = 3, kw["video_length"], kw["sample_size"]
    net = LatteT2V(num_attention_heads=2, attention_head_dim=64, num_layers=layers, sample_size=S, video_length=F,
                   caption_channels=256).to(dev).eval()
    net.compute_dtype = kw["dtype"]
    net.use_fp8 = kw["fp8"]
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 4, F, S, S, generator=g).to(dev)
    text = torch.randn(2, 20, 256, generator=g).to(dev)
    t = torch.tensor([3, 500], device=dev)
    mask = torch.ones(2, 20, device=dev)
    mask[1, 12:] = 0
    run = lambda: net(x, t, encoder_hidden_states=text, encoder_attention_mask=mask,
                      enable_temporal_attentions=kw["temporal"], return_dict=False)
    assert _launches(run) == t2v_launches(layers, kw["temporal"]), f"{case}: [GEMM, attention, LN, other]"
