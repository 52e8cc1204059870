"""GPU: temporal attention and LatteT2V at any video length in [1, 128], including text-to-image (video_length = 1).

A temporal attention tile holds G = floor(128 / F) tokens x F frames; when F is not a power of two the tile is not full
(G * F < 128) and when G does not divide N the last group of tokens is partial.  The op is checked against an fp32 torch
restatement on both, LatteT2V against goldens of the unmodified reference at F = 1, 3 and 12
(oracle/make_golden_t2v_frames.py), and the class-conditional Latte, which runs the same kernel, against its oracle."""
import ast
import json
import os
from types import SimpleNamespace

import pytest
import torch
from golden_sample import as_stored  # noqa: E402

pytestmark = pytest.mark.gpu

TOL = {torch.float16: 4e-3, torch.bfloat16: 3e-2}


def _close(got, ref, tol):
    got, ref = got.float(), ref.float()
    assert torch.isfinite(got).all()
    err = (got - ref).abs()
    bad = err > tol + tol * ref.abs()
    assert not bad.any(), f"max err {err.max().item():.3e}, {bad.float().mean().item() * 100:.3f}% outside tol {tol}"


def _temporal_ref(qkv, batch, frames, tokens, heads):
    """softmax(q k^T / sqrt(hd)) v over the F frames of each (sample, token, head), fp32; rows (b, f, n) as the op."""
    D = qkv.shape[1] // 3
    hd = D // heads
    x = qkv.float().reshape(batch, frames, tokens, 3, heads, hd).permute(3, 0, 2, 4, 1, 5)   # (3, B, N, H, F, hd)
    q, k, v = x[0], x[1], x[2]
    o = torch.softmax(q @ k.transpose(-1, -2) * hd ** -0.5, dim=-1) @ v
    return o.permute(0, 3, 1, 2, 4).reshape(batch * frames * tokens, D)


# (F, N): G = floor(128 / F) and whether the last token group is partial
CASES = [
    (1, 200),     # G = 128, 200 = 128 + 72
    (2, 100),     # G = 64, partial
    (3, 256),     # G = 42, 256 = 6 * 42 + 4
    (5, 77),      # G = 25, partial
    (12, 256),    # G = 10, 256 = 25 * 10 + 6
    (16, 40),     # G = 8, whole groups (the power-of-two tile of the benchmarks)
    (24, 64),     # G = 5, partial
    (48, 20),     # G = 2, whole groups, 96 of 128 rows used
    (100, 9),     # G = 1, 100 rows
    (128, 6),     # G = 1, full tile
]


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("hd", [64, 72, 80])
@pytest.mark.parametrize("case", CASES, ids=[f"F{f}_N{n}" for f, n in CASES])
def test_temporal_attention_any_length(case, hd, dt):
    from latte_b200 import ops
    F, N = case
    b, h = 2, 2
    g = torch.Generator().manual_seed(F * 1000 + N + hd)
    qkv = (torch.randn(b * F * N, 3 * h * hd, generator=g) * 1.5).cuda().to(dt)
    _close(ops.attention(qkv, b, F, N, h, True), _temporal_ref(qkv, b, F, N, h), TOL[dt])


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("hd", [64, 72, 80])
def test_one_frame_is_v(hd, dt):
    """At F = 1 the softmax is over one key and is exactly 1: the output is the V columns of qkv, bit for bit."""
    from latte_b200 import ops
    b, N, h = 2, 300, 3
    g = torch.Generator().manual_seed(hd)
    qkv = (torch.randn(b * N, 3 * h * hd, generator=g) * 4).cuda().to(dt)
    out = ops.attention(qkv, b, 1, N, h, True)
    assert torch.equal(out, qkv[:, 2 * h * hd:])


@pytest.mark.parametrize("hd", [64, 80])
@pytest.mark.parametrize("F", [3, 5, 12, 24, 100])
def test_unloaded_tile_rows_do_not_leak(F, hd):
    """Constant q and k make every frame equally weighted, so the output is the mean of V over the frames.  The tile rows
    [G*F, 128) that no load fills must not contribute: a spatial attention over an all-NaN qkv runs first, so that stale
    shared memory of the same kernel is likely to hold NaN bits (a check of the zeroing only when that memory is
    non-finite; it does not replace reading it)."""
    from latte_b200 import ops
    b, N, h = 2, 64, 2
    D = h * hd
    nan_qkv = torch.full((80 * 256, 3 * D), float("nan"), dtype=torch.float16, device="cuda")
    ops.attention(nan_qkv, 80, 1, 256, h, False)          # 320 CTAs: every SM runs at least one
    qkv = torch.empty(b, F, N, 3, D)
    qkv[:, :, :, 0] = 0.25
    qkv[:, :, :, 1] = 0.5
    frame_v = 1024.0 * (torch.arange(F) % 8 + 1)                   # exactly representable, and so is every partial sum
    qkv[:, :, :, 2] = frame_v.view(1, F, 1, 1)
    qkv = qkv.reshape(b * F * N, 3 * D).cuda().half()
    out = ops.attention(qkv, b, F, N, h, True)
    assert torch.isfinite(out).all()
    want = torch.full_like(out, frame_v.double().mean().item(), dtype=torch.float32)
    _close(out, want, 1e-3)


def _golden_case(golden_dir, tag):
    import numpy as np
    from oracle import t2v_oracle as T
    g = np.load(os.path.join(golden_dir, f"t2v_{tag}.npz"))
    kw = ast.literal_eval(str(g["cfg"]))
    cfg = T.T2VConfig(**kw)
    sd = T.make_weights(cfg, int(g["wseed"]))
    x, t, text = T.make_inputs(cfg, int(g["batch"]), int(g["text_len"]), int(g["iseed"]))
    mask = torch.from_numpy(g["mask"]) if "mask" in g else None
    return g, kw, sd, x, t, text, mask


def _run_golden(golden_dir, tag):
    from latte_b200 import LatteT2V
    g, kw, sd, x, t, text, mask = _golden_case(golden_dir, tag)
    net = LatteT2V(**kw)
    net.load_state_dict(sd, strict=True)
    del sd
    net = net.cuda().eval()
    with torch.no_grad():
        out = net(x.cuda(), t.cuda(), encoder_hidden_states=text.cuda(),
                  encoder_attention_mask=mask.cuda() if mask is not None else None,
                  enable_temporal_attentions=bool(int(g["temporal"])), return_dict=False)[0]
    ref = torch.from_numpy(g["out"])
    err = (as_stored(out.cpu(), g, "out") - ref).abs()
    assert err.max().item() < 1e-2, f"{tag}: max-abs {err.max():.3e} vs the reference module (output magnitude {ref.abs().max():.2f})"
    return err


@pytest.mark.parametrize("tag", ["f1_b2_l20", "f1_b2_l20_notemporal", "f1_b2_l20_masked", "f12_b1_l20", "f3_b2_l20"])
def test_t2v_matches_reference_golden(golden_dir, tag):
    _run_golden(golden_dir, tag)


def test_t2v_latte1_t2i_matches_reference_golden(golden_dir):
    """The Latte-1 text-to-image call: 28 layer pairs, D = 1152, 1 x 512 x 512 (1024 tokens), 120 prompt tokens, a CFG pair
    with the first prompt masked to 12 tokens."""
    if not os.path.exists(os.path.join(golden_dir, "t2v_f1_latte1_b2_l120.npz")):
        pytest.skip("t2v_f1_latte1_b2_l120.npz not generated (oracle/make_golden_t2v_frames.py --full)")
    err = _run_golden(golden_dir, "f1_latte1_b2_l120")
    assert err.mean().item() < 1e-3, f"mean-abs {err.mean():.3e}"


T2I_TINY = dict(num_attention_heads=8, attention_head_dim=72, num_layers=2, sample_size=32, video_length=1, caption_channels=256)


def test_t2i_through_get_models(tmp_path):
    """The reference's sample_t2x.py path: get_models(model="LatteT2V", video_length=1) -> from_pretrained of a
    `transformer/` directory (config.json + weights), then forward on a CFG pair with a padded prompt."""
    from latte_b200.models import get_models
    from oracle import t2v_oracle as T
    cfg = T.T2VConfig(**T2I_TINY)
    sd = T.make_weights(cfg, 21)
    root = tmp_path / "Latte-1"
    (root / "transformer").mkdir(parents=True)
    conf = {k: v for k, v in T2I_TINY.items() if k != "video_length"}
    conf.update(_class_name="LatteT2V", in_channels=4, out_channels=8, patch_size=2, norm_type="ada_norm_single",
                activation_fn="gelu-approximate", attention_bias=True, video_length=16)
    (root / "transformer" / "config.json").write_text(json.dumps(conf))
    torch.save(sd, root / "transformer" / "diffusion_pytorch_model.bin")
    net = get_models(SimpleNamespace(model="LatteT2V", pretrained_model_path=str(root), video_length=1))
    assert net.config.video_length == 1
    net = net.cuda().eval()
    x, t, text = T.make_inputs(cfg, 1, 40, 22)
    x, t, text = x.repeat(2, 1, 1, 1, 1), t.repeat(2), torch.cat([torch.zeros_like(text), text])   # (negative, positive)
    mask = torch.ones(2, 40, dtype=torch.int64)
    mask[0, 3:] = 0
    assert x.shape == (2, 4, 1, 32, 32)
    with torch.no_grad():
        out = net(x.cuda(), t.cuda(), encoder_hidden_states=text.cuda(), encoder_attention_mask=mask.cuda(),
                  enable_temporal_attentions=True, return_dict=False)[0]
    ref = T.t2v_forward(sd, cfg, x, t, text, enable_temporal=True, text_mask=mask)
    assert out.shape == ref.shape == (2, 8, 1, 32, 32)
    err = (out.cpu() - ref).abs().max().item()
    assert err < 1e-2, f"max-abs {err:.3e} (output magnitude {ref.abs().max():.2f})"


def test_t2i_too_few_tokens_is_rejected():
    """64 tokens per sample (sample_size 16, one frame) is not a multiple of 128: a clear error, not a launch."""
    from latte_b200 import LatteT2V
    kw = dict(T2I_TINY, sample_size=16)
    net = LatteT2V(**kw).cuda().eval()
    with pytest.raises(RuntimeError, match="multiple of 128"):
        net(torch.randn(1, 4, 1, 16, 16, device="cuda"), torch.tensor([3], device="cuda"),
            encoder_hidden_states=torch.randn(1, 8, 256, device="cuda"))


def test_latte_twelve_frames_matches_oracle():
    """The class-conditional Latte runs the same temporal kernel: num_frames = 12 (G = 10, 64 tokens = 6 * 10 + 4)."""
    from latte_b200 import Latte
    from oracle import latte_oracle as O
    cfg = O.make_config("Latte-tiny72/2", input_size=16, num_frames=12)
    sd = O.make_weights(cfg, 31)
    x, t, y = O.make_inputs(cfg, 2, 32)
    net = Latte(input_size=cfg.input_size, hidden_size=cfg.hidden_size, depth=cfg.depth, num_heads=cfg.num_heads,
                num_frames=cfg.num_frames, num_classes=cfg.num_classes, learn_sigma=True, extras=2)
    net.load_state_dict(sd, strict=True)
    net = net.cuda().eval()
    with torch.no_grad():
        out = net(x.cuda(), t.cuda(), y=y.cuda())
    ref = O.latte_forward(sd, cfg, x, t, y)
    assert out.shape == ref.shape
    err = (out.cpu() - ref).abs().max().item()
    assert err < 2e-2, f"max-abs {err:.3e} (output magnitude {ref.abs().max():.2f})"
