"""GPU: LatteT2V video + image joint training (`use_image_num` > 0) on the native path -- the step against the UNMODIFIED
reference's gradients (tests/golden/train_t2v_img_*.npz; tests/test_gpu_train_t2v.py's bars: every gradient norm within 1 % in
fp16, 8 % in bf16, plus the stored full gradients and the output), the checkpointed step against the plain one, the Latte-1
layer geometry against the fp32 torch restatement, a full Latte-1 optimizer step and the refusals."""
import os

import numpy as np
import pytest
import torch

from oracle import t2v_img_oracle as TI
from oracle import t2v_oracle as T
from oracle.train_t2v_ops_oracle import T2VTorchOps

pytestmark = pytest.mark.gpu

DTS = [torch.float16, torch.bfloat16]
NORM_TOL = {torch.float16: 1e-2, torch.bfloat16: 8e-2}
FULL_TOL = {torch.float16: 2e-2, torch.bfloat16: 1e-1}
TAGS = ["tiny_f4_i3_b2_l20", "tiny_f4_i3_b2_l20_masked", "hd72_f8_i2_b1_l120_masked", "f1_i2_b2_l20"]


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


def _module(cfg, sd, dev):
    from latte_b200 import LatteT2V
    m = LatteT2V(num_attention_heads=cfg.num_attention_heads, attention_head_dim=cfg.attention_head_dim,
                 in_channels=cfg.in_channels, out_channels=cfg.out_channels, num_layers=cfg.num_layers, patch_size=cfg.patch_size,
                 sample_size=cfg.sample_size, caption_channels=cfg.caption_channels, video_length=cfg.video_length)
    m.load_state_dict(sd, strict=True)
    return m.to(dev).train()


def _sample(z, key, a):
    if key + "_sample" in z:
        axis, step = (int(v) for v in z[key + "_sample"])
        sl = [slice(None)] * a.ndim
        sl[axis] = slice(None, None, step)
        a = a[tuple(sl)]
    return a


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


# ---------------------------------------------------------------------------------------------------------- the goldens
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("tag", TAGS)
def test_native_step_matches_reference_gradients(dev, golden_dir, dt, tag):
    z = np.load(os.path.join(golden_dir, f"train_t2v_img_{tag}.npz"))
    cfg = T.T2VConfig(**eval(str(z["cfg"])))
    I = int(z["images"])
    x, t, text = TI.make_img_inputs(cfg, int(z["batch"]), I, int(z["text_len"]), int(z["iseed"]))
    m = _module(cfg, T.make_weights(cfg, int(z["wseed"])), dev)
    m.train_dtype = dt
    mask = torch.from_numpy(z["mask"]).to(dev) if "mask" in z else None
    out = m(x.to(dev), t.to(dev), encoder_hidden_states=text.to(dev), encoder_attention_mask=mask, use_image_num=I).sample
    assert out.grad_fn is not None and out.shape == (x.shape[0], cfg.out_channels, cfg.video_length + I) + x.shape[3:]
    gco = torch.randn(out.shape, generator=torch.Generator().manual_seed(int(z["gseed"]))).to(dev)
    (out * gco).sum().backward()
    names = [str(n) for n in z["grad_names"]]
    named = dict(m.named_parameters())
    assert all(named[n].grad is not None and torch.isfinite(named[n].grad).all() for n in names)
    want = z["grad_norms"]
    got = np.array([named[n].grad.double().norm().item() for n in names])
    # exactly-zero gradients (key biases; q / k of a one-frame temporal attention) are rounding noise: an absolute bound
    one = cfg.video_length == 1
    zero = np.array([n.endswith("to_k.bias") or (one and n.startswith("temporal_") and (".to_q." in n or ".to_k." in n))
                     for n in names])
    assert np.all(got[zero] < NORM_TOL[dt] * np.median(want))
    err = np.abs(got - want)[~zero] / want[~zero]
    assert err.max() < NORM_TOL[dt], (np.array(names)[~zero][int(np.argmax(err))], err.max())
    full = {}
    for k in (k[6:] for k in z.files if k.startswith("grad::") and not k.endswith("_sample")):
        if one and k == "temporal_transformer_blocks.0.attn1.to_q.weight":
            continue
        full[k] = _rel(_sample(z, "grad::" + k, named[k].grad.double().cpu().numpy()), z["grad::" + k])
    assert len(full) >= 9 and max(full.values()) < FULL_TOL[dt], full
    o = _rel(_sample(z, "out", out.detach().double().cpu().numpy()), z["out"])
    print(f"{tag} {dt}: norms {err.max():.2e}, full gradients {max(full.values()):.2e}, output {o:.2e}")
    assert o < NORM_TOL[dt] / 2


# ---------------------------------------------------------------------------------------------------------- checkpointing
FLOOR = {torch.float32: 1e-5, torch.float16: 2.0 ** -10}


def _img_case(dev):
    """F = 4 video frames + I = 3 images of 32^2 latents (256 tokens per frame), batch 2, a 3-D caption mask."""
    cfg = T.T2VConfig(num_attention_heads=2, attention_head_dim=64, num_layers=2, sample_size=32, video_length=4,
                      caption_channels=256)
    m = _module(cfg, T.make_weights(cfg, 9), dev)
    x, t, text = TI.make_img_inputs(cfg, 2, 3, 20, 10)
    mask = torch.ones(2, 4, 20)
    mask[1, 0, 12:] = 0
    mask[0, 2, 3:] = 0
    mask[1, 3, :] = 0
    x, t, text, mask = x.to(dev), t.to(dev), text.to(dev), mask.to(dev)

    def step(model):
        return model(x, t, encoder_hidden_states=text, encoder_attention_mask=mask, use_image_num=3).sample
    return m, step


def _run(m, step, precision, ckpt):
    m.zero_grad(set_to_none=True)
    m.gradient_checkpointing = ckpt
    if precision == "bf16_autocast":
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = step(m)
    else:
        out = step(m)
    gco = torch.randn(out.shape, generator=torch.Generator().manual_seed(4)).to(out.device, out.dtype)
    out.backward(gco)
    torch.cuda.synchronize()
    return out.detach().clone(), {k: p.grad.detach().clone() for k, p in m.named_parameters() if p.grad is not None}


@pytest.mark.parametrize("precision", ["bf16_autocast", "fp16_params"])
def test_checkpointed_step_matches_plain(dev, precision):
    """The bar of tests/test_gpu_train_checkpointing.py: outputs bit-identical; GEMM weight gradients that no atomic feeds
    bit-identical; the rest within the spread of two plain runs or the floor (1e-5 fp32, 2^-10 fp16, of their norm)."""
    m, step = _img_case(dev)
    if precision == "fp16_params":
        m.half()
    o1, g1 = _run(m, step, precision, False)
    o2, g2 = _run(m, step, precision, False)
    oc, gc = _run(m, step, precision, True)
    assert torch.equal(o1, o2) and torch.equal(o1, oc), "forward output differs"
    assert g1.keys() == g2.keys() == gc.keys() and len(gc) > 0
    det = [k for k in g1 if k.endswith(".weight") and "adaln_single" not in k]
    for k in det:
        assert torch.equal(g1[k], g2[k]) and torch.equal(gc[k], g1[k]), k
    med = torch.tensor([g.double().norm().item() for g in g1.values()]).median().item()
    worst = 0.0
    for k in g1.keys() - set(det):
        diff, spread = (gc[k].double() - g1[k].double()).norm().item(), (g2[k].double() - g1[k].double()).norm().item()
        floor = FLOOR[g1[k].dtype] * max(g1[k].double().norm().item(), med)
        worst = max(worst, diff / floor)
        assert torch.isfinite(gc[k]).all() and diff <= max(spread, floor), (k, diff, spread, floor)
    print(f"images {precision}: {len(det)} GEMM weight gradients bit-identical, {len(g1) - len(det)} others within "
          f"{worst:.3g} of their floor")


# ---------------------------------------------------------------------------------------------------------- Latte-1 shapes
def test_latte1_layer_geometry_against_torch_restatement(dev):
    """D 1152, 16 x 72, caption 4096, N 1024 (512^2), two layer pairs, batch 2 x (4 video frames + 2 images), L 120 with a 3-D
    mask: the native bf16 engine against the same engine on the fp32 torch restatement of its ops, on the GPU."""
    from latte_b200 import training_t2v
    from latte_b200.train_ops import NativeOps
    cfg = T.T2VConfig(num_attention_heads=16, attention_head_dim=72, num_layers=2, sample_size=64, video_length=4,
                      caption_channels=4096)
    I = 2
    sd = T.make_weights(cfg, 17)
    x, t, text = TI.make_img_inputs(cfg, 2, I, 120, 18)
    x, t, text = x.to(dev), t.to(dev), text.to(dev)
    bias = torch.zeros(2, 1 + I, 128, device=dev)
    bias[0, 0, 40:120] = -10000.0
    bias[1, 1, 12:120] = -10000.0
    bias[1, 2, 90:120] = -10000.0
    gco = torch.randn(2, 8, 4 + I, 64, 64, generator=torch.Generator().manual_seed(19)).to(dev)
    grads = []
    for ops, dt in ((NativeOps(torch.bfloat16), torch.bfloat16), (T2VTorchOps(torch.float32), torch.float32)):
        m = _module(cfg, sd, dev)
        emb = training_t2v.conditioning(m, t)
        out = training_t2v.train_forward(m, ops, dt, x, emb, text, bias, images=I)
        (out * gco).sum().backward()
        grads.append({k: p.grad.double().norm().item() for k, p in m.named_parameters()})
        del m, out
    got, want = grads
    for k in want:
        if k.endswith("to_k.bias"):
            continue
        assert abs(got[k] - want[k]) < 8e-2 * want[k], (k, got[k], want[k])


def test_latte1_full_checkpointed_step_with_adamw(dev):
    """The released Latte-1 geometry (28 layer pairs) at 1 x (16 + 4) x 512^2, L 120, with gradient checkpointing under bf16
    autocast: loss.backward(), clip_grad_norm_ and an AdamW step leave every .grad and every parameter finite."""
    from latte_b200 import LatteT2V
    torch.manual_seed(0)
    m = LatteT2V(video_length=16, sample_size=64).to(dev).train()
    m.enable_gradient_checkpointing()
    opt = torch.optim.AdamW(m.parameters(), lr=1e-4, weight_decay=0)
    x = torch.randn(1, 4, 20, 64, 64, device=dev)
    text = torch.randn(1, 5, 120, 4096, device=dev) * 0.5
    mask = torch.zeros(1, 5, 120, device=dev)
    for k, n in enumerate((30, 12, 120, 1, 64)):
        mask[0, k, :n] = 1
    with torch.autocast("cuda", dtype=torch.bfloat16):
        out = m(x, torch.tensor([500], device=dev), encoder_hidden_states=text, encoder_attention_mask=mask,
                use_image_num=4).sample
        loss = (out.float() ** 2).mean()
    assert out.shape == (1, 8, 20, 64, 64)
    loss.backward()
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in m.parameters())
    torch.nn.utils.clip_grad_norm_(m.parameters(), 1.0)
    opt.step()
    assert all(torch.isfinite(p).all() for p in m.parameters())


# ---------------------------------------------------------------------------------------------------------- refusals
def test_image_joint_refusals(dev):
    m, _ = _img_case(dev)
    cfg = T.T2VConfig(num_attention_heads=2, attention_head_dim=64, num_layers=2, sample_size=32, video_length=4,
                      caption_channels=256)
    x, t, text = (a.to(dev) for a in TI.make_img_inputs(cfg, 2, 3, 20, 10))
    mask3 = torch.ones(2, 4, 20, device=dev)
    with pytest.raises(ValueError, match="encoder_attention_mask"):         # a 2-D mask breaks the reference with images
        m(x, t, encoder_hidden_states=text, encoder_attention_mask=mask3[:, 0], use_image_num=3)
    with pytest.raises(ValueError, match="hidden_states"):
        m(x[:, :, :6], t, encoder_hidden_states=text, use_image_num=3)
    with pytest.raises(ValueError, match="encoder_hidden_states"):
        m(x, t, encoder_hidden_states=text[:, 0], use_image_num=3)
    with pytest.raises(NotImplementedError):
        m(x, t, encoder_hidden_states=text, attention_mask=torch.ones(2, 256, device=dev), use_image_num=3)
    with pytest.raises(NotImplementedError):
        m(x, t, encoder_hidden_states=text, use_image_num=3, enable_temporal_attentions=False)
    with pytest.raises(NotImplementedError, match="training only"):           # the reference's eval path fails with images
        with torch.no_grad():
            m(x, t, encoder_hidden_states=text, use_image_num=3)
    with pytest.raises(NotImplementedError, match="training only"):
        m.eval()(x, t, encoder_hidden_states=text, encoder_attention_mask=mask3, use_image_num=3)
    m.train()
    m64 = _module(T.T2VConfig(num_attention_heads=2, attention_head_dim=64, num_layers=1, sample_size=16, video_length=4,
                              caption_channels=256), T.make_weights(T.T2VConfig(num_attention_heads=2, attention_head_dim=64,
                                                                                num_layers=1, sample_size=16, video_length=4,
                                                                                caption_channels=256), 1), dev)
    with pytest.raises(NotImplementedError, match="128"):                     # N = 64: the images need whole 128-row tiles
        m64(torch.zeros(1, 4, 6, 16, 16, device=dev), t[:1], encoder_hidden_states=text[:1, :3], use_image_num=2)
    # use_image_num = 0 is untouched: the same module still trains on plain videos
    out = m(x[:, :, :4], t, encoder_hidden_states=text[:, 0], encoder_attention_mask=mask3[:, 0]).sample
    assert out.grad_fn is not None and out.shape[2] == 4
