"""GPU: LatteT2V training on the native path -- the cross-attention backward kernel against fp64 autograd, the step against the
UNMODIFIED reference's gradients (tests/golden/train_t2v_*.npz; tests/test_gpu_train.py's bars: every gradient norm within 1 %
in fp16, 8 % in bf16), the Latte-1 layer geometry against an fp32 torch restatement, and a full Latte-1 optimizer step."""
import os

import numpy as np
import pytest
import torch

from oracle import t2v_oracle as T
from oracle.train_t2v_ops_oracle import T2VTorchOps

pytestmark = pytest.mark.gpu

DTS = [torch.float16, torch.bfloat16]
NORM_TOL = {torch.float16: 1e-2, torch.bfloat16: 8e-2}


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


# ---------------------------------------------------------------------------------------------------------- the op
def _xattn_ref(q, kv, bias, do, B, rows, L, H):
    """fp64 autograd of softmax(q k^T / sqrt(hd) + bias) v on the 16-bit operands."""
    qq = q.double().requires_grad_(True)
    kk = kv.double().requires_grad_(True)
    D = q.shape[1]
    hd = D // H
    qh = qq.reshape(B, rows, H, hd).transpose(1, 2)
    kvh = kk.reshape(B, L, 2, H, hd)
    s = qh @ kvh[:, :, 0].transpose(1, 2).transpose(-1, -2) * hd ** -0.5
    if bias is not None:
        s = s + bias.double()[:, None, None, :L]
    o = (s.softmax(-1) @ kvh[:, :, 1].transpose(1, 2)).transpose(1, 2).reshape(B * rows, D)
    (o * do.double()).sum().backward()
    return o.detach(), qq.grad, kk.grad


CASES = [  # (batch, q_rows_per_batch, kv_len, heads, hd, mask)  mask: None, "partial", "all" (last sample fully masked)
    (1, 128, 1, 2, 64, None), (2, 128, 20, 4, 72, "partial"), (3, 4096, 77, 2, 64, "all"), (2, 4096, 120, 4, 72, "partial"),
    (1, 16384, 128, 2, 72, None), (1, 16384, 120, 16, 72, "partial"), (3, 128, 128, 2, 64, "all"), (2, 4096, 1, 2, 72, "all"),
]


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("case", CASES)
def test_cross_attention_bwd_op(dev, dt, case):
    from latte_b200.train_ops import NativeOps
    B, rows, L, H, hd = case[:5]
    D = H * hd
    g = torch.Generator(device=dev).manual_seed(rows + L + hd)
    q = torch.randn(B * rows, D, device=dev, generator=g).to(dt)
    kv_all = torch.randn(B * L, 3 * 2 * D, device=dev, generator=g).to(dt)      # a column window of a wider stacked buffer
    col = 2 * D
    kv = kv_all[:, col:col + 2 * D]
    bias = None
    if case[5] is not None:
        bias = torch.zeros(B, 128, device=dev)
        bias[0, L // 2 + 1:L] = -10000.0
        if case[5] == "all":
            bias[B - 1, :L] = -10000.0
    do = (torch.randn(B * rows, D, device=dev, generator=g) * 1e-2).to(dt)
    ops = NativeOps(dt)
    o = ops.cross_attention(q, kv, B, rows, L, H, bias)
    o_ref, dq_ref, dkv_ref = _xattn_ref(q, kv.contiguous(), bias, do, B, rows, L, H)
    assert (o.double() - o_ref).abs().max().item() < 2e-2
    res = []
    for _ in range(2):
        dkv = torch.full((B * L, 4 * 2 * D), float("nan"), device=dev, dtype=dt)
        dq = ops.cross_attention_bwd(q, kv, o, do, B, rows, L, H, bias, dkv, col + 8)
        torch.cuda.synchronize()
        res.append((dq, dkv))
    dq, dkv = res[0]
    assert torch.equal(res[1][0], dq) and torch.equal(res[1][1].nan_to_num(7.0), dkv.nan_to_num(7.0)), "reruns differ"
    win = dkv[:, col + 8:col + 8 + 2 * D]
    assert torch.isfinite(dq).all() and torch.isfinite(win).all()
    assert torch.isnan(dkv[:, :col + 8]).all() and torch.isnan(dkv[:, col + 8 + 2 * D:]).all(), "bytes outside the window written"
    eps = {torch.float16: 2e-2, torch.bfloat16: 6e-2}[dt]
    # with one key dQ and dK are exactly zero (P = 1, dS = 0): the kernel's rounding noise is held to the scale of dO instead
    floor = do.double().norm().item()
    for got, want in ((dq, dq_ref), (win, dkv_ref)):
        err = ((got.double() - want).norm() / max(want.norm().item(), floor)).item()
        assert err < eps, err


def test_cross_attention_bwd_refusals(dev):
    from latte_b200 import _lib
    lib = _lib.load()
    assert lib.b200_cross_attention_bwd_workspace_bytes(1, 128, 20, 2, 80) == 0 and "head_dim 80" in _lib.last_error()
    assert lib.b200_cross_attention_bwd_workspace_bytes(1, 128, 129, 2, 64) == 0
    assert lib.b200_cross_attention_bwd_workspace_bytes(1, 192, 20, 2, 64) == 0
    rc = lib.b200_cross_attention_bwd(None, None, None, None, None, None, None, 0, 0, 1, 128, 20, 160, 320, 2, 80, _lib.BF16,
                                      None, 0, None)
    assert rc == -7 and "head_dim 80" in _lib.last_error()          # B200_ERR_UNSUPPORTED


# ---------------------------------------------------------------------------------------------------------- the step
def _module(cfg, sd, dev):
    from latte_b200 import LatteT2V
    m = LatteT2V(num_attention_heads=cfg.num_attention_heads, attention_head_dim=cfg.attention_head_dim,
                 in_channels=cfg.in_channels, out_channels=cfg.out_channels, num_layers=cfg.num_layers, patch_size=cfg.patch_size,
                 sample_size=cfg.sample_size, caption_channels=cfg.caption_channels, video_length=cfg.video_length)
    m.load_state_dict(sd, strict=True)
    return m.to(dev).train()


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("tag", ["tiny_b2_l20", "tiny_b2_l20_masked", "hd72_b2_l120_masked", "f1_b2_l20"])
def test_native_step_matches_reference_gradients(dev, golden_dir, dt, tag):
    z = np.load(os.path.join(golden_dir, f"train_t2v_{tag}.npz"))
    cfg = T.T2VConfig(**eval(str(z["cfg"])))
    x, t, text = T.make_inputs(cfg, int(z["batch"]), int(z["text_len"]), int(z["iseed"]))
    m = _module(cfg, T.make_weights(cfg, int(z["wseed"])), dev)
    m.train_dtype = dt
    mask = torch.from_numpy(z["mask"]).to(dev) if "mask" in z else None
    out = m(x.to(dev), t.to(dev), encoder_hidden_states=text.to(dev), encoder_attention_mask=mask).sample
    assert out.grad_fn is not None
    gco = torch.randn(out.shape, generator=torch.Generator().manual_seed(int(z["gseed"]))).to(dev)
    (out * gco).sum().backward()
    names = [str(n) for n in z["grad_names"]]
    named = dict(m.named_parameters())
    assert all(named[n].grad is not None for n in names)
    want = z["grad_norms"]
    got = np.array([named[n].grad.double().norm().item() for n in names])
    # exactly-zero gradients (key biases; q / k of a one-frame temporal attention) are rounding noise: an absolute bound
    zero = np.array([n.endswith("to_k.bias") or (cfg.video_length == 1 and n.startswith("temporal_") and
                                                  (".to_q." in n or ".to_k." in n)) for n in names])
    assert np.all(got[zero] < NORM_TOL[dt] * np.median(want))
    err = np.abs(got - want)[~zero] / want[~zero]
    assert err.max() < NORM_TOL[dt], (np.array(names)[~zero][int(np.argmax(err))], err.max())
    ref_out = torch.from_numpy(z["out"])
    o = out.detach().cpu()
    if "out_sample" in z:
        o = o[:, :, ::int(z["out_sample"][1])]
    assert ((o - ref_out).norm() / ref_out.norm()).item() < NORM_TOL[dt] / 2


LATTE1_LAYER = dict(num_attention_heads=16, attention_head_dim=72, num_layers=2, sample_size=32, video_length=16, caption_channels=4096)


def test_latte1_layer_geometry_against_torch_restatement(dev):
    """D 1152, 16 x 72, caption 4096, L 120 (12 valid in sample 1), two layer pairs, 16 x 256^2: the native bf16 engine against
    the same engine on the fp32 torch restatement of its ops, on the GPU."""
    from latte_b200 import training_t2v
    from latte_b200.train_ops import NativeOps
    cfg = T.T2VConfig(**LATTE1_LAYER)
    sd = T.make_weights(cfg, 17)
    x, t, text = T.make_inputs(cfg, 2, 120, 18)
    x, t, text = x.to(dev), t.to(dev), text.to(dev)
    bias = torch.zeros(2, 128, device=dev)
    bias[1, 12:120] = -10000.0
    gco = torch.randn(2, 8, 16, 32, 32, generator=torch.Generator().manual_seed(19)).to(dev)
    grads = []
    for ops, dt in ((NativeOps(torch.bfloat16), torch.bfloat16), (T2VTorchOps(torch.float32), torch.float32)):
        m = _module(cfg, sd, dev)
        emb = training_t2v.conditioning(m, t)
        out = training_t2v.train_forward(m, ops, dt, x, emb, text, bias)
        (out * gco).sum().backward()
        grads.append({k: p.grad.double().norm().item() for k, p in m.named_parameters()})
        del m, out
    got, want = grads
    for k in want:
        if k.endswith("to_k.bias"):
            continue
        assert abs(got[k] - want[k]) < 8e-2 * want[k], (k, got[k], want[k])


def test_latte1_full_step_with_adamw(dev):
    """The released Latte-1 geometry (28 layer pairs, 16 x 512^2, batch 1, L 120) under bf16 autocast: loss.backward(),
    clip_grad_norm_ and an AdamW step leave every .grad and every parameter finite."""
    from latte_b200 import LatteT2V
    torch.manual_seed(0)
    m = LatteT2V(video_length=16, sample_size=64).to(dev).train()
    opt = torch.optim.AdamW(m.parameters(), lr=1e-4, weight_decay=0)
    x = torch.randn(1, 4, 16, 64, 64, device=dev)
    text = torch.randn(1, 120, 4096, device=dev) * 0.5
    mask = torch.ones(1, 120, device=dev)
    mask[:, 30:] = 0
    with torch.autocast("cuda", dtype=torch.bfloat16):
        out = m(x, torch.tensor([500], device=dev), encoder_hidden_states=text, encoder_attention_mask=mask).sample
        loss = (out.float() ** 2).mean()
    loss.backward()
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in m.parameters())
    torch.nn.utils.clip_grad_norm_(m.parameters(), 1.0)
    opt.step()
    assert all(torch.isfinite(p).all() for p in m.parameters())


def test_training_refusals(dev):
    cfg = T.T2VConfig(num_attention_heads=2, attention_head_dim=64, num_layers=1, sample_size=16, video_length=8, caption_channels=256)
    m = _module(cfg, T.make_weights(cfg, 1), dev)
    x = torch.zeros(1, 4, 8, 16, 16, device=dev)
    t = torch.tensor([1], device=dev)
    text = torch.zeros(1, 20, 256, device=dev)
    with pytest.raises(NotImplementedError):
        m(x, t, encoder_hidden_states=text, use_image_num=2)
    with pytest.raises(NotImplementedError):
        m(x, t, encoder_hidden_states=text, enable_temporal_attentions=False)
    with pytest.raises(NotImplementedError):
        m(x, t, encoder_hidden_states=text.clone().requires_grad_(True))
    m80 = _module(T.T2VConfig(num_attention_heads=2, attention_head_dim=80, num_layers=1, sample_size=16, video_length=8,
                              caption_channels=256), T.make_weights(T.T2VConfig(num_attention_heads=2, attention_head_dim=80,
                                                                                num_layers=1, sample_size=16, video_length=8,
                                                                                caption_channels=256), 1), dev)
    with pytest.raises(NotImplementedError):
        m80(x, t, encoder_hidden_states=text)
    with pytest.raises(ValueError):
        m(x[:, :, :4], t, encoder_hidden_states=text)
    # grad-free and eval calls keep the sampling path: no autograd node
    with torch.no_grad():
        assert m(x, t, encoder_hidden_states=text).sample.grad_fn is None
    assert m.eval()(x, t, encoder_hidden_states=text).sample.grad_fn is None
