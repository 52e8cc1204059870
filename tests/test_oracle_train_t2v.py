"""CPU: LatteT2V training -- the torch oracle and the training engine (latte_b200/training_t2v.py on the torch restatement of its
ops) against the vector-Jacobian products of the UNMODIFIED reference module (tests/golden/train_t2v_*.npz,
oracle/make_golden_train_t2v.py)."""
import os

import numpy as np
import pytest
import torch

from oracle import t2v_oracle as T
from oracle.train_t2v_ops_oracle import T2VTorchOps

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TAGS = ["tiny_b2_l20", "tiny_b2_l20_masked", "hd72_b2_l120_masked", "f1_b2_l20"]


def load(tag):
    z = np.load(os.path.join(GOLDEN, f"train_t2v_{tag}.npz"))
    cfg = T.T2VConfig(**eval(str(z["cfg"])))
    B, L = int(z["batch"]), int(z["text_len"])
    sd = T.make_weights(cfg, int(z["wseed"]))
    x, t, text = T.make_inputs(cfg, B, L, int(z["iseed"]))
    mask = torch.from_numpy(z["mask"]) if "mask" in z else None
    return z, cfg, sd, x, t, text, mask


def cotangent(z, shape):
    return torch.randn(shape, generator=torch.Generator().manual_seed(int(z["gseed"])))


def sample(z, key, a):
    """The entries of `a` that the golden stores under `key` (strided along one axis for the larger arrays)."""
    if key + "_sample" in z:
        axis, step = (int(v) for v in z[key + "_sample"])
        sl = [slice(None)] * a.ndim
        sl[axis] = slice(None, None, step)
        a = a[tuple(sl)]
    return a


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def compare(z, out, grads, tol_norm, tol_full, tol_out):
    assert rel(sample(z, "out", out), z["out"]) < tol_out
    names = [str(n) for n in z["grad_names"]]
    assert sorted(names) == sorted(grads), set(names) ^ set(grads)
    got = np.array([np.linalg.norm(grads[n].astype(np.float64)) for n in names])
    want = z["grad_norms"]
    # Gradients that are exactly zero in exact arithmetic have norms of rounding noise on both sides; they are held to an
    # absolute bound instead: every key bias (softmax is shift-invariant), and q / k of a temporal attention over one frame.
    frames = T.T2VConfig(**eval(str(z["cfg"]))).video_length
    zero = np.array([n.endswith("to_k.bias") or (frames == 1 and n.startswith("temporal_") and
                                                  (".to_q." in n or ".to_k." in n)) for n in names])
    floor = tol_norm * np.median(want)
    assert np.all(got[zero] < floor) and np.all(want[zero] < floor), [n for n, zz in zip(names, zero) if zz]
    err = np.abs(got - want)[~zero] / want[~zero]
    assert err.max() < tol_norm, (np.array(names)[~zero][int(np.argmax(err))], err.max())
    full = [k[6:] for k in z.files if k.startswith("grad::") and not k.endswith("_sample")]
    assert len(full) == 10
    for k in full:
        if frames == 1 and k == "temporal_transformer_blocks.0.attn1.to_q.weight":
            continue                        # exactly zero, see above
        assert rel(sample(z, "grad::" + k, grads[k]), z["grad::" + k]) < tol_full, k


@pytest.mark.parametrize("tag", TAGS)
def test_oracle_autograd_matches_reference(tag):
    z, cfg, sd, x, t, text, mask = load(tag)
    sd = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    out = T.t2v_forward(sd, cfg, x, t, text, text_mask=mask)
    (out * cotangent(z, out.shape)).sum().backward()
    compare(z, out.detach().numpy(), {k: v.grad.numpy() for k, v in sd.items()}, 1e-4, 1e-4, 1e-5)


def build_module(cfg, sd):
    from latte_b200 import LatteT2V
    m = LatteT2V(num_attention_heads=cfg.num_attention_heads, attention_head_dim=cfg.attention_head_dim,
                 in_channels=cfg.in_channels, out_channels=cfg.out_channels, num_layers=cfg.num_layers, patch_size=cfg.patch_size,
                 sample_size=cfg.sample_size, caption_channels=cfg.caption_channels, video_length=cfg.video_length)
    m.load_state_dict(sd, strict=True)
    return m.train()


def engine_step(tag, dtype):
    from latte_b200 import training_t2v
    z, cfg, sd, x, t, text, mask = load(tag)
    m = build_module(cfg, sd)
    bias = None
    if mask is not None:
        bias = torch.zeros(mask.shape[0], 128)
        bias[:, : mask.shape[1]] = (1.0 - mask.float()) * -10000.0
    emb = training_t2v.conditioning(m, t)
    out = training_t2v.train_forward(m, T2VTorchOps(dtype), dtype, x, emb, text, bias)
    (out * cotangent(z, out.shape)).sum().backward()
    return z, out.detach().numpy(), {k: p.grad.numpy() for k, p in m.named_parameters()}


@pytest.mark.parametrize("tag", TAGS)
def test_engine_fp32_matches_reference(tag):
    z, out, grads = engine_step(tag, torch.float32)
    compare(z, out, grads, 1e-5, 1e-5, 1e-5)


@pytest.mark.parametrize("tag", ["tiny_b2_l20_masked", "f1_b2_l20"])
def test_engine_bf16_operands(tag):
    """bf16 operand rounding at every GEMM / attention input (the GPU's arithmetic, on the CPU): gradient norms within 5 %."""
    z, out, grads = engine_step(tag, torch.bfloat16)
    compare(z, out, grads, 5e-2, 6e-2, 2e-2)


def test_cross_attention_bwd_matches_autograd():
    """T2VTorchOps.cross_attention_bwd against torch autograd of T2VTorchOps.cross_attention, with a partial mask, an
    all-masked sample and a K/V column window of a wider stacked buffer."""
    g = torch.Generator().manual_seed(3)
    B, rows, L, H, hd = 3, 128, 20, 2, 72
    D = H * hd
    q = torch.randn(B * rows, D, generator=g, dtype=torch.float64)
    kv_all = torch.randn(B * L + 4, 3 * 2 * D, generator=g, dtype=torch.float64)
    bias = torch.zeros(B, 128, dtype=torch.float64)
    bias[1, 7:L] = -10000.0
    bias[2, :L] = -10000.0
    do = torch.randn(B * rows, D, generator=g, dtype=torch.float64)
    ops = T2VTorchOps(torch.float64)              # fp32 math inside, like the kernels
    col0 = 2 * D
    qq, kk = q.clone().requires_grad_(True), kv_all[:, col0:col0 + 2 * D].clone().requires_grad_(True)
    o = ops.cross_attention(qq, kk, B, rows, L, H, bias)
    (o * do).sum().backward()
    dkv = torch.full_like(kv_all, float("nan"))
    dq = ops.cross_attention_bwd(q, kv_all[:, col0:col0 + 2 * D], o.detach(), do, B, rows, L, H, bias, dkv, col0)
    torch.testing.assert_close(dq, qq.grad, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(dkv[: B * L, col0:col0 + 2 * D], kk.grad[: B * L], rtol=1e-5, atol=1e-5)
    assert torch.isnan(dkv[:, :col0]).all() and torch.isnan(dkv[:, col0 + 2 * D:]).all() and torch.isnan(dkv[B * L:]).all()
    # the all-masked sample is the reference's softmax of equally shifted scores: finite, and the unmasked softmax up to the fp32
    # rounding of (score - 10000)
    o_free = ops.cross_attention(q, kv_all[:, col0:col0 + 2 * D], B, rows, L, H, None)
    assert torch.isfinite(o).all() and torch.isfinite(dq).all()
    torch.testing.assert_close(o.detach()[2 * rows:], o_free[2 * rows:], rtol=0, atol=2e-3)


def test_trainable_names_cover_every_parameter():
    from latte_b200 import training_t2v
    z, cfg, sd, *_ = load("tiny_b2_l20")
    m = build_module(cfg, sd)
    names = training_t2v.trainable_names(m)
    rest = [n for n, _ in m.named_parameters() if n not in names]
    assert rest and all(n.startswith("adaln_single.emb.") for n in rest)
    assert len(names) + len(rest) == len(list(m.parameters())) == len(z["grad_names"])


def test_training_refusals_before_any_launch():
    """The training path refuses what it does not build before touching a device (CPU tensors reach these checks)."""
    from latte_b200 import LatteT2V
    z, cfg, sd, x, t, text, mask = load("tiny_b2_l20")
    m = build_module(cfg, sd)
    with pytest.raises(NotImplementedError, match="temporal"):
        m._run_train(x, t, text, None, False, True)
    with pytest.raises(NotImplementedError, match="require grad"):
        m._run_train(x, t, text.clone().requires_grad_(True), None, True, True)
    with pytest.raises(ValueError, match="hidden_states"):
        m._run_train(x[:, :, :4], t, text, None, True, True)
    m80 = LatteT2V(num_attention_heads=2, attention_head_dim=80, num_layers=1, sample_size=16, video_length=8,
                   caption_channels=256).train()
    with pytest.raises(NotImplementedError, match="head_dim 80"):
        m80._run_train(torch.zeros(1, 4, 8, 16, 16), t[:1], torch.zeros(1, 4, 256), None, True, True)
    with pytest.raises(RuntimeError, match="CUDA"):
        m(x, t, encoder_hidden_states=text)
