"""GPU: training at video lengths above 16 frames.  (1) The temporal attention backward for 17..128 frames (the two-kernel
tensor-core backward over strided rows, csrc/train.cu) against the fp32 torch restatement of the op
(oracle/train_ops_oracle.TorchOps), including token counts that are not multiples of anything, stale NaN in the output and
statistics buffers, and an all-NaN sequence next to finite ones; (2) the whole native training step against the UNMODIFIED
reference at F = 1, 20 and 32 (tests/golden/train_tiny64_f*.npz) and, at the XL head geometry (head_dim 72, 256 tokens,
32 frames), against the same engine through TorchOps in fp32.  Tolerances as tests/test_gpu_train.py."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DTS = [torch.float16, torch.bfloat16]
EPS = {torch.float16: 1e-3, torch.bfloat16: 8e-3}


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


def _ops(dt):
    from latte_b200.train_ops import NativeOps
    from oracle.train_ops_oracle import TorchOps
    return NativeOps(dt), TorchOps(dt)


def _rel(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


def _inputs(dev, dt, B, Fr, N, H, hd, seed):
    g = torch.Generator().manual_seed(seed)
    T, D = B * Fr * N, H * hd
    return torch.randn(T, 3 * D, generator=g).to(dev).to(dt), torch.randn(T, D, generator=g).to(dev).to(dt)


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("hd", [64, 72])
@pytest.mark.parametrize("frames", [17, 20, 24, 31, 32, 48, 64, 100, 128])
def test_temporal_attention_backward(dev, dt, hd, frames):
    """dqkv of softmax(QK^T hd^-1/2)V over the F frames of each (b, n): 3 tokens per frame (so the forward's last token group
    is partial at every F here) and 3 heads; F = 64 / 128 fill whole 64-row blocks, the others end in a partial one."""
    nat, ref = _ops(dt)
    B, N, H = 2, 3, 3
    D = H * hd
    qkv, do = _inputs(dev, dt, B, frames, N, H, hd, frames * 10 + hd)
    o = nat.attention(qkv, B, frames, N, H, True)
    got = nat.attention_bwd(qkv, o, do, B, frames, N, H, True)
    want = ref.attention_bwd(qkv, o, do, B, frames, N, H, True)
    for k, name in enumerate(("dq", "dk", "dv")):
        e = _rel(got[:, k * D:(k + 1) * D], want[:, k * D:(k + 1) * D])
        assert e < 3 * EPS[dt], f"{name}: relative Frobenius error {e:.3e}"


def _bwd_raw(qkv, o, do, dqkv, stats, B, Fr, N, H, hd, dt):
    from latte_b200 import _lib
    rc = _lib.load().b200_attention_bwd(qkv.data_ptr(), o.data_ptr(), do.data_ptr(), dqkv.data_ptr(),
                                        stats.data_ptr() if stats is not None else None, B, Fr, N, H, hd,
                                        _lib.BF16 if dt == torch.bfloat16 else _lib.FP16, 1,
                                        torch.cuda.current_stream(qkv.device).cuda_stream)
    return rc


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("frames", [20, 100])
def test_temporal_backward_stale_nan_and_nan_sequence(dev, dt, frames):
    """Every row of dqkv is written (a NaN-filled output and statistics buffer leave no trace), and an all-NaN sequence --
    token n = 2 of sample 1, every frame -- changes no bit of the other sequences' gradients."""
    from latte_b200 import _lib
    nat, _ = _ops(dt)
    B, N, H, hd = 2, 5, 2, 72
    qkv, do = _inputs(dev, dt, B, frames, N, H, hd, 77 + frames)
    o = nat.attention(qkv, B, frames, N, H, True)
    clean = nat.attention_bwd(qkv, o, do, B, frames, N, H, True)
    dqkv = torch.full_like(qkv, float("nan"))
    stats = torch.full((2 * B * frames * H * N,), float("nan"), dtype=torch.float32, device=dev)
    _lib.check(_bwd_raw(qkv, o, do, dqkv, stats, B, frames, N, H, hd, dt), "b200_attention_bwd")
    torch.cuda.synchronize()
    assert torch.equal(dqkv, clean)
    rows = torch.tensor([(1 * frames + f) * N + 2 for f in range(frames)], device=dev)
    q2, o2, do2 = qkv.clone(), o.clone(), do.clone()
    for t in (q2, o2, do2):
        t[rows] = float("nan")
    dqkv.fill_(float("nan"))
    stats.fill_(float("nan"))
    _lib.check(_bwd_raw(q2, o2, do2, dqkv, stats, B, frames, N, H, hd, dt), "b200_attention_bwd")
    torch.cuda.synchronize()
    keep = torch.ones(qkv.shape[0], dtype=torch.bool, device=dev)
    keep[rows] = False
    assert torch.isfinite(dqkv[keep]).all()
    assert torch.equal(dqkv[keep], clean[keep])


def test_temporal_backward_head_dim_80_is_unsupported(dev):
    nat, _ = _ops(torch.bfloat16)
    B, N, H, hd = 1, 2, 2, 80
    for Fr in (8, 32):                     # the one-warp kernel (<= 16 frames) and the strided two-kernel path
        qkv, do = _inputs(dev, torch.bfloat16, B, Fr, N, H, hd, 3)
        o = torch.zeros_like(do)
        with pytest.raises(RuntimeError, match="UNSUPPORTED"):
            nat.attention_bwd(qkv, o, do, B, Fr, N, H, True)


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("frames", [1, 20, 32])
def test_training_step_matches_reference_gradients(dev, golden_dir, dt, frames):
    """model.train() + diffusion.training_losses + loss.backward() on the native path at F = 1, 20, 32."""
    from latte_b200 import Latte
    from latte_b200.diffusion import create_diffusion
    from oracle import latte_oracle as O
    g = np.load(os.path.join(golden_dir, f"train_tiny64_f{frames}.npz"))
    cfg = O.make_config("Latte-tiny64/2", input_size=16, num_frames=frames)
    m = Latte(input_size=16, hidden_size=128, depth=2, num_heads=2, num_frames=frames, num_classes=101, extras=2)
    m.load_state_dict(O.make_weights(cfg, 21), strict=True)
    m = m.to(dev).train()
    m.y_embedder.dropout_prob = 0.0          # the golden was generated without label dropout (no RNG in the comparison)
    m.train_dtype = dt
    d = create_diffusion(timestep_respacing="")
    x0, noise = torch.from_numpy(g["x0"]).to(dev), torch.from_numpy(g["noise"]).to(dev)
    t, y = torch.from_numpy(g["t"]).to(dev), torch.from_numpy(g["y"]).to(dev)
    terms = d.training_losses(m, x0, t, dict(y=y), noise=noise)
    loss = terms["loss"].mean()
    assert abs(loss.item() - float(g["loss"])) < 10 * EPS[dt] * abs(float(g["loss"]))
    loss.backward()
    named = dict(m.named_parameters())
    for k, want in zip([str(n) for n in g["grad_names"]], g["grad_norms"]):
        got = named[k].grad.double().norm().item()
        assert abs(got - want) <= 10 * EPS[dt] * want, (k, got, want)
    for key in g.files:
        if key.startswith("grad::"):
            e = _rel(named[key[6:]].grad, torch.from_numpy(g[key]).to(dev))
            assert e < 10 * EPS[dt], (key, e)


@pytest.mark.parametrize("dt", DTS)
def test_training_step_xl_head_geometry_32_frames(dev, dt):
    """head_dim 72, 256 tokens, 32 frames, depth 4 (Latte-tiny72/2): native engine vs the same engine through TorchOps in fp32."""
    from latte_b200 import Latte, training
    from latte_b200.train_ops import NativeOps
    from oracle import latte_oracle as O
    from oracle.train_ops_oracle import TorchOps
    cfg = O.make_config("Latte-tiny72/2", input_size=32, num_frames=32)
    m = Latte(input_size=32, hidden_size=576, depth=4, num_heads=8, num_frames=32, num_classes=101, extras=2)
    m.load_state_dict(O.make_weights(cfg, 5), strict=True)
    m = m.to(dev)
    gen = torch.Generator().manual_seed(19)
    x = torch.randn(2, 32, 4, 32, 32, generator=gen).to(dev)
    t = torch.tensor([3, 700], device=dev)
    y = torch.tensor([4, 101], device=dev)
    dout = torch.randn(2, 32, 8, 32, 32, generator=gen).to(dev)
    grads = []
    for ops, od in ((NativeOps(dt), dt), (TorchOps(torch.float32), torch.float32)):
        m.zero_grad(set_to_none=True)
        out = training.train_forward(m, ops, od, x, training.conditioning(m, t, y))
        out.backward(dout)
        grads.append(({k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None}, out.detach()))
    (gn, on), (gr, orf) = grads
    assert _rel(on, orf) < 3 * EPS[dt]
    assert set(gn) == set(gr)
    for k in gr:
        e = _rel(gn[k], gr[k])
        assert e < 8 * EPS[dt], (k, e)


def test_autocast_training_step_at_32_frames_is_finite(dev):
    """Latte(num_frames=32) in training mode under torch.autocast(bfloat16): loss.backward() completes, every gradient finite."""
    from latte_b200 import Latte
    from latte_b200.diffusion import create_diffusion
    torch.manual_seed(0)
    m = Latte(input_size=16, hidden_size=128, depth=2, num_heads=2, num_frames=32, num_classes=11, extras=2).to(dev).train()
    d = create_diffusion(timestep_respacing="")
    g = torch.Generator().manual_seed(4)
    x = torch.randn(2, 32, 4, 16, 16, generator=g).to(dev)
    y = torch.tensor([1, 7], device=dev)
    t = torch.tensor([10, 900], device=dev)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        loss = d.training_losses(m, x, t, dict(y=y))["loss"].mean()
    loss.backward()
    assert torch.isfinite(loss)
    grads = [p.grad for p in m.parameters() if p.requires_grad]
    assert all(gr is not None and torch.isfinite(gr).all() for gr in grads)
