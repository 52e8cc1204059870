"""GPU: the training step (BASELINE config 5).  (1) every kernel of csrc/train.cu against the torch restatement of the same op
(oracle/train_ops_oracle.TorchOps: fp32 math on the same 16-bit inputs, one rounding at the output); (2) the whole native
forward + backward through `model(x, t, y)` / `loss.backward()` against the gradients of the UNMODIFIED reference
(tests/golden/train_tiny64.npz) and, at the XL head geometry (head_dim 72, 256 tokens, 16 frames), against the same engine
driven through TorchOps in fp32 on the GPU.  Tolerances: 16-bit operand rounding (fp16 2^-11, bf16 2^-8 relative per operand)."""
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


def _close(a, b, tol, what=""):
    a, b = a.float(), b.float()
    err = (a - b).abs().max().item()
    scale = b.abs().max().item() + 1e-12
    assert err <= tol * scale, f"{what}: max-abs {err:.3e} vs scale {scale:.3e} (tol {tol})"


@pytest.mark.parametrize("dt", DTS)
def test_transpose_cast_colsum(dev, dt):
    nat, ref = _ops(dt)
    g = torch.Generator().manual_seed(1)
    for R, Cc in [(1536, 128), (4096, 1152), (512, 32), (130, 68)]:
        a = torch.randn(R, Cc, generator=g).to(dev).to(dt)
        assert torch.equal(nat.transpose(a), a.t().contiguous())
        base = torch.randn(Cc, generator=g).to(dev)                      # reductions accumulate into the buffer handed in
        _close(nat.colsum(a, base.clone()), ref.colsum(a, base.clone()), 1e-5, "colsum16")
    w = torch.randn(384, 1152, generator=g).to(dev)
    assert torch.equal(nat.cast(w), w.to(dt))
    x = torch.randn(2048, 384, generator=g).to(dev)
    assert torch.equal(nat.to_operand(x), x.to(dt))
    _close(nat.colsum(x, torch.zeros(384, device=dev)), x.sum(0), 1e-5, "colsum32")


@pytest.mark.parametrize("dt", DTS)
def test_linear_accum_small_and_wgrad_shapes(dev, dt):
    """wgrad = dY^T . X through the residual epilogue with a unit gate (fp32 accumulate into the gradient), incl. M = 32
    (final layer), N = 64 (patch embed) and M = 5 (adaLN rows through the 16-bit epilogue)."""
    nat, ref = _ops(dt)
    g = torch.Generator().manual_seed(2)
    for M, N, K in [(32, 1152, 2048), (1152, 64, 4096), (384, 128, 1536), (3456, 1152, 8192)]:
        a = torch.randn(M, K, generator=g).to(dev).to(dt)
        w = torch.randn(N, K, generator=g).to(dev).to(dt)
        base = torch.randn(M, N, generator=g).to(dev)
        got = nat.linear_accum(base.clone(), a, w)
        want = ref.linear_accum(base.clone(), a, w)
        _close(got, want, 2e-5, f"linear_accum {M}x{N}x{K}")
    a = torch.randn(5, 1152, generator=g).to(dev).to(dt)
    w = (torch.randn(6912 + 2304, 1152, generator=g) / 34).to(dev).to(dt)
    b = torch.randn(6912 + 2304, generator=g).to(dev)
    _close(nat.linear(a, w, b), ref.linear(a, w, b), EPS[dt], "linear M=5")


@pytest.mark.parametrize("dt", DTS)
def test_wgrad_reads_untransposed_operands(dev, dt):
    """dW += dY^T X with both activations as they lie in memory (the GEMM's MN-major wgmma descriptors, 64-wide block loads):
    full tiles, the half-width edge tile (n_in = 1152 = 4.5 x 256), ragged n_out (32, 1152 = 4.5 x 256 rows), stream-K."""
    nat, ref = _ops(dt)
    g = torch.Generator().manual_seed(7)
    for rows, n_out, n_in in [(2048, 32, 1152), (4096, 1152, 128), (1536, 384, 128), (8192, 3456, 1152), (20480, 1152, 4608),
                              (4096, 512, 256), (2048, 1152, 576), (20480, 1152, 1152), (4096, 1152, 1152)]:   # last two: 25 tiles of 256 cut into 3 K-segments each
        dy = torch.randn(rows, n_out, generator=g).to(dev).to(dt)
        x = torch.randn(rows, n_in, generator=g).to(dev).to(dt)
        base = torch.randn(n_out, n_in, generator=g).to(dev)
        got = nat.wgrad(base.clone(), dy, x)
        want = ref.wgrad(base.clone(), dy, x)
        _close(got, want, 3e-5, f"wgrad {rows}x{n_out}x{n_in}")
        again = nat.wgrad(base.clone(), dy, x)
        assert torch.equal(got, again), "ordered stream-K must be bit-reproducible"


@pytest.mark.parametrize("dt", DTS)
def test_dgrad_reads_the_weight_in_place(dev, dt):
    """dX = dY W with W in its nn.Linear [out, in] layout: A K-major, W through an MN-major wgmma descriptor (no W^T copy);
    n_in = 576 takes the explicit-transpose fallback."""
    nat, ref = _ops(dt)
    g = torch.Generator().manual_seed(8)
    for rows, n_out, n_in in [(4096, 1152, 1152), (2048, 4608, 1152), (2048, 1152, 4608), (1536, 384, 128), (2048, 64, 1152),
                              (20480, 3456, 1152), (1024, 576, 576), (200, 128, 256)]:
        dy = torch.randn(rows, n_out, generator=g).to(dev).to(dt)
        w = (torch.randn(n_out, n_in, generator=g) / n_out ** 0.5).to(dev).to(dt)
        _close(nat.dgrad(dy, w), ref.dgrad(dy, w), EPS[dt], f"dgrad {rows}x{n_out}x{n_in}")


@pytest.mark.parametrize("dt", DTS)
def test_elementwise_forward_ops(dev, dt):
    nat, ref = _ops(dt)
    g = torch.Generator().manual_seed(3)
    B, Fr, N, D = 3, 8, 64, 384
    T, rpb = B * Fr * N, Fr * N
    x = torch.randn(T, D, generator=g).to(dev)
    m = torch.randn(T, D, generator=g).to(dev).to(dt)
    mod = torch.randn(B, 6 * D, generator=g).to(dev)
    gate = mod[:, 2 * D:3 * D]
    temp = torch.randn(Fr, D, generator=g).to(dev)
    _close(nat.gate_residual(x, m, gate, rpb), ref.gate_residual(x, m, gate, rpb), 1e-6, "gate_residual")
    _close(nat.gate_residual(x, m, gate, rpb, row_add=temp, tokens=N), ref.gate_residual(x, m, gate, rpb, row_add=temp, tokens=N),
           1e-6, "gate_residual+temp")


@pytest.mark.parametrize("dt", DTS)
def test_elementwise_backward_ops(dev, dt):
    nat, ref = _ops(dt)
    g = torch.Generator().manual_seed(4)
    B, Fr, N, D = 3, 8, 64, 384
    T, rpb = B * Fr * N, Fr * N
    dx = torch.randn(T, D, generator=g).to(dev)
    m = torch.randn(T, D, generator=g).to(dev).to(dt)
    mod = torch.randn(B, 6 * D, generator=g).to(dev)
    gate, shift, scale = mod[:, 2 * D:3 * D], mod[:, 0:D], mod[:, D:2 * D]
    dmod0 = torch.randn(B, 6 * D, generator=g).to(dev)               # outputs accumulate into strided views of a dmod-like buffer
    outs = []
    for o in (nat, ref):
        dmod, dbias = dmod0.clone(), torch.ones(D, device=dev)
        dm = o.gate_bwd(dx, m, gate, rpb, dmod[:, 2 * D:3 * D], dbias)
        outs.append((dm, dmod, dbias))
    for got, want, name in zip(outs[0], outs[1], ("dm", "dgate", "dbias")):
        _close(got, want, EPS[dt] if name == "dm" else 2e-5, "gate_bwd " + name)
    u = (torch.randn(T, 4 * D, generator=g) * 2).to(dev).to(dt)
    da = torch.randn(T, 4 * D, generator=g).to(dev).to(dt)
    db, db_r = torch.zeros(4 * D, device=dev), torch.zeros(4 * D, device=dev)
    du = nat.gelu_bwd(da, u, db)
    du_r = ref.gelu_bwd(da, u, db_r)
    _close(du, du_r, EPS[dt], "gelu_bwd du")
    _close(db, db_r, 3e-3, "gelu_bwd dbias")      # sum of fp32 values vs sum of the same values: order only
    x = (torch.randn(T, D, generator=g) * 3 + 1).to(dev)
    dh = torch.randn(T, D, generator=g).to(dev).to(dt)
    acc0 = torch.randn(T, D, generator=g).to(dev)
    acc_n, acc_r = acc0.clone(), acc0.clone()
    dm_n, dm_r = dmod0.clone(), dmod0.clone()
    nat.ln_modulate_bwd(dh, x, shift, scale, rpb, acc_n, dm_n[:, 0:D], dm_n[:, D:2 * D])
    ref.ln_modulate_bwd(dh, x, shift, scale, rpb, acc_r, dm_r[:, 0:D], dm_r[:, D:2 * D])
    _close(acc_n, acc_r, 2e-5, "ln_modulate_bwd dx")
    _close(dm_n, dm_r, 2e-5, "ln_modulate_bwd dshift / dscale")


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("geom", [(2, 8, 64, 2, 64), (1, 16, 256, 8, 72), (2, 16, 128, 3, 72), (1, 8, 1024, 2, 72)])
@pytest.mark.parametrize("temporal", [False, True])
def test_attention_backward(dev, dt, geom, temporal):
    """dqkv of softmax(QK^T hd^-1/2)V (latte.py:48-77) for spatial sequences (tensor cores, scores recomputed) and temporal
    sequences (F <= 16), at head_dim 64 and 72; the forward output comes from the sampling path's attention kernel."""
    nat, ref = _ops(dt)
    B, Fr, N, H, hd = geom
    g = torch.Generator().manual_seed(B * 1000 + N + hd)
    T, D = B * Fr * N, H * hd
    qkv = torch.randn(T, 3 * D, generator=g).to(dev).to(dt)
    do = torch.randn(T, D, generator=g).to(dev).to(dt)
    o = nat.attention(qkv, B, Fr, N, H, temporal)
    got = nat.attention_bwd(qkv, o, do, B, Fr, N, H, temporal)
    want = ref.attention_bwd(qkv, o, do, B, Fr, N, H, temporal)
    for k, name in enumerate(("dq", "dk", "dv")):
        e = _rel(got[:, k * D:(k + 1) * D], want[:, k * D:(k + 1) * D])
        assert e < 3 * EPS[dt], f"{name}: relative Frobenius error {e:.3e}"


@pytest.mark.parametrize("dt", DTS)
def test_adaln_gradients(dev, dt):
    nat, ref = _ops(dt)
    g = torch.Generator().manual_seed(6)
    B, D, NA = 5, 384, 4 * 6 * 384 + 2 * 384
    dmod = torch.randn(B, NA, generator=g).to(dev)
    sc = torch.randn(B, D, generator=g).to(dev).to(dt)
    w = (torch.randn(NA, D, generator=g) / 20).to(dev).to(dt)
    _close(nat.ada_outer(dmod, sc), ref.ada_outer(dmod, sc), 2e-5, "ada_outer")
    _close(nat.ada_dsc(dmod, w), ref.ada_dsc(dmod, w), 2e-5, "ada_dsc")


@pytest.mark.parametrize("dt", DTS)
def test_fused_gelu_epilogues(dev, dt):
    """Training-mode fc1: u and gelu(u) from one epilogue."""
    nat, ref = _ops(dt)
    g = torch.Generator().manual_seed(12)
    a = torch.randn(2048, 384, generator=g).to(dev).to(dt)
    w = (torch.randn(1536, 384, generator=g) / 384 ** 0.5).to(dev).to(dt)
    b = torch.randn(1536, generator=g).to(dev)
    u, act = nat.linear_gelu_both(a, w, b)
    u_r, act_r = ref.linear_gelu_both(a, w, b)
    _close(u, u_r, EPS[dt], "fc1 pre-activation")
    _close(act, ref.gelu(u), EPS[dt], "gelu of the kernel's own u")
    _close(act, act_r, 2 * EPS[dt], "gelu(u)")


def test_fused_training_loss_matches_torch_expressions(dev):
    """`b200_training_loss` (values and gradient w.r.t. the model output) against the module's own elementwise torch version, with
    a t == 0 sample (decoder NLL branch) and x_0 values outside [-0.999, 0.999] (the clamped CDF branches)."""
    from latte_b200.diffusion import create_diffusion
    d = create_diffusion(timestep_respacing="")
    g = torch.Generator().manual_seed(13)
    B, Fr, Cc, H = 4, 3, 4, 8
    x0 = (torch.randn(B, Fr, Cc, H, H, generator=g) * 0.8).to(dev)
    x0[0, 0, 0, 0, :4] = torch.tensor([-1.0, 1.0, -0.9995, 0.9995], device=dev)
    noise = torch.randn(B, Fr, Cc, H, H, generator=g).to(dev)
    t = torch.tensor([0, 1, 500, 999], device=dev)
    mo0 = torch.randn(B, Fr, 2 * Cc, H, H, generator=g).to(dev)
    outs = []
    for fused in (True, False):
        mo = mo0.clone().requires_grad_(True)
        model = lambda x, tt, **kw: mo          # noqa: E731
        terms = d.training_losses(model, x0, t, None, noise) if fused else d._training_losses_torch(model, x0, t, None, noise)
        w = torch.tensor([1.0, 0.5, 2.0, 1.5], device=dev)
        ((terms["loss"] * w).sum() + 0.3 * terms["mse"].sum() + 0.7 * (terms["vb"] * w).sum()).backward()
        outs.append((terms, mo.grad.clone()))
    (tf, gf), (tt_, gt) = outs
    for k in ("loss", "mse", "vb"):
        assert torch.allclose(tf[k], tt_[k], rtol=2e-4, atol=1e-6), (k, tf[k], tt_[k])
    assert torch.allclose(gf, gt, rtol=2e-3, atol=1e-7), (gf - gt).abs().max()


def _golden_model(golden_dir, dev):
    from latte_b200 import Latte
    from oracle import latte_oracle as O
    g = np.load(os.path.join(golden_dir, "train_tiny64.npz"))
    cfg = O.make_config("Latte-tiny64/2", input_size=16, num_frames=8)
    m = Latte(input_size=16, hidden_size=128, depth=2, num_heads=2, num_frames=8, num_classes=101, extras=2)
    m.load_state_dict(O.make_weights(cfg, 21), strict=True)
    return g, m.to(dev)


@pytest.mark.parametrize("dt", DTS)
def test_training_step_matches_reference_gradients(dev, golden_dir, dt):
    """model.train() + diffusion.training_losses + loss.backward() -- the reference's train.py:206-222 -- on the native path."""
    from latte_b200.diffusion import create_diffusion
    g, m = _golden_model(golden_dir, dev)
    m.train()
    m.y_embedder.dropout_prob = 0.0          # the golden was generated without label dropout (no RNG in the comparison)
    m.train_dtype = dt
    d = create_diffusion(timestep_respacing="")
    x0, noise = torch.from_numpy(g["x0"]).to(dev), torch.from_numpy(g["noise"]).to(dev)
    t, y = torch.from_numpy(g["t"]).to(dev), torch.from_numpy(g["y"]).to(dev)
    terms = d.training_losses(m, x0, t, dict(y=y), noise=noise)
    loss = terms["loss"].mean()
    assert abs(loss.item() - float(g["loss"])) < 3 * EPS[dt] * abs(float(g["loss"]))
    loss.backward()
    named = dict(m.named_parameters())
    worst = 0.0
    for k, want in zip([str(n) for n in g["grad_names"]], g["grad_norms"]):
        got = named[k].grad.double().norm().item()
        worst = max(worst, abs(got - want) / want)
        assert abs(got - want) <= 10 * EPS[dt] * want, (k, got, want)
    for key in g.files:
        if key.startswith("grad::"):
            ref = torch.from_numpy(g[key]).to(dev)
            e = _rel(named[key[6:]].grad, ref)
            assert e < 10 * EPS[dt], (key, e)


@pytest.mark.parametrize("dt", DTS)
def test_training_step_xl_head_geometry(dev, dt):
    """head_dim 72, 256 tokens, 16 frames, depth 4 (Latte-tiny72/2): native engine vs the same engine through TorchOps in fp32."""
    from latte_b200 import Latte, training
    from latte_b200.train_ops import NativeOps
    from oracle import latte_oracle as O
    from oracle.train_ops_oracle import TorchOps
    cfg = O.make_config("Latte-tiny72/2", input_size=32, num_frames=16)
    m = Latte(input_size=32, hidden_size=576, depth=4, num_heads=8, num_frames=16, num_classes=101, extras=2)
    m.load_state_dict(O.make_weights(cfg, 5), strict=True)
    m = m.to(dev)
    gen = torch.Generator().manual_seed(9)
    x = torch.randn(2, 16, 4, 32, 32, generator=gen).to(dev)
    t = torch.tensor([3, 700], device=dev)
    y = torch.tensor([4, 101], device=dev)
    dout = torch.randn(2, 16, 8, 32, 32, generator=gen).to(dev)
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


def test_clip_grad_norm_and_update_ema(dev):
    """latte_b200.utils (utils.py:72-125, 190-200 of the reference): one multi-tensor launch each, same numbers as the python loops."""
    from latte_b200 import utils as U
    g = torch.Generator().manual_seed(11)
    shapes = [(1152, 1152), (4608,), (7,), (33, 5), (1153,), (102, 1152), (1, 16, 1152)]
    params = [torch.nn.Parameter(torch.randn(*s, generator=g).to(dev)) for s in shapes]
    for p in params:
        p.grad = torch.randn(p.shape, generator=g).to(dev) * 3
    params.append(torch.nn.Parameter(torch.zeros(5, device=dev)))          # no grad: skipped like the reference does
    want_grads = [p.grad.clone() for p in params[:-1]]
    ref_params = [torch.nn.Parameter(p.detach().clone()) for p in params[:-1]]
    for p, gr in zip(ref_params, want_grads):
        p.grad = gr.clone()
    want_norm = torch.nn.utils.clip_grad_norm_(ref_params, 1.5)
    got_norm = U.clip_grad_norm_(params, 1.5)
    assert got_norm.dim() == 0 and abs(got_norm.item() - want_norm.item()) < 1e-5 * want_norm.item()
    for p, r in zip(params[:-1], ref_params):
        assert torch.allclose(p.grad, r.grad, rtol=1e-5, atol=1e-7)
    before = [p.grad.clone() for p in params[:-1]]
    n2 = U.clip_grad_norm_(params, 1.5, clip_grad=False)                    # train.py:226 -- measure only
    assert abs(n2.item() - 1.5) < 1e-3 and all(torch.equal(a, p.grad) for a, p in zip(before, params[:-1]))
    assert U.clip_grad_norm_(params, 1e9).item() == pytest.approx(n2.item(), rel=1e-6)   # coefficient clamped to 1: unchanged
    assert all(torch.equal(a, p.grad) for a, p in zip(before, params[:-1]))

    net = torch.nn.Sequential(torch.nn.Linear(33, 17), torch.nn.Linear(17, 5)).to(dev)
    import copy
    ema = copy.deepcopy(net)
    with torch.no_grad():
        for p in net.parameters():
            p.add_(torch.randn(p.shape, generator=g).to(dev))
    want = [e.detach() * 0.99 + p.detach() * 0.01 for e, p in zip(ema.parameters(), net.parameters())]
    U.update_ema(ema, net, decay=0.99)
    for e, w in zip(ema.parameters(), want):
        assert torch.allclose(e, w, rtol=1e-6, atol=1e-7)
    U.update_ema(ema, net, decay=0)                                         # train.py:163 -- initialise the EMA with the weights
    for e, p in zip(ema.parameters(), net.parameters()):
        assert torch.equal(e, p)


def test_train_loop_like_train_py(dev):
    """train.py:206-235 in miniature on the native path: training_losses under bf16 autocast, backward, clip, AdamW, EMA; the
    loss on a fixed batch must go down and everything stays finite."""
    import copy
    from latte_b200 import Latte, utils as U
    from latte_b200.diffusion import create_diffusion
    torch.manual_seed(0)
    m = Latte(input_size=16, hidden_size=128, depth=2, num_heads=2, num_frames=8, num_classes=11, extras=2).to(dev)
    ema = copy.deepcopy(m)
    U.requires_grad(ema, False)
    U.update_ema(ema, m, decay=0)
    m.train()
    opt = torch.optim.AdamW(m.parameters(), lr=2e-3, weight_decay=0)
    d = create_diffusion(timestep_respacing="")
    g = torch.Generator().manual_seed(3)
    x = torch.randn(4, 8, 4, 16, 16, generator=g).to(dev)
    y = torch.randint(0, 11, (4,), generator=g).to(dev)
    t = torch.tensor([50, 300, 600, 900], device=dev)
    noise = torch.randn(x.shape, generator=g).to(dev)
    losses = []
    for _ in range(12):
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = d.training_losses(m, x, t, dict(y=y), noise=noise)["mse"].mean()
        loss.backward()
        norm = U.clip_grad_norm_(m.parameters(), 1.0)
        opt.step()
        opt.zero_grad()
        U.update_ema(ema, m)
        assert torch.isfinite(loss) and torch.isfinite(norm)
        losses.append(loss.item())
    assert losses[-1] < 0.9 * losses[0], losses
    assert all(torch.isfinite(p).all() for p in ema.parameters())
