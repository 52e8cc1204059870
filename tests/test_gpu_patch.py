"""GPU: the patch-4 and patch-8 Latte / LatteIMG models on the native path.

  * The new kernel paths against fp64, element by element, with the bounds of tests/fp64_bounds.py: the patch embedding at
    K = C*p*p = 64 and 256 (patch_embed_wide_kernel) and the tensor-core head at p*p*C_out = 64, 128, 256 and 512, through a
    Latte whose blocks add exactly 0 (as test_gpu_forward_ops_fp64.test_embedding_and_head does at patch 2); the spatial
    attention backward at N = 4 and 16 tokens per frame (routed to the <= 16-row temporal kernel), with the cases and bounds of
    test_gpu_train_ops_fp64.
  * The whole forward against the reference's goldens (oracle/make_golden_patch.py) and the training step against the
    reference's gradients, at the tolerances of test_gpu_model.py, test_gpu_train.py and test_gpu_train_img.py.
  * For one /4 and one /8 model: CUDA-graph replay and trajectory conditioning bit-identical to eager launches, FP8 within
    test_gpu_fp8.py's tolerance factor, gradient checkpointing equal to the plain step up to the float-atomic reductions
    (test_gpu_train_checkpointing.py's rule).
  * A grid the spatial attention does not take (6 x 6 patches) is refused before anything is launched."""
import ctypes as C
import math

import pytest
import torch

import patch_golden as PG
from fp64_bounds import A, B, DTS, SUB, U16, U32, Checker, report_worst, sqfloor  # noqa: E402
from oracle import latte_oracle as O

pytestmark = pytest.mark.gpu

EPS = {torch.float16: 1e-3, torch.bfloat16: 8e-3}
FP8_TOL_FACTOR = 6.0          # tests/test_gpu_fp8.py
_WORST = {}


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    report_worst(_WORST)


def _golden_net(golden_dir, fname, dev):
    """(golden, config, eval-mode Latte on dev, (x, t, y) on dev) of a forward golden."""
    from latte_b200 import Latte
    g, cfg = PG.load(golden_dir, fname)
    batch, wseed, iseed = PG.seeds(g)
    net = PG.build(Latte, cfg)
    net.load_state_dict(O.make_weights(cfg, wseed), strict=True)
    x, t, y = O.make_inputs(cfg, batch, iseed)
    return g, cfg, net.to(dev).eval(), (x.to(dev), t.to(dev), y.to(dev) if cfg.extras == 2 else None)


# ------------------------------------------------------------------------------------------------ kernels against fp64
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("D,heads", [(384, 6), (1152, 16)])
@pytest.mark.parametrize("p", [4, 8])
@pytest.mark.parametrize("learn_sigma", [True, False], ids=["sigma", "nosigma"])
def test_embedding_and_head(dev, dt, D, heads, p, learn_sigma):
    """A depth-2 Latte at input 32 whose gate_msa / gate_mlp adaLN rows are zero, so the output is patch_embed + pos_embed
    (K = 64 or 256) -> + temp_embed -> final LayerNorm + modulate -> the tensor-core head (n_out = 64 .. 512) -> unpatchify,
    against the oracle in fp64 on the shift / scale rows and the 16-bit head weights the kernels read.  The bound terms are
    those of test_gpu_forward_ops_fp64.test_embedding_and_head."""
    from latte_b200 import Latte
    chk = Checker(dt, _WORST)
    Bb, Fr, S, depth = 2, 4, 32, 2
    cfg = O.LatteConfig(input_size=S, patch_size=p, hidden_size=D, depth=depth, num_heads=heads, num_frames=Fr,
                        num_classes=10, learn_sigma=learn_sigma, extras=2)
    sd = O.make_weights(cfg, D + p + learn_sigma)
    for i in range(depth):               # gate_msa / gate_mlp rows: each block is the identity on x
        for c in (2, 5):
            sd[f"blocks.{i}.adaLN_modulation.1.weight"][c * D:(c + 1) * D] = 0
            sd[f"blocks.{i}.adaLN_modulation.1.bias"][c * D:(c + 1) * D] = 0
    net = PG.build(Latte, cfg)
    net.load_state_dict(sd, strict=True)
    net = net.to(dev).eval()
    net.compute_dtype = dt
    sd = {k: v.to(dev) for k, v in sd.items()}
    C_ = cfg.in_channels
    g = torch.Generator(device=dev).manual_seed(D + p)
    x = torch.randn(Bb, Fr, C_, S, S, device=dev, generator=g)
    t = torch.tensor([999, 0], device=dev)
    y = torch.tensor([10, 4], device=dev)
    with torch.no_grad():
        got = net(x, t, y=y)
    mod = net.precompute_conditioning(t[None], y)[0].double()
    _, _, T, _ = net._pack()
    net.clear_conditioning()
    N, K = cfg.num_patches, C_ * p * p
    mf = mod[:, depth * 6 * D:]
    shift, scale = mf[:, :D].repeat_interleave(Fr, 0)[:, None], mf[:, D:].repeat_interleave(Fr, 0)[:, None]
    tc = sd["temp_embed"].double()[0].repeat(Bb, 1)[:, None]
    sd64 = {k: v.double() for k, v in sd.items()}
    x64 = x.double()
    h = O.patch_embed(sd64, cfg, x64, torch.float64) + tc
    xp = x64.reshape(Bb * Fr, C_, S // p, p, S // p, p).permute(0, 2, 4, 1, 3, 5).reshape(Bb * Fr, N, K)
    wp = sd64["x_embedder.proj.weight"].reshape(D, K)
    e_x = U32 * math.sqrt(K + 2) * (xp.abs() @ wp.abs().t() + sd64["x_embedder.proj.bias"].abs() + sd64["pos_embed"].abs() + tc.abs())
    mean = h.mean(-1, keepdim=True)
    rstd = (((h - mean) ** 2).mean(-1, keepdim=True) + 1e-6).rsqrt()
    xh = (h - mean) * rstd
    e_xh = rstd * (e_x + e_x.mean(-1, keepdim=True) + xh.abs() * (xh.abs() * e_x).mean(-1, keepdim=True)) + \
        U32 * (math.sqrt(D) * (rstd * h.abs().mean(-1, keepdim=True) + xh.abs()) + 3 * xh.abs())
    yv = xh * (1 + scale) + shift
    c1 = (1 + scale).abs()
    e_y = c1 * e_xh + U32 * (2 * xh.abs() * c1 + shift.abs()) + U16[dt] * yv.abs()     # + the 16-bit head operand
    wf = T["final_w16"].double()
    bf = sd64["final_layer.linear.bias"]
    out = yv @ wf.t() + bf
    e_o = e_y @ wf.abs().t() + U32 * math.sqrt(D) * (yv.abs() @ wf.abs().t() + bf.abs())
    bnd = A * U32 * out.abs() + B * e_o
    if SUB[dt]:
        bnd = bnd + sqfloor(yv, wf.t(), SUB[dt])
    unp = lambda z: O.unpatchify(cfg, z).reshape(Bb, Fr, cfg.out_channels, S, S)     # noqa: E731
    ref, bnd = unp(out), unp(bnd)
    n_out = p * p * cfg.out_channels
    chk.add(f"embedding K={K} + head n_out={n_out}", f"D={D}", got, ref, bnd,
            lambda i: f"sample {i[0]}, frame {i[1]}, channel {i[2]}, pixel ({i[3]}, {i[4]})")
    chk.done()
    wrong = got.reshape(Bb, Fr, cfg.out_channels, S // p, p, S // p, p).transpose(4, 6).reshape(got.shape)
    m = Checker(dt)
    m.add("unpatchify with the patch transposed", "wrong result", wrong, ref, bnd, str)
    assert m.bad, "the bound accepts a transposed patch"


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("H,hd", [(16, 72), (6, 64)])
@pytest.mark.parametrize("N,Bf", [(4, (2, 8)), (16, (2, 8))])
def test_attention_bwd_spatial_short(dev, dt, H, hd, N, Bf):
    """Spatial sequences of 4 and 16 tokens (patch 8 at 256^2 and the small grids) through the <= 16-row kernel."""
    from test_gpu_train_ops_fp64 import _attention_case
    _attention_case(dev, dt, Bf[0], Bf[1], N, H, hd, False)


# ------------------------------------------------------------------------------------------------ whole model
@pytest.mark.parametrize("fname", PG.FORWARD)
def test_forward_matches_reference_golden(dev, golden_dir, fname):
    g, cfg, net, (x, t, y) = _golden_net(golden_dir, fname, dev)
    ref = torch.from_numpy(g["out"])
    half = torch.from_numpy(g["out_cfg_half_eps"])
    with torch.no_grad():
        for dt, tol in ((torch.float16, 1e-2), (torch.bfloat16, float(g["ref_bf16_maxabs"]))):
            net.compute_dtype = dt
            out = net(x, t, y=y).cpu()
            assert out.shape == ref.shape
            err = (out - ref).abs().max().item()
            assert err < tol, f"{fname} {dt}: max-abs {err:.3e} >= {tol:.3e}"
            oc = net.forward_with_cfg(x, t, y=y, cfg_scale=7.0).cpu()
            b = out.shape[0]
            assert (oc[: b // 2, :, :4] - half).abs().max().item() < 13 * tol
            assert torch.equal(oc[: b // 2, :, :4], oc[b // 2:, :, :4])


def _train_net(golden_dir, fname, dev):
    from latte_b200 import Latte, LatteIMG
    g, cfg = PG.load(golden_dir, fname)
    images = int(g["images"]) if "images" in g.files else 0
    m = PG.build(LatteIMG if images else Latte, cfg)
    m.load_state_dict(O.make_weights(cfg, int(g["wseed"])), strict=True)
    return g, cfg, images, m.to(dev)


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("fname", PG.TRAIN + [PG.TRAIN_IMG])
def test_training_step_matches_reference_gradients(dev, golden_dir, dt, fname):
    """model.train() + diffusion.training_losses + loss.backward() on the native path (LatteIMG: 3 images per video)."""
    from latte_b200.diffusion import create_diffusion
    g, cfg, images, m = _train_net(golden_dir, fname, dev)
    m.train()
    m.train_dtype = dt
    x0, noise, t = (torch.from_numpy(g[k]).to(dev) for k in ("x0", "noise", "t"))
    if images:
        kw = dict(use_image_num=images)
    else:
        m.y_embedder.dropout_prob = 0.0      # the golden was made without label dropout
        kw = dict(y=torch.from_numpy(g["y"]).to(dev))
    terms = create_diffusion(timestep_respacing="").training_losses(m, x0, t, kw, noise=noise)
    loss = terms["loss"].mean()
    assert abs(loss.item() - float(g["loss"])) < 3 * EPS[dt] * abs(float(g["loss"]))
    loss.backward()
    PG.check_grads(g, dict(m.named_parameters()), 10 * EPS[dt], 10 * EPS[dt], frobenius=True)


def test_img_eval_forward_with_images(dev, golden_dir):
    g, cfg, images, m = _train_net(golden_dir, PG.TRAIN_IMG, dev)
    m.eval()
    m.train_dtype = torch.float16
    x0, t = torch.from_numpy(g["x0"]).to(dev), torch.from_numpy(g["t"]).to(dev)
    with torch.no_grad():
        out = m(x0, t, use_image_num=images)
    ref = torch.from_numpy(g["eval_out"]).to(dev)
    assert out.shape == ref.shape
    assert (out - ref).abs().max().item() < 2e-2 * ref.abs().max().item()


# ------------------------------------------------------------------------------------------------ one /4 and one /8 model
PAIR = ["patch_tiny72_4_b2.npz", "patch_tiny72_8_b2.npz"]


@pytest.mark.parametrize("fname", PAIR)
def test_graph_and_trajectory_are_bit_identical(dev, golden_dir, fname):
    _, _, net, (x, t, y) = _golden_net(golden_dir, fname, dev)
    with torch.no_grad():
        net.use_cuda_graphs = False
        eager = net.forward_with_cfg(x, t, y=y, cfg_scale=4.0)
        plain = net(x, t, y=y)
        net.use_cuda_graphs = True
        outs = [net.forward_with_cfg(x, t, y=y, cfg_scale=4.0) for _ in range(3)]      # eager, capture, replay
        assert net._graphs and all(st["graph"] is not None for st in net._graphs.values())
        net.precompute_conditioning(t.view(1, -1), y)
        traj = net.forward_with_cfg(x, t, y=y, cfg_scale=4.0, trajectory_step=0)
        traj_plain = net(x, t, y=y, trajectory_step=0)
        net.clear_conditioning()
    for o in outs + [traj]:
        assert torch.equal(o, eager)
    assert torch.equal(traj_plain, plain)


@pytest.mark.parametrize("fname", PAIR)
def test_fp8_forward_matches_golden(dev, golden_dir, fname):
    g, _, net, (x, t, y) = _golden_net(golden_dir, fname, dev)
    ref = torch.from_numpy(g["out"])
    tol = FP8_TOL_FACTOR * float(g["ref_bf16_maxabs"])
    net.use_fp8 = True
    with torch.no_grad():
        for dt in DTS:
            net.compute_dtype = dt
            err = (net(x, t, y=y).cpu() - ref).abs().max().item()
            assert err < tol, f"{fname} fp8 + {dt}: max-abs {err:.3e} >= {tol:.3e}"


@pytest.mark.parametrize("precision", ["bf16_autocast", "fp16_params"])
@pytest.mark.parametrize("fname", ["patch_train_tiny64_4.npz", "patch_train_tiny64_8.npz"])
def test_checkpointed_step_matches_plain(dev, golden_dir, fname, precision):
    from test_gpu_train_checkpointing import FLOOR, _deterministic, _run
    g, cfg, _, m = _train_net(golden_dir, fname, dev)
    m.train()
    m.y_embedder.dropout_prob = 0.0
    if precision == "fp16_params":
        m.half()
    x0, t, y = (torch.from_numpy(g[k]).to(dev) for k in ("x0", "t", "y"))

    def step(model):
        return model(x0, t, y=y)
    o1, g1 = _run(m, step, precision, False)
    o2, g2 = _run(m, step, precision, False)
    oc, gc = _run(m, step, precision, True)
    assert torch.equal(o1, o2) and torch.equal(o1, oc), "forward output differs"
    assert g1.keys() == g2.keys() == gc.keys() and len(gc) > 0
    det = [k for k in g1 if _deterministic(k)]
    for k in det:
        assert torch.equal(g1[k], g2[k]) and torch.equal(gc[k], g1[k]), k
    med = torch.tensor([v.double().norm().item() for v in g1.values()]).median().item()
    for k in g1.keys() - set(det):
        diff, spread = (gc[k].double() - g1[k].double()).norm().item(), (g2[k].double() - g1[k].double()).norm().item()
        floor = FLOOR[g1[k].dtype] * max(g1[k].double().norm().item(), med)
        assert torch.isfinite(gc[k]).all() and diff <= max(spread, floor), (k, diff, spread, floor)


def test_unsupported_grid_is_refused_before_any_launch(dev):
    """Input 24 at patch 4 is 6 x 6 = 36 tokens per frame, which the spatial attention does not take: the module raises before
    launching, and the C ABI returns B200_ERR_UNSUPPORTED without touching its output."""
    from latte_b200 import Latte, _lib
    kw = dict(hidden_size=128, depth=2, num_heads=2, num_frames=2, num_classes=10, patch_size=4)
    bad = Latte(input_size=24, **kw).to(dev).eval()
    x = torch.randn(2, 2, 4, 24, 24, device=dev)
    t = torch.tensor([1, 2], device=dev)
    y = torch.tensor([1, 2], device=dev)
    with torch.no_grad(), pytest.raises(RuntimeError, match="6 x 6 patches per frame"):
        bad(x, t, y=y)
    # the same call through the ABI with a valid packing and a workspace that would fit
    good = Latte(input_size=32, **kw).to(dev).eval()
    shape, w, _, _ = good._pack()
    lib = _lib.load()
    need = lib.b200_latte_workspace_bytes(C.byref(shape), 2)
    ws = torch.empty(need + 1024, dtype=torch.uint8, device=dev)
    base = (ws.data_ptr() + 1023) // 1024 * 1024
    shape.input_size = 24
    out = torch.zeros(2, 2, 8, 24, 24, device=dev)
    rc = lib.b200_latte_forward(C.byref(shape), C.byref(w), x.data_ptr(), t.data_ptr(), y.data_ptr(), 2, 0, 0.0,
                                out.data_ptr(), base, need, torch.cuda.current_stream(dev).cuda_stream)
    torch.cuda.synchronize()
    assert _lib.ERR_NAMES.get(rc) == "UNSUPPORTED" and "6 x 6 patches per frame" in _lib.last_error()
    assert not out.any(), "a rejected call launched"
