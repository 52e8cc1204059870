"""CPU: gradient checkpointing of the training step (`enable_gradient_checkpointing()` on Latte, LatteIMG and LatteT2V).

With the flag set, the engines (latte_b200/training.py, training_t2v.py) keep each block's input only and rerun the block's
forward in the backward.  Driven through the torch restatements of their ops (oracle/train_ops_oracle.TorchOps,
oracle/train_t2v_ops_oracle.T2VTorchOps), the checkpointed step must
  * match the UNMODIFIED reference's goldens within the bars the plain engine meets on the same fixture;
  * give outputs and parameter gradients bit-identical to the plain step, in fp32 and with bf16 operands (the same ops run on
    the same inputs);
  * hold exactly one fp32 (rows x D) tensor per block plus the once-per-step state after its forward (the memory policy)."""
import copy
import os

import numpy as np
import pytest
import torch

from latte_b200 import Latte, LatteIMG, LatteT2V, training, training_t2v
from latte_b200.diffusion import create_diffusion
from oracle import latte_oracle as O
from oracle import t2v_oracle as T
from oracle.train_ops_oracle import TorchOps
from oracle.train_t2v_ops_oracle import T2VTorchOps

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
T2V_TAGS = ["tiny_b2_l20", "tiny_b2_l20_masked", "hd72_b2_l120_masked", "f1_b2_l20"]


# ------------------------------------------------------------------------------------------------------------- set-ups
def _latte(name):
    """(golden, model, step(model, ops, dtype) -> output): Latte 'f8' / 'f1' / 'f20', LatteIMG 'img_e1' / 'img_e2'."""
    if name.startswith("img"):
        extras, F, I = int(name[-1]), 4, 3
        g = np.load(os.path.join(GOLDEN, f"train_img_tiny64_{name[4:]}.npz"))
        cfg = O.make_config("Latte-tiny64/2", input_size=16, num_frames=F, extras=extras, class_dropout_prob=0.0)
        m = LatteIMG(input_size=16, hidden_size=128, depth=2, num_heads=2, num_frames=F, num_classes=101, extras=extras,
                     class_dropout_prob=0.0)
    else:
        F, I = int(name[1:]), 0
        g = np.load(os.path.join(GOLDEN, "train_tiny64.npz" if F == 8 else f"train_tiny64_f{F}.npz"))
        cfg = O.make_config("Latte-tiny64/2", input_size=16, num_frames=F)
        m = Latte(input_size=16, hidden_size=128, depth=2, num_heads=2, num_frames=F, num_classes=101, extras=2)
    m.load_state_dict(O.make_weights(cfg, 21), strict=True)
    t, y = torch.from_numpy(g["t"]), torch.from_numpy(g["y"])
    yi = torch.from_numpy(g["y_image"]) if I and m.extras == 2 else None

    def step(model, ops, dtype, x):
        if I:
            c = training.frame_conditioning(model, t, y if model.extras == 2 else None, yi, I)
        else:
            c = training.conditioning(model, t, y)
        return training.train_forward(model, ops, dtype, x, c, images=I)
    return g, m, step


def _t2v(tag):
    z = np.load(os.path.join(GOLDEN, f"train_t2v_{tag}.npz"))
    cfg = T.T2VConfig(**eval(str(z["cfg"])))
    x, t, text = T.make_inputs(cfg, int(z["batch"]), int(z["text_len"]), int(z["iseed"]))
    m = LatteT2V(num_attention_heads=cfg.num_attention_heads, attention_head_dim=cfg.attention_head_dim,
                 in_channels=cfg.in_channels, out_channels=cfg.out_channels, num_layers=cfg.num_layers, patch_size=cfg.patch_size,
                 sample_size=cfg.sample_size, caption_channels=cfg.caption_channels, video_length=cfg.video_length)
    m.load_state_dict(T.make_weights(cfg, int(z["wseed"])), strict=True)
    bias = None
    if "mask" in z:
        mask = torch.from_numpy(z["mask"]).float()
        bias = torch.zeros(mask.shape[0], 128)
        bias[:, :mask.shape[1]] = (1.0 - mask) * -10000.0

    def step(model, ops, dtype, x_):
        return training_t2v.train_forward(model, ops, dtype, x_, training_t2v.conditioning(model, t), text, bias)
    return z, m.train(), step, x


def _saved_blocks(out):
    """The engine behind a training output (the autograd node's context) and what it keeps per block."""
    eng = out.grad_fn.engine
    return eng, eng.saved["blocks"]


# ------------------------------------------------------------------------------------------------------------- 1. goldens
@pytest.mark.parametrize("name", ["f8", "f1", "f20", "img_e1", "img_e2"])
def test_checkpointed_latte_matches_reference(name):
    """The bars of tests/test_oracle_train*.py for the same fixtures: loss within 2e-5 (1e-4 with images), every gradient norm
    and every stored full gradient within 1e-4."""
    g, m, step = _latte(name)
    m.train().enable_gradient_checkpointing()
    x0, noise, t = torch.from_numpy(g["x0"]), torch.from_numpy(g["noise"]), torch.from_numpy(g["t"])
    ops = TorchOps(torch.float32)
    seen = []

    def model_fn(x, tt, **kw):
        out = step(m, ops, torch.float32, x)
        seen.append(_saved_blocks(out))
        return out
    terms = create_diffusion(timestep_respacing="").training_losses(model_fn, x0, t, {}, noise=noise)
    eng, blocks = seen[0]
    assert eng.checkpoint and all(isinstance(b, torch.Tensor) for b in blocks)
    loss = terms["loss"].mean()
    tol_loss = 1e-4 if name.startswith("img") else 2e-5
    assert abs(loss.item() - float(g["loss"])) < tol_loss * abs(float(g["loss"]))
    loss.backward()
    named = dict(m.named_parameters())
    names = [str(k) for k in g["grad_names"]]
    assert set(names) == {k for k, p in named.items() if p.grad is not None}
    for k, want in zip(names, g["grad_norms"]):
        got = named[k].grad.double().norm().item()
        assert abs(got - want) <= 1e-4 * want + 1e-9, (k, got, want)
    for key in g.files:
        if key.startswith("grad::"):
            ref = torch.from_numpy(g[key])
            err = (named[key[6:]].grad - ref).abs().max().item()
            assert err <= 1e-4 * ref.abs().max().item() + 1e-8, (key, err)


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


@pytest.mark.parametrize("tag", T2V_TAGS)
def test_checkpointed_t2v_matches_reference(tag):
    """tests/test_oracle_train_t2v.py's fp32 bars: output, gradient norms and stored gradients within 1e-5 relative; the
    gradients that are exactly zero in exact arithmetic (key biases, q / k of a one-frame temporal attention) below 1e-5 of
    the median norm."""
    z, m, step, x = _t2v(tag)
    m.enable_gradient_checkpointing()
    out = step(m, T2VTorchOps(torch.float32), torch.float32, x)
    assert _saved_blocks(out)[0].checkpoint
    (out * torch.randn(out.shape, generator=torch.Generator().manual_seed(int(z["gseed"])))).sum().backward()
    grads = {k: p.grad.numpy() for k, p in m.named_parameters()}

    def sample(key, a):
        if key + "_sample" in z:
            axis, stride = (int(v) for v in z[key + "_sample"])
            sl = [slice(None)] * a.ndim
            sl[axis] = slice(None, None, stride)
            a = a[tuple(sl)]
        return a
    assert _rel(sample("out", out.detach().numpy()), z["out"]) < 1e-5
    names = [str(n) for n in z["grad_names"]]
    assert sorted(names) == sorted(grads)
    frames = m.config.video_length
    zero = np.array([n.endswith("to_k.bias") or (frames == 1 and n.startswith("temporal_") and (".to_q." in n or ".to_k." in n))
                     for n in names])
    got = np.array([np.linalg.norm(grads[n].astype(np.float64)) for n in names])
    want = z["grad_norms"]
    assert np.all(got[zero] < 1e-5 * np.median(want))
    assert (np.abs(got - want)[~zero] / want[~zero]).max() < 1e-5
    for k in (k[6:] for k in z.files if k.startswith("grad::") and not k.endswith("_sample")):
        if frames == 1 and k == "temporal_transformer_blocks.0.attn1.to_q.weight":
            continue
        assert _rel(sample("grad::" + k, grads[k]), z["grad::" + k]) < 1e-5, k


# ------------------------------------------------------------------------------------------------------------- 2. bit-identical
CASES = ["f8", "f20", "img_e2", "t2v:tiny_b2_l20_masked", "t2v:f1_b2_l20"]


def _both_steps(case, dtype):
    """(output, {name: grad}) of the plain and the checkpointed step on the same model, inputs and cotangent."""
    if case.startswith("t2v:"):
        _, m, step, x = _t2v(case[4:])
        ops = T2VTorchOps(dtype)
    else:
        g, m, step = _latte(case)
        m.train()
        x = torch.from_numpy(g["x0"])
        ops = TorchOps(dtype)
    res = []
    for ckpt in (False, True):
        m.zero_grad(set_to_none=True)
        m.gradient_checkpointing = ckpt
        out = step(m, ops, dtype, x)
        (out * torch.randn(out.shape, generator=torch.Generator().manual_seed(5))).sum().backward()
        res.append((out.detach(), {k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None}))
    return res


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("case", CASES)
def test_checkpointed_step_is_bit_identical_to_plain(case, dtype):
    (o0, g0), (o1, g1) = _both_steps(case, dtype)
    assert torch.equal(o0, o1)
    assert g0.keys() == g1.keys() and len(g0) > 0
    for k in g0:
        assert torch.equal(g0[k], g1[k]), k


# ------------------------------------------------------------------------------------------------------------- 3. memory policy
def _tensors(obj):
    """Every tensor in a nest of lists / tuples (a plain block keeps a list, LatteT2V's cross-attention a tuple or None)."""
    if isinstance(obj, torch.Tensor):
        return [obj]
    return [t for o in (obj or ()) for t in _tensors(o)]


def _held_bytes(tensors):
    """Bytes of the distinct storages behind `tensors`."""
    seen = {}
    for t in tensors:
        s = t.untyped_storage()
        seen[s.data_ptr()] = s.nbytes()
    return sum(seen.values())


@pytest.mark.parametrize("case", ["f8", "img_e2", "t2v:tiny_b2_l20_masked"])
def test_checkpointed_forward_keeps_one_fp32_row_block_per_block(case):
    """After a checkpointed forward the engine holds exactly: one contiguous fp32 (rows x D) tensor per block -- for LatteIMG
    the full residual stream, image rows included -- plus the state kept once per step (conditioning c, silu(c), the
    modulation rows, the patch operand, the last residual and its LayerNorm, and for LatteT2V the caption operand, its
    projection and the stacked K/V of all layers).  The plain forward keeps several times more."""
    dtype = torch.bfloat16
    held = {}
    for ckpt in (False, True):
        if case.startswith("t2v:"):
            _, m, step, x = _t2v(case[4:])
            ops, once = T2VTorchOps(dtype), {"c", "sc", "mod", "xp", "x_last", "hf", "text16", "cu", "ca", "txt", "kv"}
            nb, D = 2 * m.config.num_layers, m.inner_dim
        else:
            g, m, step = _latte(case)
            x = torch.from_numpy(g["x0"])
            ops, once = TorchOps(dtype), {"c", "sc", "mod", "xp", "x_last", "hf"}
            nb, D = m.depth, m.hidden_size
        m.train().gradient_checkpointing = ckpt
        eng, blocks = _saved_blocks(step(m, ops, dtype, x))
        S = eng.saved
        assert set(S) == once | {"B", "blocks"} and len(blocks) == nb
        rows = S["x_last"].shape[0]
        held[ckpt] = _held_bytes(_tensors(blocks) + [S[k] for k in once])
        if ckpt:
            assert all(b.dtype == torch.float32 and b.shape == (rows, D) and b.is_contiguous() for b in blocks)
            assert len({b.data_ptr() for b in blocks} | {S["x_last"].data_ptr()}) == nb + 1
            assert held[True] == nb * rows * D * 4 + _held_bytes([S[k] for k in once])
    assert held[False] > 3 * held[True]


# ------------------------------------------------------------------------------------------------------------- 4. public surface
def _tiny_models():
    return [Latte(input_size=16, hidden_size=128, depth=2, num_heads=2, num_frames=4, num_classes=11, extras=2),
            LatteIMG(input_size=16, hidden_size=128, depth=2, num_heads=2, num_frames=4, num_classes=11),
            LatteT2V(num_attention_heads=2, attention_head_dim=64, num_layers=1, sample_size=16, video_length=4,
                     caption_channels=64)]


def test_gradient_checkpointing_api():
    for m in _tiny_models():
        cls = type(m)
        assert cls._supports_gradient_checkpointing is True
        assert m.gradient_checkpointing is False and m.is_gradient_checkpointing is False
        shapes = {k: v.shape for k, v in m.state_dict().items()}
        m.enable_gradient_checkpointing()
        assert m.gradient_checkpointing is True and m.is_gradient_checkpointing is True
        assert {k: v.shape for k, v in m.state_dict().items()} == shapes
        ema = copy.deepcopy(m)                                   # train.py's EMA copy, made after enabling
        assert ema.is_gradient_checkpointing and ema is not m
        with pytest.raises(AttributeError):
            m.is_gradient_checkpointing = False                  # read-only: the methods switch it
        m.disable_gradient_checkpointing()
        assert not m.is_gradient_checkpointing and ema.is_gradient_checkpointing


@pytest.mark.parametrize("case", ["f8", "t2v:tiny_b2_l20"])
def test_checkpointed_backward_is_single_use(case):
    if case.startswith("t2v:"):
        _, m, step, x = _t2v(case[4:])
        ops = T2VTorchOps(torch.float32)
    else:
        g, m, step = _latte(case)
        x, ops = torch.from_numpy(g["x0"]), TorchOps(torch.float32)
    m.enable_gradient_checkpointing()
    out = step(m, ops, torch.float32, x)
    out.sum().backward(retain_graph=True)
    with pytest.raises(RuntimeError, match="backward called twice"):
        out.sum().backward()
