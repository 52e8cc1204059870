"""GPU: gradient checkpointing of the native training step (`enable_gradient_checkpointing()`), against the plain step.

* The forward kernels are deterministic, so the output with checkpointing must be bit-identical to the plain output.
* The bias, gate and adaLN reductions accumulate with float atomics, so two plain runs need not agree bit for bit on those
  gradients, or on anything computed from them.  The weight gradients of the GEMMs, which no atomic feeds, must be
  bit-identical across two plain runs and with checkpointing.  Every other gradient must differ from the first plain run by
  no more than the two plain runs differ from each other, or by a floor: 1e-5 for fp32 gradients (fp32 sums of the same
  terms in another order differ by a few ulps of 1.2e-7 per partial sum, far below it), and 2^-10 for fp16 gradients (one
  rounding step of the gradient's own type in every element), times the tensor's norm.  On an H100 the largest difference
  seen was 2.4 % of its floor.  (A rule that required bit-identity for whatever happened to agree across two plain runs
  failed on bias gradients that agreed there by chance.)
* Peak memory above the pre-step level, on a deep, narrow LatteT2V where activations dominate, is bounded by
  NB*T*D*4 (one fp32 input per block) + one block's activations (46*T*D bytes) + the once-per-step state, plus a stated slack,
  and is at most a third of the plain step's.
* A full checkpointed step with AdamW, clip_grad_norm_ and update_ema leaves everything finite."""
import copy

import pytest
import torch

from oracle import latte_oracle as O
from oracle import t2v_oracle as T

pytestmark = pytest.mark.gpu

PRECISIONS = ["bf16_autocast", "fp16_params"]
FLOOR = {torch.float32: 1e-5, torch.float16: 2.0 ** -10}


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


# ------------------------------------------------------------------------------------------------------------- cases
def _latte_case(name, dev):
    """Latte at F = 16 / 20, LatteIMG with I = 2: (model, step() -> output), seeded weights (every path carries signal)."""
    from latte_b200 import Latte, LatteIMG
    B = 2
    if name == "img_i2":
        F, I = 4, 2
        cfg = O.make_config("Latte-tiny64/2", input_size=16, num_frames=F, class_dropout_prob=0.0)
        m = LatteIMG(input_size=16, hidden_size=128, depth=2, num_heads=2, num_frames=F, num_classes=101, class_dropout_prob=0.0)
    else:
        F, I = int(name[1:]), 0
        cfg = O.make_config("Latte-tiny64/2", input_size=16, num_frames=F, class_dropout_prob=0.0)
        m = Latte(input_size=16, hidden_size=128, depth=2, num_heads=2, num_frames=F, num_classes=101, extras=2,
                  class_dropout_prob=0.0)
    m.load_state_dict(O.make_weights(cfg, 21), strict=True)
    g = torch.Generator().manual_seed(F + I)
    x = torch.randn(B, F + I, 4, 16, 16, generator=g).to(dev)
    t = torch.tensor([120, 870], device=dev)
    y = torch.tensor([3, 57], device=dev)
    yi = torch.tensor([[1, 2], [3, 4]], device=dev)
    m = m.to(dev).train()

    def step(model):
        if I:
            return model(x, t, y=y, y_image=yi, use_image_num=I)
        return model(x, t, y=y)
    return m, step


def _t2v_case(name, dev):
    """LatteT2V with a masked caption (12 of 20 tokens in sample 1) at F = 1 (32^2 latents) and F = 12 (16^2 latents)."""
    from latte_b200 import LatteT2V
    F = int(name[4:])
    cfg = T.T2VConfig(num_attention_heads=2, attention_head_dim=64, num_layers=2, sample_size=32 if F == 1 else 16,
                      video_length=F, caption_channels=256)
    m = LatteT2V(num_attention_heads=2, attention_head_dim=64, num_layers=2, sample_size=cfg.sample_size, video_length=F,
                 caption_channels=256)
    m.load_state_dict(T.make_weights(cfg, 9), strict=True)
    x, t, text = T.make_inputs(cfg, 2, 20, 10)
    mask = torch.ones(2, 20)
    mask[1, 12:] = 0
    x, t, text, mask = x.to(dev), t.to(dev), text.to(dev), mask.to(dev)
    m = m.to(dev).train()

    def step(model):
        return model(x, t, encoder_hidden_states=text, encoder_attention_mask=mask).sample
    return m, step


CASES = ["f16", "f20", "img_i2", "t2v_1", "t2v_12"]


def _run(m, step, precision, ckpt):
    """One forward + backward with a fixed cotangent; (output, {name: gradient})."""
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


def _deterministic(name):
    """Weight gradients of the GEMMs (ordered stream-K, no atomics) whose inputs are themselves atomics-free: every Linear and
    the patch embedding, except the adaLN ones and the embedders, which are fed by the atomic per-sample reductions."""
    return name.endswith(".weight") and not any(s in name for s in ("adaLN_modulation", "adaln_single", "t_embedder",
                                                                     "y_embedder"))


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("case", CASES)
def test_checkpointed_step_matches_plain(dev, case, precision):
    m, step = (_t2v_case if case.startswith("t2v") else _latte_case)(case, dev)
    if precision == "fp16_params":
        m.half()
    o1, g1 = _run(m, step, precision, False)
    o2, g2 = _run(m, step, precision, False)
    oc, gc = _run(m, step, precision, True)
    assert torch.equal(o1, o2) and torch.equal(o1, oc), "forward output differs"
    assert g1.keys() == g2.keys() == gc.keys() and len(gc) > 0
    det = [k for k in g1 if _deterministic(k)]
    for k in det:
        assert torch.equal(g1[k], g2[k]) and torch.equal(gc[k], g1[k]), k
    # the rest come from float-atomic reductions: a coincidence of two plain runs proves nothing, so each is held to the two
    # runs' spread or the floor, relative to its own norm or -- for gradients that are rounding noise in exact arithmetic
    # (LatteT2V's key biases, softmax being shift-invariant) -- to the median gradient norm
    med = torch.tensor([g.double().norm().item() for g in g1.values()]).median().item()
    worst = 0.0
    for k in g1.keys() - set(det):
        diff, spread = (gc[k].double() - g1[k].double()).norm().item(), (g2[k].double() - g1[k].double()).norm().item()
        floor = FLOOR[g1[k].dtype] * max(g1[k].double().norm().item(), med)
        worst = max(worst, diff / floor)
        assert torch.isfinite(gc[k]).all() and diff <= max(spread, floor), (k, diff, spread, floor)
    print(f"{case} {precision}: {len(det)} GEMM weight gradients bit-identical, {len(g1) - len(det)} others within "
          f"{worst:.3g} of their floor")


# ------------------------------------------------------------------------------------------------------------- memory
DEEP = dict(num_attention_heads=2, attention_head_dim=64, num_layers=8, sample_size=32, video_length=16, caption_channels=256)


def _deep(dev):
    """8 layer pairs, D = 128, 16 frames x 32^2 latents (256 tokens per frame), batch 2: activations dominate."""
    from latte_b200 import LatteT2V
    cfg = T.T2VConfig(**DEEP)
    m = LatteT2V(**DEEP)
    m.load_state_dict(T.make_weights(cfg, 3), strict=True)
    x, t, text = T.make_inputs(cfg, 2, 20, 4)
    mask = torch.ones(2, 20, device=dev)
    mask[0, 15:] = 0
    return m.to(dev).train(), x.to(dev), t.to(dev), text.to(dev), mask


def test_checkpointed_peak_memory(dev):
    m, x, t, text, mask = _deep(dev)
    B, NB, D = 2, 2 * DEEP["num_layers"], 128
    Tr = B * DEEP["video_length"] * (DEEP["sample_size"] // 2) ** 2          # token rows, 8192

    def step(ckpt):
        m.gradient_checkpointing = ckpt
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = m(x, t, encoder_hidden_states=text, encoder_attention_mask=mask).sample
        out.backward(torch.ones_like(out))

    for ckpt in (False, True):                       # first calls build the persistent operand copies and workspaces
        step(ckpt)
    inc = {}
    for ckpt in (False, True):
        m.zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated(dev)
        torch.cuda.reset_peak_memory_stats(dev)
        step(ckpt)
        torch.cuda.synchronize()
        inc[ckpt] = torch.cuda.max_memory_allocated(dev) - base
    grads = sum(p.numel() * 4 for p in m.parameters())                     # the fp32 .grad tensors the step creates
    Rp = 64                                                                  # caption rows, padded to 64
    # kept once per step: x_last (fp32) and its LayerNorm (16-bit), the patch operand (64 columns), c / silu(c) / the modulation
    # rows, and the caption operand, its projection (3 x D) and every layer's K/V (16-bit)
    once = (4 + 2) * Tr * D + Tr * 64 * 2 + 2 * B * (NB * 6 + 2) * D * 4 + Rp * (256 + 3 * D + NB * D) * 2
    formula = NB * Tr * D * 4 + 46 * Tr * D + once
    # slack: the backward's own buffers next to one rerun block -- dx (fp32, 4 bytes per token and channel), the widest
    # gradient temporaries (fc2's gradient, its dgrad and the GELU gradient: 2 + 8 + 8), the cross-attention's cast and
    # out-of-place dx (2 + 4), rounded up to 32 -- plus the fp32 parameter gradients and the output with its cotangent
    out_bytes = B * 8 * DEEP["video_length"] * DEEP["sample_size"] ** 2 * 4
    slack = 32 * Tr * D + grads + 2 * out_bytes
    print(f"peak above pre-step level: plain {inc[False] / 2**20:.1f} MiB, checkpointed {inc[True] / 2**20:.1f} MiB, "
          f"formula {formula / 2**20:.1f} MiB + slack {slack / 2**20:.1f} MiB")
    assert inc[True] <= formula + slack, (inc, formula, slack)
    assert inc[True] * 3 <= inc[False], inc


def test_checkpointed_full_step_with_adamw_clip_and_ema(dev):
    from latte_b200 import utils as U
    m, x, t, text, mask = _deep(dev)
    m.enable_gradient_checkpointing()
    ema = copy.deepcopy(m)
    assert ema.is_gradient_checkpointing
    U.requires_grad(ema, False)
    U.update_ema(ema, m, decay=0)
    opt = torch.optim.AdamW(m.parameters(), lr=1e-4, weight_decay=0)
    for _ in range(2):
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = m(x, t, encoder_hidden_states=text, encoder_attention_mask=mask).sample
            loss = (out.float() ** 2).mean()
        loss.backward()
        assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in m.parameters())
        norm = U.clip_grad_norm_(m.parameters(), 1.0)
        opt.step()
        opt.zero_grad(set_to_none=True)
        U.update_ema(ema, m)
        assert torch.isfinite(loss) and torch.isfinite(norm)
    assert all(torch.isfinite(p).all() for p in m.parameters())
    assert all(torch.isfinite(p).all() for p in ema.parameters())
