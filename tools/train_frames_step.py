"""Latte-XL/2 training step (forward + backward) at several video lengths on the GPU: fp32 parameters under
torch.autocast(bfloat16), `diffusion.training_losses(...)["loss"].mean().backward()` as train.py runs it, synthetic latents
(input 32 = 256 tokens per frame), seeded weights.  The local batch shrinks as the frame count grows so that every length
trains the same number of tokens per step (default: 4 x 16, 2 x 32, 1 x 64 frames).

Prints one JSON line per frame count:
  ms_per_step           CUDA events around `steps` back-to-back steps (zero_grad + loss + backward), after `warmup` steps
  attn_bwd_ms           device time of the attention backward per step, temporal and spatial blocks, from CUDA events
                        around every `attention_bwd` call of the training backend, in a separate pass
  attn_bwd_share        attn_bwd_ms (both kinds) / ms_per_step
  gpu, power_limit_w    read from nvidia-smi in the same run
Usage:  python tools/train_frames_step.py [--frames 16 32 64] [--steps 5] [--warmup 2]
"""
import argparse
import os
import sys
from types import SimpleNamespace

import torch

from harness import Timed, card, emit, ms_per_step, require_cuda

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BATCH = {16: 4, 32: 2, 64: 1}


def measure(frames, batch, steps, warmup, dev):
    from latte_b200 import Latte_models
    from latte_b200.diffusion import create_diffusion
    torch.manual_seed(0)
    m = Latte_models["Latte-XL/2"](input_size=32, num_classes=101, num_frames=frames, learn_sigma=True, extras=2).to(dev)
    with torch.no_grad():                      # adaLN-Zero leaves the blocks at identity: give every zero weight some values
        for p in m.parameters():
            if p.requires_grad and float(p.abs().max()) == 0.0:
                p.normal_(0, 0.02)
    m.train()
    d = create_diffusion(timestep_respacing="")
    g = torch.Generator().manual_seed(1)
    x = torch.randn(batch, frames, 4, 32, 32, generator=g).to(dev)
    y = torch.randint(0, 101, (batch,), generator=g).to(dev)
    t = torch.randint(0, 1000, (batch,), generator=g).to(dev)

    def step():
        m.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = d.training_losses(m, x, t, dict(y=y))["loss"].mean()
        loss.backward()

    for _ in range(warmup):
        step()
    [ms] = ms_per_step(step, steps)

    ops = m._train_backend[torch.bfloat16]     # the backend object the warm-up steps created
    # Timed brackets every call of one attribute: route temporal and spatial calls to an attribute each, each timed apart
    kinds = SimpleNamespace(temporal=ops.attention_bwd, spatial=ops.attention_bwd)
    timers = [Timed(kinds, "temporal"), Timed(kinds, "spatial")]
    ops.attention_bwd = lambda qkv, o, do, B, Fr, N, H, temporal: \
        (kinds.temporal if temporal else kinds.spatial)(qkv, o, do, B, Fr, N, H, temporal)
    for _ in range(steps):
        step()
    torch.cuda.synchronize()
    del ops.attention_bwd
    tmp, spa = (tm.ms() / steps for tm in timers)
    peak = torch.cuda.max_memory_allocated(dev) / 2 ** 30
    del m
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats(dev)
    return {"workload": f"Latte-XL/2 training step, {batch} x {frames} frames x 256 tokens, bf16 autocast",
            "frames": frames, "local_batch": batch, "steps": steps, "warmup": warmup, "ms_per_step": ms,
            "attn_bwd_ms": {"temporal": tmp, "spatial": spa}, "attn_bwd_share": (tmp + spa) / ms, "peak_mem_gib": peak}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, nargs="+", default=[16, 32, 64])
    ap.add_argument("--batch", type=int, default=None, help="local batch for every frame count (default: 64 frames per step)")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    require_cuda()
    dev = torch.device("cuda", 0)
    info = card()
    for f in args.frames:
        batch = args.batch or BATCH.get(f, max(1, 64 // f))
        res = measure(f, batch, args.steps, max(args.warmup, 1), dev)
        res.update(info)
        emit(res)


if __name__ == "__main__":
    main()
