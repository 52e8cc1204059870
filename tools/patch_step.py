"""Latte-XL at patch 2, 4 and 8 on the GPU: one sampling step and one training step per patch size.

  sampling  forward_with_cfg on a classifier-free-guidance pair (batch 2) of 16 frames x 256 x 256 (32 x 32 latents), fp16
            operands, timed as the module runs by default (CUDA-graph replay); per-class device time from the library's
            event profiler in a separate eager pass.
  training  fp32 parameters under torch.autocast(bfloat16), diffusion.training_losses(...)["loss"].mean().backward() as
            train.py runs it, on a local batch of --train-batch videos of 16 frames x 256 x 256.

Tokens per frame are 256, 64 and 16, so the token-row count T of every GEMM shrinks 4x per patch step (a CFG pair at patch 8
is T = 512 rows).  Random weights (adaLN not zero, so every path carries signal); times do not depend on the values.
Prints one JSON line: per model, sample_ms (median over rounds of the per-round mean, CUDA events), sample_per_class_ms,
sample_launches, train_ms (the same over training steps), and the card's name and power limit, read in the same run.
Usage:  python tools/patch_step.py [--patches 2 4 8] [--steps 20] [--warmup 5] [--rounds 5] [--train-batch 4] [--out DIR]
"""
import argparse
import os
import statistics
import sys

import torch

from harness import card, emit, ms_per_step, profile, require_cuda

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def timed(fn, steps, rounds):
    """Median over rounds of the per-round mean device time, and the rounds."""
    per = ms_per_step(fn, steps, rounds)
    return statistics.median(per), [round(v, 4) for v in per]


def measure(p, args, dev):
    from latte_b200 import Latte_models
    from latte_b200.diffusion import create_diffusion

    torch.manual_seed(p)
    m = Latte_models[f"Latte-XL/{p}"](input_size=32, num_classes=1000, num_frames=16, learn_sigma=True, extras=2).to(dev)
    with torch.no_grad():
        for prm in m.parameters():
            if prm.requires_grad:
                prm.normal_(0.0, 0.02)
    g = torch.Generator(device=dev).manual_seed(p)
    res = {"model": f"Latte-XL/{p}", "tokens_per_frame": (32 // p) ** 2}

    # ---- sampling: a CFG pair
    m.eval()
    x = torch.randn(2, 16, 4, 32, 32, device=dev, generator=g)
    t = torch.tensor([500, 500], device=dev)
    y = torch.tensor([7, 1000], device=dev)
    with torch.no_grad():
        step = lambda: m.forward_with_cfg(x, t, y=y, cfg_scale=4.0)   # noqa: E731
        for _ in range(args.warmup):
            step()
        res["sample_ms"], res["sample_round_ms"] = timed(step, args.steps, args.rounds)
        res["sample_per_class_ms"], res["sample_launches"] = profile(step, args.steps)

    # ---- training: fwd + bwd under bf16 autocast
    m.train()
    d = create_diffusion(timestep_respacing="")
    B = args.train_batch
    x0 = torch.randn(B, 16, 4, 32, 32, device=dev, generator=g)
    tt = torch.randint(0, 1000, (B,), device=dev, generator=g)
    yy = torch.randint(0, 1000, (B,), device=dev, generator=g)

    def train_step():
        m.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = d.training_losses(m, x0, tt, dict(y=yy))["loss"].mean()
        loss.backward()
    for _ in range(max(2, args.warmup // 2)):
        train_step()
    res["train_batch"] = B
    res["train_ms"], res["train_round_ms"] = timed(train_step, max(2, args.steps // 4), args.rounds)
    del m
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--patches", type=int, nargs="+", default=[2, 4, 8])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--train-batch", type=int, default=4)
    ap.add_argument("--out", default=None, help="directory for patch_step.json (nothing is written without it)")
    args = ap.parse_args()
    require_cuda()
    dev = torch.device("cuda:0")
    res = {**card(clock=True), "workload": "Latte-XL, 16 x 256^2, sampling: CFG pair fp16 graph replay; training: bf16 autocast",
           "models": [measure(p, args, dev) for p in args.patches]}
    emit(res, args.out, "patch_step.json")


if __name__ == "__main__":
    main()
