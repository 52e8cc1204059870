"""LatteT2V (Latte-1 geometry: 28 layer pairs, 16 heads x 72, caption 4096) training forward + backward on the GPU: fp32
parameters under torch.autocast(bfloat16), seeded weights, synthetic latents and a 120-token prompt (40 tokens valid),
loss = mean(out^2).  Three shapes: 16 x 256^2 x batch 4, 16 x 512^2 x batch 1, 1 x 512^2 x batch 8 (text-to-image).

Prints one JSON line per shape:
  ms_per_step        CUDA events around `steps` back-to-back steps (zero_grad + forward + loss + backward), after `warmup` steps
  xattn_bwd_ms       device time per step of the 28 cross-attention backward calls, CUDA events around them, separate pass
  peak_mem_gib       torch.cuda.max_memory_allocated over the measured steps
  gpu, power_limit_w read from nvidia-smi in the same run
Usage:  python tools/train_t2v_step.py [--steps 3] [--warmup 1]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from train_img_step import _Timed, card  # noqa: E402

SHAPES = [(16, 32, 4), (16, 64, 1), (1, 64, 8)]      # (frames, latent size, batch)


def measure(frames, size, batch, steps, warmup, dev):
    from latte_b200 import LatteT2V
    torch.manual_seed(0)
    m = LatteT2V(video_length=frames, sample_size=size).to(dev).train()
    g = torch.Generator().manual_seed(1)
    x = torch.randn(batch, 4, frames, size, size, generator=g).to(dev)
    t = torch.randint(0, 1000, (batch,), generator=g).to(dev)
    text = (torch.randn(batch, 120, 4096, generator=g) * 0.5).to(dev)
    mask = torch.zeros(batch, 120, device=dev)
    mask[:, :40] = 1

    def step():
        m.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = m(x, t, encoder_hidden_states=text, encoder_attention_mask=mask).sample
            loss = (out.float() ** 2).mean()
        loss.backward()

    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    peak = torch.cuda.max_memory_allocated(dev) / 2 ** 30
    ops = m._train_backend[torch.bfloat16]
    timer = _Timed(ops, "cross_attention_bwd")
    for _ in range(steps):
        step()
    torch.cuda.synchronize()
    timer.restore()
    res = {"workload": f"LatteT2V (Latte-1) training step, {batch} x {frames} frames x {size * 8}^2, L 120, bf16 autocast",
           "batch": batch, "frames": frames, "latent": size, "steps": steps, "warmup": warmup, "ms_per_step": ms,
           "xattn_bwd_ms": timer.ms() / steps, "peak_mem_gib": peak}
    del m, ops
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "train_t2v_step.py measures on a CUDA device"
    dev = torch.device("cuda", 0)
    info = card()
    for frames, size, batch in SHAPES:
        res = measure(frames, size, batch, args.steps, max(args.warmup, 1), dev)
        res.update(info)
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
