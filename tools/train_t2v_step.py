"""LatteT2V (Latte-1 geometry: 28 layer pairs, 16 heads x 72, caption 4096) training forward + backward on the GPU: fp32
parameters under torch.autocast(bfloat16), seeded weights, synthetic latents and a 120-token prompt (40 tokens valid),
loss = mean(out^2).  Three shapes: 16 x 256^2 x batch 4, 16 x 512^2 x batch 1, 1 x 512^2 x batch 8 (text-to-image).
With --images I, video + image joint training (use_image_num = I, one caption per image, each with its own 3-D mask row) in
the same run: 2 x (16 + I) x 256^2 plain and 1 x (16 + I) x 512^2 with gradient checkpointing, each next to the same shape
without images (2 x 16 x 256^2 plain, 1 x 16 x 512^2 checkpointed).

Prints one JSON line per shape:
  ms_per_step        CUDA events around `steps` back-to-back steps (zero_grad + forward + loss + backward), after `warmup` steps
  xattn_bwd_ms       device time per step of the 28 cross-attention backward calls, CUDA events around them, separate pass
  peak_mem_gib       torch.cuda.max_memory_allocated over the measured steps
  gpu, power_limit_w read from nvidia-smi in the same run
Usage:  python tools/train_t2v_step.py [--steps 3] [--warmup 1] [--images 8]
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
IMAGE_SHAPES = [(16, 32, 2, False), (16, 64, 1, True)]  # (frames, latent size, batch, gradient checkpointing), with and without images


def measure(frames, size, batch, steps, warmup, dev, images=0, checkpoint=False):
    from latte_b200 import LatteT2V
    torch.manual_seed(0)
    m = LatteT2V(video_length=frames, sample_size=size).to(dev).train()
    m.gradient_checkpointing = checkpoint
    g = torch.Generator().manual_seed(1)
    x = torch.randn(batch, 4, frames + images, size, size, generator=g).to(dev)
    t = torch.randint(0, 1000, (batch,), generator=g).to(dev)
    caps = (1 + images,) if images else ()
    text = (torch.randn(batch, *caps, 120, 4096, generator=g) * 0.5).to(dev)
    mask = torch.zeros(batch, *caps, 120, device=dev)
    mask[..., :40] = 1

    def step():
        m.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = m(x, t, encoder_hidden_states=text, encoder_attention_mask=mask, use_image_num=images).sample
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
    shape = f"{frames} + {images}" if images else f"{frames}"
    res = {"workload": f"LatteT2V (Latte-1) training step, {batch} x ({shape}) frames x {size * 8}^2, L 120, bf16 autocast"
                       + (", gradient checkpointing" if checkpoint else ""),
           "batch": batch, "frames": frames, "images": images, "latent": size, "checkpoint": checkpoint, "steps": steps,
           "warmup": warmup, "ms_per_step": ms, "xattn_bwd_ms": timer.ms() / steps, "peak_mem_gib": peak}
    del m, ops
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--images", type=int, default=0, help="also time video + image joint training with this many images")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "train_t2v_step.py measures on a CUDA device"
    dev = torch.device("cuda", 0)
    info = card()
    runs = [(frames, size, batch, 0, False) for frames, size, batch in SHAPES]
    if args.images:
        runs += [(frames, size, batch, images, ckpt) for frames, size, batch, ckpt in IMAGE_SHAPES for images in (0, args.images)]
    for frames, size, batch, images, ckpt in runs:
        res = measure(frames, size, batch, args.steps, max(args.warmup, 1), dev, images, ckpt)
        res.update(info)
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
