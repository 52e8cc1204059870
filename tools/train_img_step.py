"""Video + image joint training step of LatteIMG-XL/2 on the GPU, the shape of the reference's ucf101_img configs
(configs/ucf101/ucf101_img_train.yaml: local batch 4, 16 video frames + use_image_num 8 images, input 32 = 256 tokens per
frame): fp32 parameters under torch.autocast(bfloat16), `diffusion.training_losses(...)["loss"].mean().backward()` as
train_with_img.py runs it, synthetic latents, seeded weights.  In the same run, plain Latte-XL/2 at batch 5 x 16 frames.

Prints one JSON line per workload:
  ms_per_step           CUDA events around `steps` back-to-back steps (zero_grad + loss + backward), after `warmup` steps
  ada_grad_ms           device time per step of the two adaLN gradients (dW, dsc), CUDA events around them, separate pass
  image_rows_ms         device time per step of the temporal blocks' image-row copies, same pass
  peak_mem_gib          torch.cuda.max_memory_allocated over the measured steps
  gpu, power_limit_w    read from nvidia-smi in the same run
Usage:  python tools/train_img_step.py [--steps 5] [--warmup 2]
"""
import argparse
import os
import sys

import torch

from harness import Timed, card, emit, ms_per_step, require_cuda

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def measure(images, batch, frames, steps, warmup, dev):
    from latte_b200 import LatteIMG_models, Latte_models, training
    from latte_b200.diffusion import create_diffusion
    torch.manual_seed(0)
    table, name = (LatteIMG_models, "LatteIMG-XL/2") if images else (Latte_models, "Latte-XL/2")
    m = table[name](input_size=32, num_classes=101, num_frames=frames, learn_sigma=True, extras=2).to(dev)
    with torch.no_grad():                      # adaLN-Zero leaves the blocks at identity: give every zero weight some values
        for p in m.parameters():
            if p.requires_grad and float(p.abs().max()) == 0.0:
                p.normal_(0, 0.02)
    m.train()
    d = create_diffusion(timestep_respacing="")
    g = torch.Generator().manual_seed(1)
    x = torch.randn(batch, frames + images, 4, 32, 32, generator=g).to(dev)
    y = torch.randint(0, 101, (batch,), generator=g).to(dev)
    t = torch.randint(0, 1000, (batch,), generator=g).to(dev)
    kw = dict(y=y)
    if images:                                 # train_with_img.py:216-220: a list of B label tensors
        kw.update(y_image=[torch.randint(0, 101, (images,), generator=g) for _ in range(batch)], use_image_num=images)

    def step():
        m.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = d.training_losses(m, x, t, kw)["loss"].mean()
        loss.backward()

    for _ in range(warmup):
        step()
    torch.cuda.reset_peak_memory_stats(dev)
    [ms] = ms_per_step(step, steps)
    peak = torch.cuda.max_memory_allocated(dev) / 2 ** 30

    ops = m._train_backend[torch.bfloat16]     # the backend object the warm-up steps created
    timers = [Timed(ops, "ada_outer"), Timed(ops, "ada_dsc"), Timed(training.TrainEngine, "_join_rows")]
    for _ in range(steps):
        step()
    torch.cuda.synchronize()
    for tm in timers:
        tm.restore()
    rows = batch * (frames + images) if images else batch
    res = {"workload": f"{name} training step, {batch} x ({frames} + {images}) frames x 256 tokens, bf16 autocast",
           "local_batch": batch, "frames": frames, "images": images, "ada_rows": rows, "steps": steps, "warmup": warmup,
           "ms_per_step": ms, "ada_grad_ms": (timers[0].ms() + timers[1].ms()) / steps,
           "image_rows_ms": timers[2].ms() / steps, "peak_mem_gib": peak}
    del m
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    require_cuda()
    dev = torch.device("cuda", 0)
    info = card()
    for images, batch in ((8, 4), (0, 5)):
        res = measure(images, batch, 16, args.steps, max(args.warmup, 1), dev)
        res.update(info)
        emit(res)


if __name__ == "__main__":
    main()
