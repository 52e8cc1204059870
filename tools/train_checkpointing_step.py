"""Gradient checkpointing on the GPU: ms per training step and peak memory with and without `enable_gradient_checkpointing()`.

Workloads (fp32 parameters under torch.autocast(bfloat16), seeded weights, synthetic latents):
  Latte-1 (LatteT2V, 28 layer pairs, 16 x 72 heads, caption 4096; a 120-token prompt with 40 valid tokens, loss = mean(out^2))
    16 x 512^2, batch 1    plain and checkpointed, alternated
    16 x 512^2, batch 4    checkpointed only
    64 x 512^2, batch 1    checkpointed only
  Latte-XL/2 (diffusion.training_losses, 101 classes)
    16 x 256^2, batch 5    plain and checkpointed, alternated
Before a workload runs, its peak is predicted from the shapes (parameters, their 16-bit copies and gradients, plus the saved
activations: 46 bytes per token and channel per block plain, 4 checkpointed, plus one block's 46); a workload predicted above
85 % of the card's memory is skipped, so the script never probes for out-of-memory.

Prints one JSON line per (workload, mode, round):
  ms_per_step     CUDA events around `steps` back-to-back steps (zero_grad + forward + loss + backward), after `warmup` steps
  peak_mem_gib    torch.cuda.max_memory_allocated over the timed steps
  predicted_gib   the estimate above
  gpu, power_limit_w read from nvidia-smi in the same run
Usage:  python tools/train_checkpointing_step.py [--steps 3] [--warmup 1] [--rounds 2]
"""
import argparse
import os
import sys

import torch

from harness import card, emit, ms_per_step, require_cuda

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (model, frames, latent size, batch, modes)
WORKLOADS = [("latte1", 16, 64, 1, ("plain", "ckpt")), ("latte1", 16, 64, 4, ("ckpt",)), ("latte1", 64, 64, 1, ("ckpt",)),
             ("xl2", 16, 32, 5, ("plain", "ckpt"))]


def build(kind, frames, size, dev):
    """(model in training mode on `dev`, number of blocks, width)."""
    torch.manual_seed(0)
    if kind == "latte1":
        from latte_b200 import LatteT2V
        with torch.device(dev):
            m = LatteT2V(video_length=frames, sample_size=size)
        return m.to(dev).train(), 2 * m.config.num_layers, m.inner_dim
    from latte_b200 import Latte_models
    with torch.device(dev):
        m = Latte_models["Latte-XL/2"](input_size=size, num_classes=101, num_frames=frames, learn_sigma=True, extras=2)
    with torch.no_grad():                      # adaLN-Zero leaves the blocks at identity: give every zero weight some values
        for p in m.parameters():
            if p.requires_grad and float(p.abs().max()) == 0.0:
                p.normal_(0, 0.02)
    return m.to(dev).train(), m.depth, m.hidden_size


def make_step(kind, m, frames, size, batch, dev):
    g = torch.Generator().manual_seed(1)
    t = torch.randint(0, 1000, (batch,), generator=g).to(dev)
    if kind == "latte1":
        x = torch.randn(batch, 4, frames, size, size, generator=g).to(dev)
        text = (torch.randn(batch, 120, 4096, generator=g) * 0.5).to(dev)
        mask = torch.zeros(batch, 120, device=dev)
        mask[:, :40] = 1

        def loss_fn():
            out = m(x, t, encoder_hidden_states=text, encoder_attention_mask=mask).sample
            return (out.float() ** 2).mean()
    else:
        from latte_b200.diffusion import create_diffusion
        d = create_diffusion(timestep_respacing="")
        x = torch.randn(batch, frames, 4, size, size, generator=g).to(dev)
        y = torch.randint(0, 101, (batch,), generator=g).to(dev)

        def loss_fn():
            return d.training_losses(m, x, t, dict(y=y))["loss"].mean()

    def step():
        m.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = loss_fn()
        loss.backward()
    return step


def predicted_bytes(m, blocks, width, frames, size, batch, ckpt):
    P = sum(p.numel() for p in m.parameters())
    TD = batch * frames * (size // 2) ** 2 * width
    acts = blocks * TD * 4 + 46 * TD if ckpt else blocks * TD * 46
    return P * (4 + 2 + 4) + acts + 16 * TD          # + the backward's own buffers (dx, gradient temporaries)


def measure(step, steps, warmup, dev):
    for _ in range(warmup):
        step()
    torch.cuda.reset_peak_memory_stats(dev)
    [ms] = ms_per_step(step, steps)
    return ms, torch.cuda.max_memory_allocated(dev) / 2 ** 30


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=2, help="alternations of plain / checkpointed where both are measured")
    args = ap.parse_args()
    require_cuda()
    dev = torch.device("cuda", 0)
    info = card()
    total = torch.cuda.get_device_properties(dev).total_memory
    built = None
    for kind, frames, size, batch, modes in WORKLOADS:
        if built is None or built[0] != (kind, frames, size):
            built = m = step = None             # free the previous model before building the next one
            torch.cuda.empty_cache()
            built = ((kind, frames, size),) + build(kind, frames, size, dev)
        _, m, blocks, width = built
        name = ("Latte-1 (LatteT2V)" if kind == "latte1" else "Latte-XL/2") + f", {batch} x {frames} frames x {size * 8}^2"
        step = make_step(kind, m, frames, size, batch, dev)
        for r in range(args.rounds if len(modes) > 1 else 1):
            for mode in modes:
                ckpt = mode == "ckpt"
                pred = predicted_bytes(m, blocks, width, frames, size, batch, ckpt)
                res = {"workload": name, "mode": mode, "round": r, "batch": batch, "frames": frames, "latent": size,
                       "predicted_gib": pred / 2 ** 30}
                if pred > 0.85 * total:
                    res["skipped"] = "predicted peak above 85 % of the card's memory"
                else:
                    m.gradient_checkpointing = ckpt
                    ms, peak = measure(step, args.steps, max(args.warmup, 1), dev)
                    res.update(steps=args.steps, warmup=args.warmup, ms_per_step=ms, peak_mem_gib=peak)
                res.update(info)
                emit(res)
        m.gradient_checkpointing = False


if __name__ == "__main__":
    main()
