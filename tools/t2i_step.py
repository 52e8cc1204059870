"""One Latte-1 text-to-image denoising step on the GPU: LatteT2V with video_length = 1 at 512 x 512 (64 x 64 latents,
1024 tokens), a classifier-free-guidance pair (batch 2), 120 prompt tokens with the negative prompt masked to 12, fp16,
temporal blocks enabled (configs/t2x/t2i_sample.yaml), seeded synthetic weights.

Prints one JSON line:
  device_ms_per_step    CUDA events around `steps` back-to-back forward calls, after `warmup` calls
  host_enqueue_ms       host time of one forward call on an idle stream, without a synchronise inside the timed region
                        (the launches are queued, not finished); median over `steps` calls
  per_class_ms          device time per kernel class from the library's event profiler, in a separate pass
  gpu, power_limit_w    read from nvidia-smi in the same run
Usage:  python tools/t2i_step.py [--steps 50] [--warmup 10]
"""
import argparse
import os
import statistics
import sys
import time

import torch

from harness import card, emit, ms_per_step, profile, require_cuda

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    require_cuda()
    from latte_b200 import LatteT2V
    from oracle import t2v_oracle as T

    dev = torch.device("cuda", 0)
    cfg = T.T2VConfig(video_length=1)
    net = LatteT2V(video_length=1)
    g = torch.Generator().manual_seed(0)
    with torch.no_grad():
        for prm in net.parameters():
            prm.copy_(torch.randn(prm.shape, generator=g) * (0.05 if prm.dim() == 1 else 1.0 / prm.shape[-1] ** 0.5))
    net = net.to(dev).half().eval()
    x, t, text = T.make_inputs(cfg, 2, 120, 1)
    mask = torch.ones(2, 120, dtype=torch.int64)
    mask[0, 12:] = 0
    xd, td, txd, md = x.to(dev).half(), t.to(dev), text.to(dev).half(), mask.to(dev)
    step = lambda: net(xd, td, encoder_hidden_states=txd, encoder_attention_mask=md,   # noqa: E731
                       enable_temporal_attentions=True, return_dict=False)
    K, W = args.steps, max(args.warmup, 3)
    with torch.no_grad():
        for _ in range(W):
            step()
        [device_ms] = ms_per_step(step, K)

        host = []
        for _ in range(K):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            step()
            host.append((time.perf_counter() - t0) * 1e3)
        torch.cuda.synchronize()
        per_class, launches = profile(step, K, classes=("gemm", "attention", "layernorm", "other"))

    res = {"workload": "LatteT2V (Latte-1 config) text-to-image step: 1 x 512 x 512, CFG pair (batch 2), 120 prompt tokens, fp16",
           "steps": K, "warmup": W, "device_ms_per_step": device_ms,
           "host_enqueue_ms": statistics.median(host), "host_enqueue_ms_min": min(host),
           "per_class_ms": per_class, "launches_per_step": launches}
    res.update(card(clock=True))
    emit(res)


if __name__ == "__main__":
    main()
