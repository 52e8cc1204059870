"""LatteT2V sampling steps at several resolutions on the GPU: Latte-1 at 512 x 512, 320 x 512 and 288 x 512.

One Latte-1 (LatteT2V, 28 layer pairs, D = 1152) sampling step as pipeline_latte.py makes it: a classifier-free-guidance
pair (batch 2) with a 120-token prompt of which 40 tokens are valid (encoder_attention_mask), seeded weights
(oracle/t2v_oracle.make_weights(FULL, 0)), fp16 operands, eager launches (LatteT2V has no CUDA graph).  Shapes:
  16 x 512 x 512   64 x 64 latents, 1024 tokens per frame (whole 128-row attention tiles)
  16 x 320 x 512   40 x 64 latents,  640 tokens per frame (whole tiles)
  16 x 288 x 512   36 x 64 latents,  576 tokens per frame (ragged: the last query tile and key chunk of a frame hold 64)
   1 x 320 x 512   text-to-image, 640 tokens
The shapes are timed in alternating rounds of `steps` calls (CUDA events, after `warmup` calls each), so clock and
co-tenant drift fall on all of them alike.  Prints one JSON line with, per shape:
  device_ms_per_step     median over rounds of the per-round mean
  ms_per_1k_tokens       device_ms_per_step per thousand tokens of the step (2 x frames x tokens per frame)
  per_class_ms           device time per kernel class {gemm, attention, ln_modulate, other} per step, from the library's
                         event profiler in a separate pass
and the card's name and power limit, read in the same run.
Usage:  python tools/t2v_res_step.py [--steps 5] [--warmup 2] [--rounds 3] [--out DIR]
"""
import argparse
import os
import statistics
import sys

import torch

from harness import card, emit, ms_per_step, profile, require_cuda

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = [("16x512x512", 16, 64, 64), ("16x320x512", 16, 40, 64), ("16x288x512", 16, 36, 64), ("1x320x512", 1, 40, 64)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for t2v_res_step.json (nothing is written without it)")
    args = ap.parse_args()
    require_cuda()

    from latte_b200 import LatteT2V
    from oracle import t2v_oracle as T
    from oracle.make_golden_t2v import FULL

    dev = torch.device("cuda:0")
    sd = T.make_weights(T.T2VConfig(**FULL), 0)
    nets = {}
    for frames in sorted({s[1] for s in SHAPES}):
        net = LatteT2V(**dict(FULL, video_length=frames))
        net.load_state_dict(sd, strict=True)
        net = net.to(dev).eval()
        net.compute_dtype = torch.float16
        nets[frames] = net
    del sd
    g = torch.Generator().manual_seed(2024)
    text = (torch.randn(1, 120, FULL["caption_channels"], generator=g) * 0.5).repeat(2, 1, 1).to(dev)
    mask = torch.zeros(2, 120, dtype=torch.int64, device=dev)
    mask[:, :40] = 1
    t = torch.tensor([500, 500], device=dev)
    calls = {}
    for name, frames, h, w in SHAPES:
        x = torch.randn(1, 4, frames, h, w, generator=g).repeat(2, 1, 1, 1, 1).to(dev)
        calls[name] = (lambda net=nets[frames], x=x: net(x, t, encoder_hidden_states=text, encoder_attention_mask=mask,
                                                         return_dict=False)[0], 2 * frames * (h // 2) * (w // 2))

    res = {"workload": "Latte-1 (LatteT2V, 28 layer pairs, D = 1152) sampling step, batch 2 (CFG pair), 120-token prompt "
                       "(40 valid), fp16, eager launches", **card(clock=True), "steps": args.steps, "rounds": args.rounds}
    with torch.no_grad():
        for step, _ in calls.values():
            for _ in range(args.warmup):
                step()
        per = {name: [] for name in calls}
        for _ in range(args.rounds):
            for name, (step, _) in calls.items():
                per[name] += ms_per_step(step, args.steps)
        for name, (step, tokens) in calls.items():
            ms = statistics.median(per[name])
            r = res[name] = {"tokens_per_step": tokens, "device_ms_per_step": ms, "ms_per_1k_tokens": ms / (tokens / 1000),
                             "round_ms": [round(v, 3) for v in per[name]]}
            r["per_class_ms"], _ = profile(step, args.steps)
    emit(res, args.out, "t2v_res_step.json")


if __name__ == "__main__":
    main()
