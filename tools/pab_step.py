"""Latte-1 sampling trajectories with and without the attention cache (Pyramid Attention Broadcast, LatteT2V.enable_cache).

Workloads: LatteT2V in the Latte-1 configuration with seeded synthetic weights, a classifier-free-guidance pair (batch 2),
a 120-token prompt with 40 valid tokens (the rest masked), fp16; 50 descending timesteps 981, 961, ..., 1; at
16 x 512 x 512 (video) and 1 x 512 x 512 (text-to-image).  Each call is followed by guidance (scale 7.5) and a fixed
Euler-style update x -= eps / 50 that stands in for the sampler, so the final latents carry every call's output.
Arms, alternated within one run for 3 rounds after one warm-up trajectory each:
  off   the cache disabled
  pab   skip ranges spatial 2 / temporal 4 / cross 6, timestep windows (100, 800) / (100, 800) / (100, 900)

Prints one JSON line per workload:
  ms_per_trajectory     {arm: [per round]}: CUDA events around the 50 calls and their updates
  per_class_ms          {arm: device ms per kernel class over one trajectory}, from the library's event profiler in a
                        separate pass
  computed / reused     per kind, calls of the pab arm's trajectory
  cache_gb, peak_gb     the pab arm's cache buffers, and each arm's peak allocated memory
  final_latent_max_abs  max |x_pab - x_off| of the final latents (on seeded weights this shows the mechanics only: PAB's
                        effect on video quality rests on the published evaluation)
  gpu, power_limit_w    read from nvidia-smi in the same run
Usage:  python tools/pab_step.py [--rounds 3] [--workloads video,t2i] [--out DIR]
"""
import argparse
import os
import sys

import torch

from harness import card, emit, ms_per_step, profile, require_cuda

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TAUS = list(range(981, 0, -20))
KINDS = ("spatial", "temporal", "cross")


def _model(frames, dev):
    from latte_b200 import LatteT2V
    net = LatteT2V(video_length=frames)
    g = torch.Generator().manual_seed(0)
    with torch.no_grad():
        for prm in net.parameters():
            prm.copy_(torch.randn(prm.shape, generator=g) * (0.05 if prm.dim() == 1 else 1.0 / prm.shape[-1] ** 0.5))
    return net.to(dev).half().eval()


def run_workload(frames, rounds, dev):
    from latte_b200 import PyramidAttentionBroadcastConfig
    net = _model(frames, dev)
    g = torch.Generator().manual_seed(1)
    x0 = torch.randn(1, 4, frames, 64, 64, generator=g).to(dev).half()
    text = (torch.randn(2, 120, 4096, generator=g) * 0.5).to(dev).half()
    mask = torch.zeros(2, 120, dtype=torch.int64, device=dev)
    mask[:, :40] = 1
    ts = [torch.full((2,), tau, dtype=torch.int64, device=dev) for tau in TAUS]
    pab = PyramidAttentionBroadcastConfig(spatial_attention_block_skip_range=2, temporal_attention_block_skip_range=4,
                                          cross_attention_block_skip_range=6, cross_attention_timestep_skip_range=(100, 900))
    counts = {k: [0, 0] for k in KINDS}
    final = {}

    def trajectory(arm, count=False):
        x = x0.clone()
        for t in ts:
            out = net(torch.cat([x, x]), t, encoder_hidden_states=text, encoder_attention_mask=mask, return_dict=False)[0]
            eps_c, eps_u = out[:1, :4], out[1:, :4]
            x = x - (eps_u + 7.5 * (eps_c - eps_u)) / len(ts)
            if count:
                for k in KINDS:
                    counts[k][net._pab_state.last_modes[k] == 2] += 1
        final[arm] = x

    def arm(name):
        if name == "pab":
            net.enable_cache(pab)
        else:
            net.disable_cache()
        return lambda: trajectory(name)

    res = {"workload": f"LatteT2V (Latte-1 config) {frames} x 512 x 512, CFG pair (batch 2), 120 prompt tokens (40 valid), "
                       f"fp16, 50 timesteps 981..1",
           "ms_per_trajectory": {"off": [], "pab": []}, "per_class_ms": {}, "peak_gb": {}}
    with torch.no_grad():
        for name in ("off", "pab"):
            torch.cuda.reset_peak_memory_stats(dev)
            step = arm(name)
            step()
            torch.cuda.synchronize()
            res["peak_gb"][name] = torch.cuda.max_memory_allocated(dev) / 1e9
        for _ in range(rounds):
            for name in ("off", "pab"):
                res["ms_per_trajectory"][name] += ms_per_step(arm(name), 1)
        for name in ("off", "pab"):
            arm(name)
            res["per_class_ms"][name], _ = profile(lambda: trajectory(name, count=name == "pab"), 1)
        net.enable_cache(pab)
        trajectory("pab")
        res["cache_gb"] = sum(b.numel() * b.element_size() for b in net._pab_state.buffers.values()) / 1e9
        net.disable_cache()
        trajectory("off")
    res["computed"] = {k: c[0] for k, c in counts.items()}
    res["reused"] = {k: c[1] for k, c in counts.items()}
    res["final_latent_max_abs"] = (final["pab"].float() - final["off"].float()).abs().max().item()
    res["final_latent_absmax"] = final["off"].float().abs().max().item()
    off, on = min(res["ms_per_trajectory"]["off"]), min(res["ms_per_trajectory"]["pab"])
    res["speedup_best"] = off / on
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--workloads", default="video,t2i")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    require_cuda()
    dev = torch.device("cuda", 0)
    for w in args.workloads.split(","):
        res = run_workload({"video": 16, "t2i": 1}[w], args.rounds, dev)
        res.update(card(clock=True))
        emit(res, args.out, f"pab_step_{w}.json")
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
