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
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        name, plim, clk = (s.strip() for s in out.strip().splitlines()[0].split(","))
        return {"gpu": name, "power_limit_w": float(plim), "max_sm_clock_mhz": float(clk)}
    except Exception as e:  # noqa: BLE001
        return {"gpu": torch.cuda.get_device_name(), "power_limit_w": None, "nvidia_smi_error": repr(e)[:200]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "t2i_step.py measures on a CUDA device"
    from latte_b200 import LatteT2V, _lib
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
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(K):
            step()
        e1.record()
        torch.cuda.synchronize()
        device_ms = e0.elapsed_time(e1) / K

        host = []
        for _ in range(K):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            step()
            host.append((time.perf_counter() - t0) * 1e3)
        torch.cuda.synchronize()

        lib = _lib.load()
        _lib.profile_enable(True)
        for _ in range(K):
            step()
        torch.cuda.synchronize()
        pm, pn = (C.c_double * 4)(), (C.c_int * 4)()
        _lib.check(lib.b200_profile_collect(pm, pn, 4), "b200_profile_collect")
        _lib.profile_enable(False)

    res = {"workload": "LatteT2V (Latte-1 config) text-to-image step: 1 x 512 x 512, CFG pair (batch 2), 120 prompt tokens, fp16",
           "steps": K, "warmup": W, "device_ms_per_step": device_ms,
           "host_enqueue_ms": statistics.median(host), "host_enqueue_ms_min": min(host),
           "per_class_ms": {k: pm[i] / K for i, k in enumerate(("gemm", "attention", "layernorm", "other"))},
           "launches_per_step": int(sum(pn) // K)}
    res.update(card())
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
