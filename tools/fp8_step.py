"""FP8 against 16-bit sampling on the GPU: one Latte-XL/2 forward_with_cfg step (16 frames x 256 x 256, i.e. 32 x 32
latents, a classifier-free-guidance pair = batch 2), seeded weights of the committed XL/2 golden, fp16 operands with and
without `use_fp8` (QKV and fc1 in e4m3).

The two modes are two models holding the same weights, timed in alternating rounds of `steps` calls (CUDA events, after
`warmup` calls each, CUDA-graph replay as the module runs by default), so clock and co-tenant drift fall on both alike.
Prints one JSON line with, per mode:
  device_ms_per_step   median over rounds of the per-round mean
  per_class_ms         device time per kernel class {gemm, attention, ln_modulate, other} per step, from the library's
                       event profiler in a separate eager pass
  maxabs_vs_fp32       max |forward - golden| on the golden's inputs: the golden is the unmodified reference in fp32
and the card's name and power limit, read in the same run.
Usage:  python tools/fp8_step.py [--steps 30] [--warmup 10] [--rounds 5] [--out DIR]
"""
import argparse
import ctypes as C
import json
import os
import re
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


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
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for fp8_step.json (nothing is written without it)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fp8_step.py measures on a CUDA device; none is visible")

    from golden_sample import as_stored
    from latte_b200 import Latte, _lib
    from oracle import latte_oracle as O

    dev = torch.device("cuda:0")
    g = np.load(os.path.join(ROOT, "tests", "golden", "latte_xl_2_b2.npz"))
    m = re.match(r"(\S+) batch=(\d+) wseed=(\d+) iseed=(\d+) extras=(\d+) frames=(\d+) input=(\d+)", str(g["meta"]))
    name, batch, wseed, iseed, extras, frames, inp = m.group(1), *map(int, m.groups()[1:])
    cfg = O.make_config(name, extras=extras, num_frames=frames, input_size=inp)
    sd = O.make_weights(cfg, wseed)
    x, t, y = O.make_inputs(cfg, batch, iseed)
    x, t = x.to(dev), t.to(dev)
    y = y.to(dev) if extras == 2 else None
    ref = torch.from_numpy(g["out"])

    nets = {}
    for mode in ("fp16", "fp8"):
        net = Latte(input_size=cfg.input_size, hidden_size=cfg.hidden_size, depth=cfg.depth, num_heads=cfg.num_heads,
                    num_frames=cfg.num_frames, num_classes=cfg.num_classes, learn_sigma=True, extras=cfg.extras)
        net.load_state_dict(sd, strict=True)
        net = net.to(dev).eval()
        net.compute_dtype = torch.float16
        net.use_fp8 = mode == "fp8"
        nets[mode] = net

    res = {"workload": f"{name} forward_with_cfg, batch {batch} (CFG pair), {frames} frames, {inp * 8}x{inp * 8} px",
           **card(), "steps": args.steps, "rounds": args.rounds}
    step = lambda net: net.forward_with_cfg(x, t, y=y, cfg_scale=7.0)
    with torch.no_grad():
        for mode, net in nets.items():
            out = net(x, t, y=y).cpu()
            res.setdefault(mode, {})["maxabs_vs_fp32"] = (as_stored(out, g, "out") - ref).abs().max().item()
            for _ in range(args.warmup):
                step(net)
        torch.cuda.synchronize()
        per = {mode: [] for mode in nets}
        for _ in range(args.rounds):
            for mode, net in nets.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.steps):
                    step(net)
                e1.record()
                torch.cuda.synchronize()
                per[mode].append(e0.elapsed_time(e1) / args.steps)
        lib = _lib.load()
        for mode, net in nets.items():
            res[mode]["device_ms_per_step"] = statistics.median(per[mode])
            res[mode]["round_ms"] = [round(v, 4) for v in per[mode]]
            _lib.profile_enable(True)
            for _ in range(args.steps):
                step(net)
            torch.cuda.synchronize()
            pm, pn = (C.c_double * 4)(), (C.c_int * 4)()
            _lib.check(lib.b200_profile_collect(pm, pn, 4), "b200_profile_collect")
            _lib.profile_enable(False)
            res[mode]["per_class_ms"] = {k: pm[i] / args.steps for i, k in enumerate(("gemm", "attention", "ln_modulate", "other"))}
            res[mode]["launches_per_step"] = sum(pn) // args.steps
    res["fp8_speedup"] = res["fp16"]["device_ms_per_step"] / res["fp8"]["device_ms_per_step"]
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "fp8_step.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
