"""FP8 against 16-bit sampling on the GPU, fp16 operands with and without `use_fp8`.

--model latte (default): one Latte-XL/2 forward_with_cfg step (16 frames x 256 x 256, i.e. 32 x 32 latents, a
  classifier-free-guidance pair = batch 2), seeded weights of the committed XL/2 golden; QKV and fc1 in e4m3.  Timed as
  the module runs by default: CUDA-graph replay.
--model t2v: one Latte-1 (LatteT2V, 28 layer pairs, D = 1152) sampling step as pipeline_latte.py makes it: a CFG pair
  (batch 2) of --frames x 512 x 512 (64 x 64 latents; 16 frames, or 1 for text-to-image) with a 120-token prompt of which
  40 tokens are valid (encoder_attention_mask), seeded weights of the committed Latte-1 goldens; QKV and fc1 of every
  spatial and temporal block in e4m3.  LatteT2V has no CUDA graph: every step is timed as eager launches.

The two modes are two models holding the same weights, timed in alternating rounds of `steps` calls (CUDA events, after
`warmup` calls each), so clock and co-tenant drift fall on both alike.
Prints one JSON line with, per mode:
  device_ms_per_step   median over rounds of the per-round mean
  per_class_ms         device time per kernel class {gemm, attention, ln_modulate, other} per step, from the library's
                       event profiler in a separate eager pass
  maxabs_vs_fp32       max |forward - golden| on the golden's inputs: the golden is the unmodified reference in fp32
                       (t2v: t2v_latte1_b1_l120 at 16 frames, t2v_f1_latte1_b2_l120 at 1 frame)
and the card's name and power limit, read in the same run.
Usage:  python tools/fp8_step.py [--model latte|t2v] [--frames 16|1] [--steps 30] [--warmup 10] [--rounds 5] [--out DIR]
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
    ap.add_argument("--model", choices=("latte", "t2v"), default="latte")
    ap.add_argument("--frames", type=int, choices=(16, 1), default=16, help="t2v: video length (1 = text-to-image)")
    ap.add_argument("--out", default=None, help="directory for fp8_step.json (nothing is written without it)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fp8_step.py measures on a CUDA device; none is visible")

    from latte_b200 import _lib

    dev = torch.device("cuda:0")
    setup = setup_t2v if args.model == "t2v" else setup_latte
    workload, nets, step, maxabs = setup(dev, args)
    res = {"model": args.model, "workload": workload, **card(), "steps": args.steps, "rounds": args.rounds}
    with torch.no_grad():
        for mode, net in nets.items():
            res.setdefault(mode, {})["maxabs_vs_fp32"] = maxabs(net)
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
        name = "fp8_step.json" if args.model == "latte" else f"fp8_step_t2v_f{args.frames}.json"
        with open(os.path.join(args.out, name), "w") as f:
            f.write(line + "\n")


def setup_latte(dev, args):
    from golden_sample import as_stored
    from latte_b200 import Latte
    from oracle import latte_oracle as O

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
    workload = f"{name} forward_with_cfg, batch {batch} (CFG pair), {frames} frames, {inp * 8}x{inp * 8} px, CUDA-graph replay"
    step = lambda net: net.forward_with_cfg(x, t, y=y, cfg_scale=7.0)
    maxabs = lambda net: (as_stored(net(x, t, y=y).cpu(), g, "out") - ref).abs().max().item()
    return workload, nets, step, maxabs


def setup_t2v(dev, args):
    import ast
    from golden_sample import as_stored
    from latte_b200 import LatteT2V
    from oracle import t2v_oracle as T

    g = np.load(os.path.join(ROOT, "tests", "golden", "t2v_latte1_b1_l120.npz" if args.frames == 16 else "t2v_f1_latte1_b2_l120.npz"))
    kw = ast.literal_eval(str(g["cfg"]))
    cfg = T.T2VConfig(**kw)
    sd = T.make_weights(cfg, int(g["wseed"]))
    nets = {}
    for mode in ("fp16", "fp8"):
        net = LatteT2V(**kw)
        net.load_state_dict(sd, strict=True)
        net = net.to(dev).eval()
        net.compute_dtype = torch.float16
        net.use_fp8 = mode == "fp8"
        nets[mode] = net
    del sd
    gx, gt, gtext = T.make_inputs(cfg, int(g["batch"]), int(g["text_len"]), int(g["iseed"]))
    gmask = torch.from_numpy(g["mask"]).to(dev) if "mask" in g else None
    ref = torch.from_numpy(g["out"])
    maxabs = lambda net: (as_stored(net(gx.to(dev), gt.to(dev), encoder_hidden_states=gtext.to(dev), encoder_attention_mask=gmask,
                                        return_dict=False)[0].cpu(), g, "out") - ref).abs().max().item()
    # the timed step: a CFG pair (the same latents twice, as pipeline_latte.py concatenates them), 120-token prompts, 40 valid
    x, t, text = T.make_inputs(cfg, 2, 120, 2024)
    x, t, text = x[:1].repeat(2, 1, 1, 1, 1).to(dev), t[:1].repeat(2).to(dev), text.to(dev)
    mask = torch.zeros(2, 120, dtype=torch.int64, device=dev)
    mask[:, :40] = 1
    step = lambda net: net(x, t, encoder_hidden_states=text, encoder_attention_mask=mask, return_dict=False)[0]
    workload = (f"Latte-1 (LatteT2V, {cfg.num_layers} layer pairs, D = {cfg.inner_dim}) sampling step, batch 2 (CFG pair), "
                f"{cfg.video_length} x {cfg.sample_size * 8}x{cfg.sample_size * 8} px, 120-token prompt (40 valid), eager launches")
    return workload, nets, step, maxabs


if __name__ == "__main__":
    main()
