"""What the step timers in tools/ share: the card they ran on, CUDA-event timing, the library's per-class profile, and the
JSON line they print.  The scripts run as `python tools/<script>.py`, so `from harness import ...` finds this file."""
import ctypes as C
import json
import os
import subprocess
import sys

import torch

CLASSES = ("gemm", "attention", "ln_modulate", "other")     # the library's kernel classes, in b200_profile_collect's order


def require_cuda():
    """Exits with a one-line message when no CUDA device is visible."""
    if not torch.cuda.is_available():
        raise SystemExit(f"{os.path.basename(sys.argv[0])} measures on a CUDA device; none is visible")


def card(clock=False):
    """The card's name and power limit (and with `clock`, its max SM clock), read from nvidia-smi in the same run as the
    measurement they belong to."""
    fields = "name,power.limit" + (",clocks.max.sm" if clock else "")
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader,nounits",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        vals = [s.strip() for s in out.strip().splitlines()[0].split(",")]
        res = {"gpu": vals[0], "power_limit_w": float(vals[1])}
        if clock:
            res["max_sm_clock_mhz"] = float(vals[2])
        return res
    except Exception as e:  # noqa: BLE001
        return {"gpu": torch.cuda.get_device_name(), "power_limit_w": None, "nvidia_smi_error": repr(e)[:200]}


def ms_per_step(step, steps, rounds=1):
    """Device ms per call of `step`, one value per round: CUDA events around `steps` back-to-back calls.  The device is
    synchronized first, so the caller's warm-up calls finish before the first round starts."""
    torch.cuda.synchronize()
    per = []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            step()
        e1.record()
        torch.cuda.synchronize()
        per.append(e0.elapsed_time(e1) / steps)
    return per


class Timed:
    """Replaces `owner.name` by a wrapper that brackets each call with CUDA events."""

    def __init__(self, owner, name):
        self.owner, self.name, self.events = owner, name, []
        self.plain = getattr(owner, name)
        ev = self.events
        plain = self.plain

        def timed(*a, **k):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            r = plain(*a, **k)
            e.record()
            ev.append((s, e))
            return r
        setattr(owner, name, staticmethod(timed) if isinstance(owner, type) else timed)

    def restore(self):
        if isinstance(self.owner, type):
            setattr(self.owner, self.name, staticmethod(self.plain))
        else:
            delattr(self.owner, self.name)

    def ms(self):
        return sum(s.elapsed_time(e) for s, e in self.events)


def profile(step, steps, classes=CLASSES):
    """Device ms per step of each kernel class, and launches per step, over `steps` calls of `step` under the library's
    event profiler (b200_profile_enable: CUDA events around every launch; the modules launch eagerly while it is on)."""
    from latte_b200 import _lib
    lib = _lib.load()
    _lib.profile_enable(True)
    for _ in range(steps):
        step()
    torch.cuda.synchronize()
    pm, pn = (C.c_double * 4)(), (C.c_int * 4)()
    _lib.check(lib.b200_profile_collect(pm, pn, 4), "b200_profile_collect")
    _lib.profile_enable(False)
    return {k: pm[i] / steps for i, k in enumerate(classes)}, sum(pn) // steps


def emit(res, out=None, name=None):
    """Prints `res` as one JSON line and, when `out` is given, writes the same line to `out`/`name`."""
    line = json.dumps(res)
    print(line, flush=True)
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, name), "w") as f:
            f.write(line + "\n")
