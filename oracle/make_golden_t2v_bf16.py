"""Generate tests/golden/t2v_ref_bf16.npz: the reference LatteT2V's own bf16-autocast deviation on the inputs and weights of
existing t2v goldens, the accuracy unit of the FP8 sampling test (tests/test_gpu_fp8_t2v.py), as `ref_bf16_maxabs` is for
the Latte goldens (oracle/make_golden.py).

TEST INFRASTRUCTURE.  Runs only in the build container (the GPU box has no /root/reference); the output is committed.
Usage:  python oracle/make_golden_t2v_bf16.py [--full]      (--full adds the two Latte-1 cases, minutes of CPU each)

For each case it rebuilds the reference module, weights, inputs and prompt mask exactly as oracle/make_golden_t2v.py's
`gen_forward` did for the committed golden, checks that the fp32 output equals the committed `out` (sampled as stored),
runs the same module under `torch.autocast("cpu", torch.bfloat16)` (as oracle/make_golden.py does for Latte), and records
max |out_bf16 - out| over the whole output.  Writes only t2v_ref_bf16.npz; every existing golden is left as it is.
"""
import argparse
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import t2v_oracle as T  # noqa: E402
from oracle.make_golden_t2v import FULL, TINY, HD72, build_ref_model, load_reference, make_mask  # noqa: E402
from oracle.make_golden_t2v_frames import F1, F12, F1_FULL  # noqa: E402
from golden_sample import as_stored  # noqa: E402

# case -> (config, batch, text_len, wseed, iseed, valid prompt lengths, temporal): the arguments each golden was made with
CASES = {
    "tiny_b2_l20": (TINY, 2, 20, 3, 4, None, True),
    "tiny_b2_l20_notemporal": (TINY, 2, 20, 3, 4, None, False),
    "hd72_b2_l120_masked": (HD72, 2, 120, 5, 6, [12, 120], True),
    "f12_b1_l20": (F12, 1, 20, 13, 14, None, True),
    "f1_b2_l20": (F1, 2, 20, 11, 12, None, True),
}
FULL_CASES = {
    "f1_latte1_b2_l120": (F1_FULL, 2, 120, 0, 124, [12, 120], True),
    "latte1_b1_l120": (FULL, 1, 120, 0, 123, None, True),
}


def ref_bf16_maxabs(ref, tag, cfg_kw, batch, text_len, wseed, iseed, valid, temporal, golden_dir):
    cfg = T.T2VConfig(**cfg_kw)
    sd = T.make_weights(cfg, wseed)
    x, t, text = T.make_inputs(cfg, batch, text_len, iseed)
    m = build_ref_model(ref, cfg, sd)
    mask = make_mask(batch, text_len, valid) if valid is not None else None
    g = np.load(os.path.join(golden_dir, f"t2v_{tag}.npz"))
    assert int(g["temporal"]) == int(temporal) and int(g["batch"]) == batch and int(g["text_len"]) == text_len
    assert int(g["wseed"]) == wseed and int(g["iseed"]) == iseed and str(g["cfg"]) == repr(cfg_kw)
    t0 = time.time()
    call = lambda: m(x, t, encoder_hidden_states=text, encoder_attention_mask=mask, enable_temporal_attentions=temporal,
                     return_dict=False)[0]
    with torch.no_grad():
        out = call()
        stored = as_stored(out, g, "out").numpy()
        assert np.array_equal(stored, g["out"]), f"{tag}: fp32 output differs from the committed golden " \
            f"(max-abs {np.abs(stored - g['out']).max():.3e})"
        with torch.autocast("cpu", dtype=torch.bfloat16):
            out_bf16 = call().float()
    dev = float((out_bf16 - out).abs().max().item())
    print(f"{tag}: ref bf16-autocast max-abs deviation {dev:.3e} (output absmax {out.abs().max():.3f})  "
          f"({time.time() - t0:.1f} s)", flush=True)
    return dev


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--full", action="store_true", help="also the two Latte-1 cases (28 layers at 512 x 512)")
    args = ap.parse_args()
    torch.manual_seed(0)
    golden_dir = os.path.join(ROOT, "tests", "golden")
    ref = load_reference()
    cases = dict(CASES, **(FULL_CASES if args.full else {}))
    res = {tag: np.float32(ref_bf16_maxabs(ref, tag, *c, golden_dir)) for tag, c in cases.items()}
    path = os.path.join(golden_dir, "t2v_ref_bf16.npz")
    np.savez(path, **res)
    print(f"{path}: {len(res)} cases")
