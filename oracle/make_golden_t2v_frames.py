"""Generate tests/golden/t2v_f{1,3,12}_*.npz: LatteT2V at video lengths other than the 16 frames of the existing goldens,
from the UNMODIFIED reference /root/reference/models/latte_t2v.py (loaded exactly as in oracle/make_golden_t2v.py).

TEST INFRASTRUCTURE.  Runs only in the build container (the GPU box has no /root/reference); outputs are committed.
Usage:  python oracle/make_golden_t2v_frames.py [--full]

Writes only the files below; the goldens of make_golden_t2v.py are left as they are.
  t2v_f1_*     video_length 1 (text-to-image, configs/t2x/t2i_sample.yaml), 256 tokens per frame, head_dim 72: with the
               temporal blocks (the reference runs them at one frame, skipping only temp_pos_embed, latte_t2v.py:894),
               without them, and with a padded prompt.
  t2v_f12_*    12 frames: 10 tokens per temporal attention tile, 256 = 25 * 10 + 6 (a partial last group), head_dim 80.
  t2v_f3_*     3 frames: 42 tokens per tile, 256 = 6 * 42 + 4, head_dim 64.
  --full       t2v_f1_latte1_b2_l120: the Latte-1 text-to-image call (28 layers, 512 x 512 -> 64 x 64 latents, 4096 caption
               channels, 120 prompt tokens) on a classifier-free-guidance pair, the first prompt masked to 12 tokens.
Inputs and weights come from the seeds recorded in each file (oracle/t2v_oracle.make_weights / make_inputs).
"""
import argparse
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle.make_golden_t2v import FULL, gen_forward, load_reference  # noqa: E402

F1 = dict(num_attention_heads=8, attention_head_dim=72, num_layers=2, sample_size=32, video_length=1, caption_channels=256)
F12 = dict(num_attention_heads=4, attention_head_dim=80, num_layers=2, sample_size=32, video_length=12, caption_channels=256)
F3 = dict(num_attention_heads=2, attention_head_dim=64, num_layers=2, sample_size=32, video_length=3, caption_channels=256)
F1_FULL = dict(FULL, video_length=1)

if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--full", action="store_true", help="also the Latte-1 text-to-image shape: 28 layers, 1 x 512 x 512, L=120, batch 2")
    args = ap.parse_args()
    torch.manual_seed(0)
    out_dir = os.path.join(ROOT, "tests", "golden")
    ref = load_reference()
    gen_forward(ref, "f1_b2_l20", F1, 2, 20, 11, 12, out_dir)
    gen_forward(ref, "f1_b2_l20_notemporal", F1, 2, 20, 11, 12, out_dir, temporal=False)
    gen_forward(ref, "f1_b2_l20_masked", F1, 2, 20, 11, 12, out_dir, valid=[5, 20])
    gen_forward(ref, "f12_b1_l20", F12, 1, 20, 13, 14, out_dir)
    gen_forward(ref, "f3_b2_l20", F3, 2, 20, 15, 16, out_dir)
    if args.full:
        gen_forward(ref, "f1_latte1_b2_l120", F1_FULL, 2, 120, 0, 124, out_dir, valid=[12, 120], digest=False)
