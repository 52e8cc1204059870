"""CPU: the LatteT2V restatement (oracle/t2v_oracle.py) against goldens of the UNMODIFIED reference module at video lengths
1 (text-to-image), 3 and 12 (oracle/make_golden_t2v_frames.py).  Same tolerance as tests/test_oracle_t2v.py: 5e-4."""
import os

import numpy as np
import pytest
import torch

from oracle import t2v_oracle as T
from golden_sample import as_stored  # noqa: E402
from test_oracle_t2v import load_case

CASES = ["f1_b2_l20", "f1_b2_l20_notemporal", "f1_b2_l20_masked", "f12_b1_l20", "f3_b2_l20"]


def _check(golden_dir, tag):
    g, cfg, sd, x, t, text, mask = load_case(golden_dir, tag)
    out = T.t2v_forward(sd, cfg, x, t, text, enable_temporal=bool(int(g["temporal"])), text_mask=mask)
    ref = torch.from_numpy(g["out"])
    out = as_stored(out, g, "out")
    assert out.shape == ref.shape
    assert (out - ref).abs().max().item() < 5e-4


@pytest.mark.parametrize("tag", CASES)
def test_forward_matches_reference_golden(golden_dir, tag):
    _check(golden_dir, tag)


def test_latte1_t2i_shape_matches_reference_golden(golden_dir):
    """28 layers, 1 x 512 x 512, L = 120, CFG pair with one masked prompt (make_golden_t2v_frames.py --full)."""
    if not os.path.exists(os.path.join(golden_dir, "t2v_f1_latte1_b2_l120.npz")):
        pytest.skip("t2v_f1_latte1_b2_l120.npz not generated (make_golden_t2v_frames.py --full)")
    _check(golden_dir, "f1_latte1_b2_l120")


def test_one_frame_temporal_blocks_change_the_output(golden_dir):
    """At video_length 1 the reference still runs the temporal blocks (attention over one frame, MLP), so the goldens with
    and without them differ; only temp_pos_embed is skipped."""
    a = np.load(os.path.join(golden_dir, "t2v_f1_b2_l20.npz"))["out"]
    b = np.load(os.path.join(golden_dir, "t2v_f1_b2_l20_notemporal.npz"))["out"]
    assert np.abs(a - b).max() > 1e-2
