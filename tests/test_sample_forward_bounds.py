"""CPU: the machinery of test_gpu_sample_fp64.py rehearsed at the tiny golden shapes (latte_tiny64_2_b2,
t2v_tiny_b2_l20_masked, t2v_res_g10x16_b2_l20_masked), with the fp32 oracle standing in for the native output and the
oracle under CPU bf16 autocast as the yardstick (for the FP8 recipe: the oracle with e4m3 operands on QKV and fc1, in
fp32 as the stand-in and in fp64 as the yardstick).

* The restated attention and feed-forward of tests/sample_fp64.py, with no edit, compute exactly what the oracles compute.
* The stand-in passes the budget; an output 10 % too large fails it.
* Every wrong result the GPU test rejects exceeds the budget here too: two heads' attention outputs swapped in the last
  spatial block, the last frame missing from the temporal keys, sample 1 given sample 0's timestep, the CFG pair's labels
  swapped, guidance on all 2C channels, the caption mask ignored, layer l reading layer l - 1's text K/V, the square or
  wrongly interpolated position table of a non-square grid, and with e4m3 operands every token's activations scaled back
  with the next token's scale and the weight scale dropped on the last 32 output channels."""
import ast
import contextlib
import os

import numpy as np
import pytest
import torch

import sample_fp64 as S
from oracle import latte_oracle as O
from oracle import t2v_oracle as T
from oracle import t2v_res_oracle as R

BF = S.BUDGET["bf16"]
SHAPES = ["latte_tiny64", "t2v_tiny", "t2v_res_g10x16"]


class Shape:
    """`out(dtype, autocast=None, **kw)`: the oracle on the golden shape's weights and inputs (kw as the GPU test's
    Case.oracle: t, y, mask, guided, cfg)."""

    def __init__(self, name, golden_dir):
        self.name = name
        if name == "latte_tiny64":
            self.kind, self.p, self.cf = "latte", 2, False
            self.cfg = O.make_config("Latte-tiny64/2", extras=2, num_frames=8, input_size=16)
            self.w = O.make_weights(self.cfg, 11)
            self.x, self.t, self.y = O.make_inputs(self.cfg, 2, 12)
            self.last_spatial, self.grid = f"blocks.{self.cfg.depth - 2}.attn.", None
            return
        g = np.load(os.path.join(golden_dir, "t2v_tiny_b2_l20_masked.npz" if name == "t2v_tiny" else "t2v_res_g10x16_b2_l20_masked.npz"))
        self.kind, self.p, self.cf = "t2v", 2, True
        self.cfg = T.T2VConfig(**ast.literal_eval(str(g["cfg"])))
        self.w = T.make_weights(self.cfg, int(g["wseed"]))
        if name == "t2v_tiny":
            self.x, self.t, self.text = T.make_inputs(self.cfg, 2, int(g["text_len"]), int(g["iseed"]))
        else:
            self.x, self.t, self.text = R.make_inputs(self.cfg, 2, int(g["text_len"]), int(g["iseed"]), int(g["height"]),
                                                      int(g["width"]))
        self.mask = torch.from_numpy(g["mask"]).float()
        self.last_spatial = f"transformer_blocks.{self.cfg.num_layers - 1}.attn1"
        self.grid = (self.x.shape[3] // 2, self.x.shape[4] // 2)

    def out(self, dtype, autocast=None, **kw):
        sd = {k: v.to(dtype) for k, v in self.w.items()}
        ctx = torch.autocast("cpu", dtype=autocast) if autocast is not None else contextlib.nullcontext()
        with torch.no_grad(), ctx:
            if self.kind == "latte":
                return S.latte_out(sd, self.cfg, self.x, kw.get("t", self.t), kw.get("y", self.y), dtype, kw.get("cfg"),
                                   kw.get("guided"))
            return S.t2v_out(sd, self.cfg, self.x, self.t, self.text, kw["mask"] if "mask" in kw else self.mask, dtype)

    def edited(self, dtype=torch.float64, **kw):
        with S.edits(**kw):
            return self.out(dtype)


@pytest.fixture(scope="module", params=SHAPES)
def shape(request, golden_dir):
    s = Shape(request.param, golden_dir)
    s.o64, s.got, s.oac = s.out(torch.float64), s.out(torch.float32), s.out(torch.float32, torch.bfloat16)
    return s


def test_restated_blocks_match_the_oracles(shape):
    for dt in (torch.float64, torch.float32):
        assert torch.equal(shape.edited(dt), shape.out(dt))


def test_stand_in_passes(shape):
    res = S.check(shape.got, shape.o64, shape.oac, BF, shape.p, shape.cf)
    assert all(w.ratio <= 1.0 for w in res.values()), res


def test_scaled_output_is_rejected(shape):
    """An output 10 % too large fails in both halves (bf16 autocast is within about 1 % of fp64 here)."""
    res = S.check((shape.o64 * 1.1).float(), shape.o64, shape.oac, BF, shape.p, shape.cf)
    assert all(w.ratio > 1.0 for w in res.values()), res


def _wrong_results(s):
    out = [("swapped heads", s.edited(core=S.swap_heads(s.last_spatial))),
           ("last frame missing from the temporal keys", s.edited(core=S.drop_last_key(S.is_temporal)))]
    if s.kind == "latte":
        out.append(("sample 1 given sample 0's timestep", s.out(torch.float64, t=s.t[[0, 0]])))
    else:
        out.append(("caption mask ignored", s.out(torch.float64, mask=None)))
        out.append(("layer l - 1's text K/V", s.edited(kv_prefix=S.previous_layer_text_kv)))
    if s.grid is not None and s.grid[0] != s.grid[1]:
        for what, fn in (("square table", S.square_table), ("table of base_size grid_h", S.other_base_table)):
            with S.pos_table(fn):
                out.append((what, s.out(torch.float64)))
    return out


def test_budget_rejects_the_wrong_results(shape):
    for what, wrong in _wrong_results(shape):
        w = S.rejected(shape.got, shape.o64, shape.oac, wrong, shape.o64, BF, shape.p, shape.cf)
        assert w.ratio > 1.0, (what, w)


def test_budget_rejects_wrong_guidance(golden_dir):
    """xl2_cfg's rejections on forward_with_cfg of the tiny64 CFG pair (latte_oracle.make_inputs gives sample 1 the null
    class): labels swapped, and guidance on all 2C channels."""
    s = Shape("latte_tiny64", golden_dir)
    kw = dict(cfg=4.0)
    o64, got, oac = s.out(torch.float64, **kw), s.out(torch.float32, **kw), s.out(torch.float32, torch.bfloat16, **kw)
    assert all(w.ratio <= 1.0 for w in S.check(got, o64, oac, BF, s.p, s.cf).values())
    for what, wrong in (("labels swapped", s.out(torch.float64, y=s.y.flip(0), **kw)),
                        ("guidance on all channels", s.out(torch.float64, guided=2 * s.cfg.in_channels, **kw))):
        w = S.rejected(got, o64, oac, wrong, o64, BF, s.p, s.cf)
        assert w.ratio > 1.0, (what, w)


def test_fp8_recipe(shape):
    """The e4m3 recipe in fp32 passes against the same recipe in fp64 as its yardstick; the two FP8 defects fail."""
    budget = S.BUDGET["fp8"]
    oac = shape.edited(lin=S.fp8_recipe())
    got = shape.edited(torch.float32, lin=S.fp8_recipe())
    res = S.check(got, shape.o64, oac, budget, shape.p, shape.cf)
    assert all(w.ratio <= 1.0 for w in res.values()), res
    for defect in ("token", "w_scale"):
        w = S.rejected(got, shape.o64, oac, shape.edited(lin=S.fp8_recipe(defect)), oac, budget, shape.p, shape.cf)
        assert w.ratio > 1.0, (defect, w)


def test_qdq_rows_matches_the_weight_quantization():
    """qdq_rows is the quantization test_gpu_fp8.py pins the kernels' bytes to: amax / 448 per row, torch's e4m3 cast."""
    g = torch.Generator().manual_seed(0)
    w = torch.randn(37, 80, generator=g) * 0.03
    w[0] = 0.0
    amax = w.abs().amax(1)
    s = torch.where(amax > 0, amax / 448.0, torch.ones_like(amax))
    want = (w / s[:, None]).to(torch.float8_e4m3fn).float() * s[:, None]
    assert torch.equal(S.qdq_rows(w), want)
