"""GPU: the sampling forwards pinned to fp64 row by row, at the geometries and precisions the models sample at.

Each model runs as sampling runs it: `eval()`, no grad, default settings.  Every module call is made three times and the
three outputs must be bit-identical: for Latte the first call runs eagerly, the second captures its CUDA graph and the
third replays it; LatteT2V launches eagerly every time.  The third output is held to the budget of tests/sample_fp64.py
against the functional oracles (oracle/latte_oracle.py, oracle/t2v_oracle.py, oracle/t2v_res_oracle.py) evaluated in
fp64 on the GPU on the module's own weights and inputs, row by row (one row per sample, frame and patch token, eps and
variance halves apart), with the oracle under the recipe's own yardstick as a[r]: fp16 / bf16 autocast on the fp32
weights, fp16 autocast on the fp16 weights of `model.half()`, or the fp64 oracle with e4m3 operands on every QKV and fc1
for `use_fp8`.  The native forward must be no less accurate than its yardstick, row for row, to within K = 4.

Cases (production widths, heads and token counts; depth 4 = two block pairs, so per-layer weight and K/V offsets are used):
  xl2_cfg      Latte-XL/2 (1152 wide, 16 heads of 72), 16 frames of 32 x 32 latents (256 tokens), extras = 2:
               forward_with_cfg(cfg_scale = 4) on a (label, null) pair, and the same through precompute_conditioning /
               trajectory_step, which must be bit-identical
  xl2_t        the same model, forward on B = 2 with t = 0 and t = 999 and two labels
  xl4          Latte-XL/4, 64 tokens per frame (the packed spatial attention)
  t2v_512      a Latte-1 layer pair stack (16 heads of 72, 4096-channel captions of 120 tokens), 16 frames at 512 x 512 (1024
               tokens per frame), B = 2 as a CFG pair whose sample 1 has a caption masked to 12 tokens
  t2v_320x512  the same at a 40 x 64 latent: 640 tokens, whole tiles, a non-square interpolated position table
  t2v_288x512  36 x 64: 576 tokens, the ragged spatial attention
  t2v_t2i      video_length = 1 at 512 x 512
  xl2_full / t2v_full   28 blocks of Latte-XL/2 and 28 layer pairs of Latte-1 (fp16 only), the cfg pair and t2v_512 inputs

Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit (the whole file: 113 s; the largest peak of allocated memory
24.7 GiB, t2v_full).  "worst": the worst row's error over its budget; "K needed": the largest K any row needs; then the
native error / yardstick a[r] of the worst row, and the weakest asserted rejection in units of the budget:

    case         recipe  worst  K needed  worst row: native / a   weakest rejection           time   peak
    xl2_cfg      fp16    0.20   0.16      0.0087 / 0.0093         13.3 (last frame)           3.8 s   2.7 GiB
    xl2_cfg      bf16    0.21   0.73      0.0165 / 0.0183         2.16 (last frame)           2.9 s   2.7 GiB
    xl2_cfg      half    0.18   0         0.0085 / 0.0088         12.9 (last frame)           2.6 s   2.9 GiB
    xl2_cfg      fp8     0.28   1.09      0.259 / 0.231           2.01 (heads swapped)        2.8 s   2.7 GiB
    xl2_t        fp16    0.17   0         0.0023 / 0.0023         16.1 (last frame)           2.5 s   2.7 GiB
    xl2_t        bf16    0.24   0.78      0.0178 / 0.0179         2.66 (last frame)           2.8 s   2.7 GiB
    xl4          fp16    0.13   0         0.0034 / 0.0048         8.37 (last frame)           2.4 s   1.6 GiB
    xl4          bf16    0.18   0.53      0.0273 / 0.0363         1.36 (last frame)           2.5 s   1.6 GiB
    t2v_512      fp16    0.18   0         0.0025 / 0.0023         13.1 (last frame)           2.9 s  12.1 GiB
    t2v_512      bf16    0.25   0.85      0.0211 / 0.0201         2.01 (last frame)           2.8 s  12.1 GiB
    t2v_512      half    0.20   0         0.0028 / 0.0021         12.6 (last frame)           2.8 s  12.2 GiB
    t2v_512      fp8     0.28   1.05      0.0453 / 0.0392         1.71 (heads swapped)        3.4 s  12.1 GiB
    t2v_320x512  fp16    0.18   0         0.0023 / 0.0023         12.2 (last frame)           2.7 s   6.2 GiB
    t2v_320x512  bf16    0.24   0.83      0.0207 / 0.0203         2.0 (last frame)            2.5 s   6.2 GiB
    t2v_320x512  fp8     0.28   1.06      0.0584 / 0.0514         1.70 (heads swapped)        2.9 s   6.1 GiB
    t2v_288x512  fp16    0.20   0         0.0028 / 0.0025         11.1 (last frame)           2.4 s   5.4 GiB
    t2v_288x512  bf16    0.23   0.78      0.0198 / 0.0205         1.75 (last frame)           2.5 s   5.4 GiB
    t2v_288x512  fp8     0.27   1.02      0.0447 / 0.0399         1.78 (heads swapped)        3.1 s   5.4 GiB
    t2v_t2i      fp16    0.17   0         0.0025 / 0.0027         14.0 (heads swapped)        1.8 s   2.0 GiB
    t2v_t2i      bf16    0.23   0.78      0.0212 / 0.0220         2.36 (heads swapped)        1.7 s   2.0 GiB
    xl2_full     fp16    0.19   0.04      0.0125 / 0.0137         13.0 (heads swapped)       15.7 s  10.2 GiB
    t2v_full     fp16    0.20   0         0.0037 / 0.0036         14.5 (heads swapped)       31.9 s  24.7 GiB

No row needs K above 1.09, so the budget keeps training's K = 4, A = 1 and Z = 2^-10 (tests/sample_fp64.py BUDGET).
Over whole halves the native error is 0.55 to 0.6 of the 16-bit yardstick's, and equal to the FP8 recipe's.

The budget rejects, in every case and recipe where they apply: two heads' attention outputs swapped in the last spatial
block; the last frame missing from every temporal attention's keys (16-bit recipes); sample 1 given sample 0's timestep
(xl2_t); the CFG pair's labels swapped and guidance applied to all 2C channels instead of the first C (xl2_cfg); the
caption mask ignored and layer l reading layer l - 1's text K/V (LatteT2V); for a non-square grid the square table or one
interpolated to base_size grid_h; and with use_fp8 every token's e4m3 activations scaled back with the next token's scale
(3.3 to 5.2 x the budget) or the weight scale dropped on the last 32 output channels (44 to 59 x).

Reported, not asserted:
  * With use_fp8 the last frame missing from the temporal keys sits at 0.96 to 1.13 x the budget: the e4m3 recipe's own
    error is as large as that defect.  The temporal attention is the same 16-bit kernel with and without use_fp8, and
    the 16-bit recipes of the same cases reject the defect at 1.36 x or more.
  * The last key of every spatial sequence dropped, at 576 and 640 tokens per frame: 0.23 to 0.54 x the budget, below
    what a whole-model yardstick can see.  test_gpu_t2v_res.py holds that kernel to fp64 element by element and rejects
    the defect there.
  * One token alone scaled back with its neighbour's scale is inside the e4m3 recipe's error (tests/sample_fp64.py)."""
import contextlib
import subprocess
import time

import pytest
import torch

import sample_fp64 as S
from oracle import latte_oracle as O
from oracle import t2v_oracle as T
from oracle import t2v_res_oracle as R

pytestmark = pytest.mark.gpu

LATTE1 = dict(num_attention_heads=16, attention_head_dim=72, sample_size=64, caption_channels=4096)
GEOMETRY = {
    "xl2_cfg": dict(patch=2, depth=4), "xl2_t": dict(patch=2, depth=4), "xl4": dict(patch=4, depth=4),
    "xl2_full": dict(patch=2, depth=28),
    "t2v_512": dict(hw=(64, 64), frames=16, layers=2), "t2v_320x512": dict(hw=(40, 64), frames=16, layers=2),
    "t2v_288x512": dict(hw=(36, 64), frames=16, layers=2), "t2v_t2i": dict(hw=(64, 64), frames=1, layers=2),
    "t2v_full": dict(hw=(64, 64), frames=16, layers=28),
}
RECIPES = {"xl2_cfg": ["fp16", "bf16", "half", "fp8"], "xl2_t": ["fp16", "bf16"], "xl4": ["fp16", "bf16"],
           "t2v_512": ["fp16", "bf16", "half", "fp8"], "t2v_320x512": ["fp16", "bf16", "fp8"],
           "t2v_288x512": ["fp16", "bf16", "fp8"], "t2v_t2i": ["fp16", "bf16"], "xl2_full": ["fp16"], "t2v_full": ["fp16"]}
PAIRS = [(c, r) for c, rs in RECIPES.items() for r in rs]
AUTOCAST = {"fp16": torch.float16, "bf16": torch.bfloat16, "half": torch.float16}
CFG_SCALE = 4.0


@pytest.fixture(scope="module")
def dev():
    d = torch.device("cuda:0")
    torch.empty(0, device=d)                           # initialise CUDA before the memory statistics are reset
    return d


@pytest.fixture(scope="module", autouse=True)
def _card():
    t0 = time.perf_counter()
    yield
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        card = torch.cuda.get_device_name(0)
    print(f"\n{card}: the file took {time.perf_counter() - t0:.0f} s")


class Case:
    """The module in the recipe on `dev`, its inputs, and `oracle(dtype, ...)` on its own weights and inputs."""

    def __init__(self, name, recipe, dev):
        from latte_b200 import Latte, LatteT2V
        geo = GEOMETRY[name]
        g = torch.Generator().manual_seed(sum(map(ord, name)))
        self.name, self.dev = name, dev
        self.cfg_scale = None
        if name.startswith("xl"):
            self.kind, self.p, self.cf = "latte", geo["patch"], False
            self.cfg = O.LatteConfig(input_size=32, patch_size=geo["patch"], hidden_size=1152, depth=geo["depth"], num_heads=16,
                                     num_frames=16)
            self.m = Latte(input_size=32, patch_size=geo["patch"], hidden_size=1152, depth=geo["depth"], num_heads=16,
                           num_frames=16, num_classes=101, extras=2)
            self.m.load_state_dict(O.make_weights(self.cfg, 31), strict=True)
            x = torch.randn(2, 16, 4, 32, 32, generator=g)
            if name == "xl2_t":
                self.t, self.y = torch.tensor([0, 999]), torch.tensor([3, 57])
            elif name == "xl4":
                self.t, self.y = torch.tensor([250, 750]), torch.tensor([3, 57])
            else:                                      # a CFG pair: one latent, (label, null) at one timestep
                x[1] = x[0]
                self.t, self.y = torch.tensor([400, 400]), torch.tensor([3, self.cfg.num_classes])
                self.cfg_scale = CFG_SCALE
            self.y = self.y.to(dev)
            self.last_spatial = f"blocks.{geo['depth'] - 2}.attn."
            self.tokens, self.frames = self.cfg.num_patches, 16
        else:
            self.kind, self.p, self.cf = "t2v", 2, True
            H, W = geo["hw"]
            self.cfg = T.T2VConfig(**LATTE1, num_layers=geo["layers"], video_length=geo["frames"])
            self.m = LatteT2V(**LATTE1, num_layers=geo["layers"], video_length=geo["frames"])
            self.m.load_state_dict(T.make_weights(self.cfg, 33), strict=True)
            x, _, text = R.make_inputs(self.cfg, 2, 120, 34, H, W)
            x[1] = x[0]                                # a CFG pair: sample 1's caption is the 12-token negative prompt
            self.t = torch.tensor([400, 400])
            self.text = text.to(dev)
            self.mask = torch.ones(2, 120, device=dev)
            self.mask[1, 12:] = 0
            self.last_spatial = f"transformer_blocks.{geo['layers'] - 1}.attn1"
            self.tokens, self.frames = (H // 2) * (W // 2), geo["frames"]
            self.grid = (H // 2, W // 2)
        self.x, self.t = x.to(dev), self.t.to(dev)
        if recipe == "half":
            self.m.half()
        elif recipe == "bf16":
            self.m.compute_dtype = torch.bfloat16
        self.m.use_fp8 = recipe == "fp8"
        self.m = self.m.to(dev).eval()
        self._sd = {}

    def native(self, **kw):
        with torch.no_grad():
            if self.kind == "latte":
                if self.cfg_scale is not None:
                    return self.m.forward_with_cfg(self.x, self.t, y=self.y, cfg_scale=self.cfg_scale, **kw)
                return self.m(self.x, self.t, y=self.y, **kw)
            return self.m(self.x, self.t, encoder_hidden_states=self.text, encoder_attention_mask=self.mask, return_dict=False)[0]

    def sd(self, dtype):
        if dtype not in self._sd:
            self._sd[dtype] = {k: v.detach().to(self.dev, dtype) for k, v in self.m.state_dict().items() if v.is_floating_point()}
        return self._sd[dtype]

    def oracle(self, dtype=torch.float64, autocast=None, **kw):
        """The oracle's output; kw: t, y, mask (None: ignored) or guided (channels guidance is applied to)."""
        ctx = torch.autocast("cuda", dtype=autocast) if autocast is not None else contextlib.nullcontext()
        with torch.no_grad(), ctx:
            if self.kind == "latte":
                return S.latte_out(self.sd(dtype), self.cfg, self.x, kw.get("t", self.t), kw.get("y", self.y), dtype,
                                   self.cfg_scale, kw.get("guided"))
            return S.t2v_out(self.sd(dtype), self.cfg, self.x, self.t, self.text, kw["mask"] if "mask" in kw else self.mask,
                             dtype)

    def edited(self, **kw):
        with S.edits(**kw):
            return self.oracle()


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


def _rejections(c, recipe, oac):
    """(what, wrong fp64 output, the output it modifies) for every defect that applies to the case and recipe."""
    out = [(f"heads 0 and 1 swapped in {c.last_spatial}", lambda: c.edited(core=S.swap_heads(c.last_spatial)), None)]
    if c.frames > 1 and recipe != "fp8":
        out.append(("the last frame missing from the temporal keys", lambda: c.edited(core=S.drop_last_key(S.is_temporal)), None))
    if c.name == "xl2_t":
        out.append(("sample 1 given sample 0's timestep", lambda: c.oracle(t=c.t[[0, 0]]), None))
    if c.cfg_scale is not None:
        out.append(("the CFG pair's labels swapped", lambda: c.oracle(y=c.y.flip(0)), None))
        out.append(("guidance on all 2C channels", lambda: c.oracle(guided=2 * c.cfg.in_channels), None))
    if c.kind == "t2v":
        out.append(("the caption mask ignored", lambda: c.oracle(mask=None), None))
        out.append(("layer l reading layer l - 1's text K/V", lambda: c.edited(kv_prefix=S.previous_layer_text_kv), None))
        if c.grid[0] != c.grid[1]:
            for what, fn in (("the square position table", S.square_table), ("a table interpolated to base_size grid_h",
                                                                             S.other_base_table)):
                def wrong(fn=fn):
                    with S.pos_table(fn):
                        return c.oracle()
                out.append((what, wrong, None))
    if recipe == "fp8":
        out.append(("every token scaled back with the next token's scale", lambda: c.edited(lin=S.fp8_recipe("token")), oac))
        out.append(("w_scale dropped on the last 32 output channels", lambda: c.edited(lin=S.fp8_recipe("w_scale")), oac))
    return out


@pytest.mark.parametrize("case,recipe", PAIRS)
def test_sample_within_fp64_budget(dev, case, recipe):
    t0 = time.perf_counter()
    torch.cuda.reset_peak_memory_stats(dev)
    c = Case(case, recipe, dev)
    outs = [c.native() for _ in range(3)]
    assert all(torch.equal(o, outs[0]) for o in outs[1:]), "eager, captured and replayed outputs differ"
    got = outs[2]
    assert got.dtype == (torch.float16 if recipe == "half" else torch.float32)
    if c.cfg_scale is not None and c.kind == "latte":
        c.m.precompute_conditioning(c.t.view(1, -1), c.y)
        traj = c.native(trajectory_step=0)
        c.m.clear_conditioning()
        assert torch.equal(traj, got), "trajectory conditioning changed the output"
    o64 = c.oracle()
    if recipe == "fp8":
        oac = c.edited(lin=S.fp8_recipe())
    else:
        oac = c.oracle(torch.float32, autocast=AUTOCAST[recipe])
    budget = S.BUDGET[recipe]
    res = S.check(got, o64, oac, budget, c.p, c.cf)
    rows = {h: S.out_rows(v, c.p, c.cf) for h, v in (("got", got), ("o64", o64), ("oac", oac))}
    print(f"\n{case} {recipe}: K, A, Z = {budget[0]:g}, {budget[1]:g}, {budget[2]:.3g}")
    for h, w in res.items():
        print(f"    {h}: worst row {w.row} at {w.ratio:.3g} x its budget, largest K a row needs {max(w.need_k, 0.0):.3g}; that row |err| "
              f"{w.e:.3g}, a {w.a:.3g}, |o64| {w.r:.3g}; whole half: native {_rel(rows['got'][h], rows['o64'][h]):.3g}, "
              f"yardstick {_rel(rows['oac'][h], rows['o64'][h]):.3g} of |o64|")
    missed = []
    for what, wrong, base in _rejections(c, recipe, oac):
        w = S.rejected(got, o64, oac, wrong(), o64 if base is None else base, budget, c.p, c.cf)
        print(f"    rejects {what}: row {w.row} at {w.ratio:.3g} x its budget")
        if not w.ratio > 1.0:
            missed.append((what, w.ratio))
    unasserted = []
    if c.kind == "t2v" and c.tokens in (576, 640):
        unasserted.append(("the last key of every spatial sequence dropped", S.drop_last_key(S.is_spatial_self)))
    if c.frames > 1 and recipe == "fp8":
        unasserted.append(("the last frame missing from the temporal keys", S.drop_last_key(S.is_temporal)))
    for what, core in unasserted:
        w = S.rejected(got, o64, oac, c.edited(core=core), o64, budget, c.p, c.cf)
        print(f"    (not asserted) {what}: {w.ratio:.3g} x the budget")
    print(f"    {time.perf_counter() - t0:.1f} s, peak {torch.cuda.max_memory_allocated(dev) / 2 ** 30:.1f} GiB")
    assert max(w.ratio for w in res.values()) <= 1.0, res
    assert not missed, missed
