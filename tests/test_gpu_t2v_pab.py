"""GPU: LatteT2V's attention cache (Pyramid Attention Broadcast, `enable_cache`) against the CPU restatement in
tests/pab_oracle.py.

- Cache off, or every skip range None, is bit-identical to the plain forward.  So is a store step at these shapes: the
  out-projections' K (= D) is below the length the residual GEMM splits along K, so the whole-K store epilogue adds the
  same sums.
- A store step is within the T2V oracle's tolerances (1e-2 max-abs with fp16 operands, 8e-2 with bf16), every cached
  layer matches the oracle's pre-gate attention outputs within the same bound scaled by their magnitude, and reruns are
  bit-identical.
- A reuse step equals the oracle forward at that step with the reused outputs replaced by the GPU cache contents.
- A 12-call trajectory follows the schedule launch by launch (the library's profiler) and output by output.
- A non-square ragged grid, video_length 1, enable_temporal_attentions=False, a padded-prompt mask and FP8 operands each
  run a store and a reuse step.  FP8 is held, as in tests/test_gpu_fp8_t2v.py, to FP8_TOL_FACTOR = 6 units of a bf16
  deviation: here the oracle's own, run in bf16 on the same weights, inputs and reused outputs."""
import ctypes as C

import pytest
import torch

import pab_oracle as P
from latte_b200 import LatteT2V, PyramidAttentionBroadcastConfig, _lib
from oracle import t2v_oracle as T
from oracle import t2v_res_oracle as R

pytestmark = pytest.mark.gpu

TINY = dict(num_attention_heads=2, attention_head_dim=64, num_layers=2, sample_size=16, video_length=8, caption_channels=256)
# Latte-1's layer geometry (16 heads x 72, caption_channels 4096) at two layers and 8 x 256 x 256 px
LATTE1 = dict(num_attention_heads=16, attention_head_dim=72, num_layers=2, sample_size=32, video_length=8, caption_channels=4096)
TOL = {torch.float16: 1e-2, torch.bfloat16: 8e-2}
FP8_TOL_FACTOR = 6.0


def _pab(kinds=P.KINDS, r=2, **kw):
    return PyramidAttentionBroadcastConfig(**{f"{k}_attention_block_skip_range": r for k in kinds}, **kw)


class Case:
    """One seeded model on the GPU and the oracle beside it."""

    def __init__(self, cfg_kw, batch=2, text_len=20, seed=0, hw=None, dtype=torch.float16, masked=False):
        self.cfg = T.T2VConfig(**cfg_kw)
        self.sd = T.make_weights(self.cfg, seed)
        H, W = hw or (self.cfg.sample_size, self.cfg.sample_size)
        self.x, _, self.text = R.make_inputs(self.cfg, batch, text_len, seed + 1, H, W)
        self.batch, self.dtype = batch, dtype
        self.mask = None
        if masked:
            self.mask = torch.ones(batch, text_len)
            self.mask[0, text_len // 2:] = 0
        net = LatteT2V(**cfg_kw)
        net.load_state_dict(self.sd, strict=True)
        self.net = net.to(device="cuda", dtype=torch.bfloat16 if dtype == torch.bfloat16 else torch.float32).eval()
        # one caption tensor (and mask) for the whole trajectory: a new object starts a new one
        self.text_d = self.text.cuda()
        self.mask_d = self.mask.cuda() if masked else None

    def x_at(self, k):
        """The latent of call k: a fixed, output-independent sequence, so GPU and oracle see the same inputs."""
        return self.x * (1.0 - 0.03 * k)

    def run(self, x, tau, temporal=True):
        with torch.no_grad():
            t = torch.full((self.batch,), int(tau), dtype=torch.int64, device="cuda")
            out = self.net(x.cuda(), t, encoder_hidden_states=self.text_d, encoder_attention_mask=self.mask_d,
                           enable_temporal_attentions=temporal, return_dict=False)[0]
        return out.float().cpu()

    def oracle(self, x, tau, temporal=True, attn=None, dtype=torch.float32):
        t = torch.full((self.batch,), int(tau), dtype=torch.int64)
        out, pre = P.forward(self.sd, self.cfg, x, t, self.text, dtype=dtype, enable_temporal=temporal, text_mask=self.mask,
                             attn=attn)
        return out.float(), pre

    def cache(self, kind):
        return self.net._pab_state.buffers[kind].float().cpu()


def _err(a, b):
    return (a - b).abs().max().item()


def test_cache_off_and_every_range_none_are_bit_identical():
    c = Case(TINY)
    plain = [c.run(c.x_at(k), tau) for k, tau in enumerate((700, 600))]
    c.net.enable_cache(PyramidAttentionBroadcastConfig())
    assert c.net.is_cache_enabled
    assert all(torch.equal(c.run(c.x_at(k), tau), p) for k, (tau, p) in enumerate(zip((700, 600), plain)))
    assert not c.net._pab_state.buffers
    c.net.disable_cache()
    assert torch.equal(c.run(c.x_at(0), 700), plain[0])


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
def test_store_step(dtype):
    c = Case(TINY, dtype=dtype)
    plain = c.run(c.x, 500)
    c.net.enable_cache(_pab())
    out = c.run(c.x, 500)
    assert c.net._pab_state.last_modes == {k: _lib.CACHE_STORE for k in P.KINDS}
    assert torch.equal(out, plain)
    ref, pre = c.oracle(c.x, 500)
    assert _err(out, ref) < TOL[dtype], f"max-abs {_err(out, ref):.3e} vs the oracle"
    caches = {k: c.cache(k) for k in P.KINDS}
    for k in P.KINDS:
        scale = max(1.0, pre[k].abs().max().item())
        assert _err(caches[k], pre[k]) < TOL[dtype] * scale, f"{k}: {_err(caches[k], pre[k]):.3e} (scale {scale:.2f})"
    c.net.enable_cache(_pab())                  # a new trajectory: the same store step again
    assert torch.equal(c.run(c.x, 500), out)
    assert all(torch.equal(c.cache(k), caches[k]) for k in P.KINDS)


@pytest.fixture(scope="module")
def cases():
    return {}


@pytest.mark.parametrize("geom", ["tiny", "latte1"])
@pytest.mark.parametrize("kinds", [("spatial",), ("temporal",), ("cross",), P.KINDS], ids=["spatial", "temporal", "cross", "all"])
def test_reuse_step(cases, geom, kinds):
    if geom not in cases:
        cases[geom] = Case(TINY) if geom == "tiny" else Case(LATTE1, text_len=120)
    c = cases[geom]
    c.net.enable_cache(_pab(kinds))
    c.run(c.x_at(0), 500)
    stored = {k: c.cache(k) for k in kinds}
    out = c.run(c.x_at(1), 480)
    modes = c.net._pab_state.last_modes
    assert modes == {k: _lib.CACHE_REUSE if k in kinds else _lib.CACHE_COMPUTE for k in P.KINDS}
    assert all(torch.equal(c.cache(k), stored[k]) for k in kinds), "a reuse step wrote its cache"
    ref, _ = c.oracle(c.x_at(1), 480, attn=stored)
    assert _err(out, ref) < TOL[torch.float16], f"{geom} {kinds}: max-abs {_err(out, ref):.3e}"
    c.net.disable_cache()


def _profile_counts(lib):
    ms = (C.c_double * 4)()
    n = (C.c_int * 4)()
    _lib.check(lib.b200_profile_collect(ms, n, 4), "b200_profile_collect")
    return list(n)          # gemm, attention, ln_modulate, other


def test_trajectory_follows_the_schedule():
    """12 calls from 950 down to 30 cross both edges of the (100, 800) windows; ranges 2 / 3 / 4."""
    taus = [950, 850, 790, 720, 650, 580, 500, 420, 300, 180, 95, 30]
    ranges = {"spatial": 2, "temporal": 3, "cross": 4}
    windows = {k: (100, 800) for k in P.KINDS}
    c = Case(TINY)
    L = c.cfg.num_layers
    lib = _lib.load()
    _lib.profile_enable(True)
    try:
        _profile_counts(lib)
        c.run(c.x, 990)
        g0, a0, n0, o0 = _profile_counts(lib)
        c.net.enable_cache(PyramidAttentionBroadcastConfig(**{f"{k}_attention_block_skip_range": r for k, r in ranges.items()}))
        outs, modes = [], []
        for k, tau in enumerate(taus):
            outs.append(c.run(c.x_at(k), tau))
            m = dict(c.net._pab_state.last_modes)
            modes.append(m)
            sp, tm, cr = (int(m[k2] == _lib.CACHE_REUSE) for k2 in P.KINDS)
            want = [g0 - L * 2 * (sp + tm + cr) - 3 * cr, a0 - L * (sp + tm + cr), n0 - L * (sp + tm), o0 + L * (sp + tm) - cr]
            assert _profile_counts(lib) == want, f"call {k} (t = {tau}, modes {m})"
    finally:
        _lib.profile_enable(False)
    assert modes == P.schedule(taus, ranges, windows)
    assert sum(m[k] == _lib.CACHE_REUSE for m in modes for k in P.KINDS) > 0
    refs = P.trajectory(c.sd, c.cfg, [c.x_at(k) for k in range(len(taus))], taus, c.text, ranges, windows)
    errs = [_err(o, r) for o, r in zip(outs, refs)]
    assert max(errs) < TOL[torch.float16], f"per-call max-abs {['%.2e' % e for e in errs]}"


VARIANTS = {
    "fp8": dict(cfg=TINY),
    "ragged": dict(cfg=TINY, hw=(20, 32)),                 # 10 x 16 patches per frame, interpolated position table
    "frames1": dict(cfg={**TINY, "sample_size": 32, "video_length": 1}),
    "notemporal": dict(cfg=TINY, temporal=False),
    "masked": dict(cfg=TINY, masked=True),
}


@pytest.mark.parametrize("name", list(VARIANTS))
def test_variant_store_and_reuse(name):
    v = VARIANTS[name]
    c = Case(v["cfg"], hw=v.get("hw"), masked=v.get("masked", False))
    temporal = v.get("temporal", True)
    fp8 = name == "fp8"
    c.net.use_fp8 = fp8

    def check(step, out, ref, **oracle_kw):
        tol = TOL[torch.float16]
        if fp8:
            unit = _err(ref, c.oracle(dtype=torch.bfloat16, **oracle_kw)[0])
            tol = FP8_TOL_FACTOR * unit
            print(f"\nfp8 {step} step: max-abs {_err(out, ref):.3e} = {_err(out, ref) / unit:.2f} x the oracle's bf16 "
                  f"deviation {unit:.3e}")
        assert _err(out, ref) < tol, f"{name} {step} step: max-abs {_err(out, ref):.3e} (tolerance {tol:.3e})"

    plain = c.run(c.x_at(0), 500, temporal)
    c.net.enable_cache(_pab())
    out0 = c.run(c.x_at(0), 500, temporal)
    assert torch.equal(out0, plain)
    check("store", out0, c.oracle(c.x_at(0), 500, temporal)[0], x=c.x_at(0), tau=500, temporal=temporal)
    kinds = P.KINDS if temporal else ("spatial", "cross")
    stored = {k: c.cache(k) for k in kinds}
    out1 = c.run(c.x_at(1), 480, temporal)
    want = {k: _lib.CACHE_REUSE if k in kinds else _lib.CACHE_COMPUTE for k in P.KINDS}
    assert c.net._pab_state.last_modes == want
    check("reuse", out1, c.oracle(c.x_at(1), 480, temporal, attn=stored)[0], x=c.x_at(1), tau=480, temporal=temporal,
          attn=stored)


def test_disable_cache_returns_the_cache_bytes():
    c = Case(TINY)
    c.run(c.x, 500)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    c.net.enable_cache(_pab())
    c.run(c.x, 500)
    torch.cuda.synchronize()
    T_rows = c.batch * c.cfg.video_length * (c.cfg.sample_size // 2) ** 2
    want = 3 * c.cfg.num_layers * T_rows * c.cfg.inner_dim * 2
    assert torch.cuda.memory_allocated() - base == want
    c.net.disable_cache()
    assert torch.cuda.memory_allocated() == base


def test_training_forward_refuses_before_launching():
    c = Case(TINY)
    c.net.train()
    c.net.enable_cache(_pab())
    lib = _lib.load()
    _lib.profile_enable(True)
    try:
        _profile_counts(lib)
        t = torch.full((c.batch,), 500, dtype=torch.int64, device="cuda")
        with pytest.raises(NotImplementedError, match="disable_cache"):
            c.net(c.x.cuda(), t, encoder_hidden_states=c.text_d)
        assert _profile_counts(lib) == [0, 0, 0, 0]
    finally:
        _lib.profile_enable(False)
