"""CPU: LatteT2V's attention cache (Pyramid Attention Broadcast) without a GPU -- the config checks of `enable_cache`, the
schedule `_pab_plan` runs before each cached forward (compute / store / reuse per kind, resets, the timestep it reads),
the buffers it sizes, the refusals of `b200_t2v_forward_cached` that precede any launch, and the oracle restatement the
GPU tests compare against."""
import copy
import ctypes as C
import io

import pytest
import torch

import pab_oracle as P
from latte_b200 import LatteT2V, PyramidAttentionBroadcastConfig, _lib

TINY = dict(num_attention_heads=2, attention_head_dim=64, num_layers=2, sample_size=16, video_length=8, caption_channels=256)
KINDS = ("spatial", "temporal", "cross")
# the measured workload: 50 timesteps 981, 961, ..., 1; ranges 2 / 4 / 6; windows (100, 800) / (100, 800) / (100, 900)
TAUS = list(range(981, 0, -20))
PAB = dict(spatial_attention_block_skip_range=2, temporal_attention_block_skip_range=4, cross_attention_block_skip_range=6,
           cross_attention_timestep_skip_range=(100, 900))


def _net(**cfg):
    return LatteT2V(**{**TINY, **cfg}).eval()


def _call(net, tau, text, batch=2, hw=(16, 16), temporal=True, mask=None, od=torch.float16, dev="cpu", t=None):
    """The modes of one planned call: {kind: _lib.CACHE_*}."""
    hs = torch.zeros(batch, 4, net.config.video_length, *hw, device=dev)
    ts = torch.full((batch,), tau) if t is None else t
    cache = net._pab_plan(hs, ts, text, mask, temporal, od)
    return {k: getattr(cache, k + "_mode") for k in KINDS}


def _text(batch=2, L=20, dev="cpu"):
    return torch.zeros(batch, L, TINY["caption_channels"], device=dev)


@pytest.mark.parametrize("field,value", [
    ("spatial_attention_block_skip_range", 0), ("temporal_attention_block_skip_range", -2),
    ("cross_attention_block_skip_range", 1.5), ("spatial_attention_block_skip_range", True),
    ("cross_attention_block_skip_range", "2"), ("spatial_attention_timestep_skip_range", (800, 100)),
    ("temporal_attention_timestep_skip_range", (1, 2, 3)), ("cross_attention_timestep_skip_range", None),
    ("current_timestep_callback", 5),
])
def test_invalid_config_is_refused(field, value):
    net = _net()
    with pytest.raises(ValueError):
        net.enable_cache(PyramidAttentionBroadcastConfig(**{field: value}))
    assert not net.is_cache_enabled


def test_config_is_read_by_field_name():
    """Any object with diffusers' field names works (here a plain namespace); fields it lacks take the defaults."""
    from types import SimpleNamespace
    net = _net()
    assert not net.is_cache_enabled
    net.enable_cache(SimpleNamespace(spatial_attention_block_skip_range=3, spatial_attention_block_identifiers=["x"]))
    assert net.is_cache_enabled
    rules, cb = net._pab
    assert rules["spatial"] == (3, (100.0, 800.0)) and rules["temporal"][0] is None and cb is None
    net.disable_cache()
    assert not net.is_cache_enabled


def test_fifty_step_pattern_and_counts():
    net = _net()
    net.enable_cache(PyramidAttentionBroadcastConfig(**PAB))
    text = _text()
    got = [_call(net, tau, text) for tau in TAUS]
    want = P.schedule(TAUS, {"spatial": 2, "temporal": 4, "cross": 6},
                      {"spatial": (100, 800), "temporal": (100, 800), "cross": (100, 900)})
    assert got == want
    reused = {k: sum(m[k] == _lib.CACHE_REUSE for m in got) for k in KINDS}
    assert reused == {"spatial": 17, "temporal": 26, "cross": 33}
    assert all(got[0][k] == _lib.CACHE_STORE for k in KINDS)
    # outside the windows every call computes: 981..801 and 81..1 (cross: 981..901 and 81..1)
    assert all(m["spatial"] == _lib.CACHE_STORE for tau, m in zip(TAUS, got) if not 100 < tau < 800)
    assert all(m["cross"] == _lib.CACHE_STORE for tau, m in zip(TAUS, got) if not 100 < tau < 900)


def test_range_one_and_none():
    net = _net()
    net.enable_cache(PyramidAttentionBroadcastConfig(spatial_attention_block_skip_range=1))
    text = _text()
    modes = [_call(net, tau, text) for tau in (700, 600, 500)]
    assert all(m == {"spatial": _lib.CACHE_STORE, "temporal": _lib.CACHE_COMPUTE, "cross": _lib.CACHE_COMPUTE} for m in modes)
    assert set(net._pab_state.buffers) == {"spatial"}


def _reused_after_reset(net, base_text, **kw):
    """Two calls at 700 and 600 (range 2: store, reuse), then one call with `kw`: STORE if it started a new trajectory."""
    assert _call(net, 700, base_text)["spatial"] == _lib.CACHE_STORE
    assert _call(net, 600, base_text)["spatial"] == _lib.CACHE_REUSE
    return _call(net, kw.pop("tau", 500), kw.pop("text", base_text), **kw)["spatial"]


@pytest.mark.parametrize("change", ["none", "rising", "equal", "batch", "hw", "text_len", "text_object", "text_inplace",
                                    "mask", "dtype", "fp8", "temporal"])
def test_resets(change):
    net = _net()
    net.enable_cache(PyramidAttentionBroadcastConfig(spatial_attention_block_skip_range=2))
    text = _text()
    kw = {"none": dict(tau=500), "rising": dict(tau=650), "equal": dict(tau=600), "batch": dict(batch=4, text=_text(4)),
          "hw": dict(hw=(16, 32)), "text_len": dict(text=_text(L=30)), "text_object": dict(text=text.clone()),
          "mask": dict(mask=torch.ones(2, 20)), "dtype": dict(od=torch.bfloat16), "temporal": dict(temporal=False),
          "text_inplace": {}, "fp8": {}}[change]
    if change == "text_inplace":
        _call(net, 700, text)
        _call(net, 600, text)
        text.add_(1.0)           # a new version of the same caption tensor
        assert _call(net, 500, text)["spatial"] == _lib.CACHE_STORE
        return
    if change == "fp8":
        _call(net, 700, text)
        _call(net, 600, text)
        net.use_fp8 = True
        assert _call(net, 500, text)["spatial"] == _lib.CACHE_STORE
        return
    # call 3 of an unchanged trajectory (i = 2, 2 % 2 == 0) stores too, so look at call 4 instead
    first = _reused_after_reset(net, text, **kw)
    if change == "none":
        assert first == _lib.CACHE_STORE and _call(net, 400, text)["spatial"] == _lib.CACHE_REUSE
    else:
        assert first == _lib.CACHE_STORE
        assert net._pab_state.calls["spatial"] == 1, "the call did not start a new trajectory"


def test_enable_and_disable_reset():
    net = _net()
    cfg = PyramidAttentionBroadcastConfig(spatial_attention_block_skip_range=2)
    net.enable_cache(cfg)
    text = _text()
    _call(net, 700, text)
    assert _call(net, 600, text)["spatial"] == _lib.CACHE_REUSE
    net.enable_cache(cfg)
    assert net._pab_state is None
    assert _call(net, 500, text)["spatial"] == _lib.CACHE_STORE
    net.disable_cache()
    assert net._pab_state is None and not net.is_cache_enabled


def test_callback_takes_precedence():
    taus = iter([700, 600])
    net = _net()
    net.enable_cache(PyramidAttentionBroadcastConfig(spatial_attention_block_skip_range=2,
                                                     current_timestep_callback=lambda: next(taus)))
    text = _text()
    mixed = torch.tensor([999, 3])          # would be refused without the callback, and 999 / 3 lie outside the window
    assert _call(net, 0, text, t=mixed)["spatial"] == _lib.CACHE_STORE
    assert _call(net, 0, text, t=mixed)["spatial"] == _lib.CACHE_REUSE
    assert net._pab_state.prev_tau == 600


def test_mixed_timesteps_are_refused():
    net = _net()
    net.enable_cache(PyramidAttentionBroadcastConfig(spatial_attention_block_skip_range=2))
    with pytest.raises(ValueError, match="one timestep"):
        _call(net, 0, _text(), t=torch.tensor([500, 400]))
    # one value for all samples, given once or per sample
    assert _call(net, 0, _text(), t=torch.tensor(500))["spatial"] == _lib.CACHE_STORE


def test_cache_bytes():
    net = _net()
    net.enable_cache(PyramidAttentionBroadcastConfig(spatial_attention_block_skip_range=2, cross_attention_block_skip_range=3))
    _call(net, 500, _text(), od=torch.bfloat16)
    T = 2 * 8 * 8 * 8                       # batch x frames x (16 / 2)^2 patches
    bufs = net._pab_state.buffers
    assert set(bufs) == {"spatial", "cross"}
    for b in bufs.values():
        assert b.dtype == torch.bfloat16 and tuple(b.shape) == (2, T, 128) and b.numel() * b.element_size() == 2 * T * 128 * 2


def test_latte1_cache_bytes():
    """Latte-1 at 16 x 512 x 512 with a CFG pair: 3 x 28 x 32768 x 1152 x 2 bytes = 6.3 GB (shapes only, on the meta device)."""
    with torch.device("meta"):
        net = LatteT2V(num_layers=28, caption_channels=256).eval()
    taus = iter([500])
    net.enable_cache(PyramidAttentionBroadcastConfig(**{f"{k}_attention_block_skip_range": 2 for k in KINDS},
                                                     current_timestep_callback=lambda: next(taus)))
    hs = torch.empty(2, 4, 16, 64, 64, device="meta")
    net._pab_plan(hs, None, torch.empty(2, 120, 256, device="meta"), None, True, torch.float16)
    total = sum(b.numel() * b.element_size() for b in net._pab_state.buffers.values())
    assert total == 3 * 28 * 32768 * 1152 * 2
    assert round(total / 1e9, 1) == 6.3


def test_copies_keep_the_config_and_drop_the_buffers():
    net = _net()
    net.enable_cache(PyramidAttentionBroadcastConfig(spatial_attention_block_skip_range=2))
    _call(net, 500, _text())
    assert net._pab_state.buffers
    for other in (copy.deepcopy(net), _saved(net)):
        assert other.is_cache_enabled and other._pab_state is None
    assert net._pab_state.buffers            # the original keeps its own


def _saved(net):
    f = io.BytesIO()
    torch.save(net, f)
    f.seek(0)
    return torch.load(f, weights_only=False)


def _fake_call(lib, cache):
    """b200_t2v_forward_cached on a valid tiny shape with placeholder addresses: only checks that precede any launch."""
    shape = _lib.T2VShape(layers=2, hidden=128, heads=2, mlp_hidden=512, patch=2, in_channels=4, out_channels=8,
                          input_size=16, frames=8, caption_channels=256, dtype=_lib.FP16, input_width=0)
    w = _lib.T2VWeights()
    p = 1 << 20                              # 1024-byte aligned placeholder; never dereferenced
    return lib.b200_t2v_forward_cached(C.byref(shape), C.byref(w), p, p, p, None, 2, 20, 1, C.byref(cache), p, p, 1 << 30, None)


@pytest.mark.parametrize("bad,code,text", [
    (dict(spatial_mode=2), "SHAPE", "spatial cache mode 2 needs a buffer"),
    (dict(temporal_mode=1), "SHAPE", "temporal cache mode 1 needs a buffer"),
    (dict(cross=1 << 20, cross_mode=3), "SHAPE", "cross cache mode 3 is not 0, 1 or 2"),
    (dict(spatial=1 << 20, spatial_mode=-1), "SHAPE", "spatial cache mode -1"),
    (dict(temporal=(1 << 20) + 8, temporal_mode=2), "ALIGN", "temporal cache buffer must be 16-byte aligned"),
])
def test_c_refuses_bad_cache_before_launching(bad, code, text):
    """Checked before the architecture, so the refusal is the same with or without a GPU."""
    lib = _lib.load()
    rc = _fake_call(lib, _lib.T2VCache(**bad))
    assert _lib.ERR_NAMES.get(rc) == code and text in _lib.last_error(), (rc, _lib.last_error())


def test_oracle_forward_without_overrides_is_the_t2v_oracle():
    from oracle import t2v_oracle as T
    cfg = T.T2VConfig(**TINY)
    sd = T.make_weights(cfg, 3)
    x, t, text = T.make_inputs(cfg, 2, 20, 4)
    ref = T.t2v_forward(sd, cfg, x, t, text)
    out, used = P.forward(sd, cfg, x, t, text)
    assert torch.allclose(out, ref, atol=1e-5, rtol=0)
    assert all(tuple(used[k].shape) == (2, 2 * 8 * 64, 128) for k in KINDS)
    # feeding the outputs back in changes nothing
    again, _ = P.forward(sd, cfg, x, t, text, attn=used)
    assert torch.allclose(again, out, atol=1e-5, rtol=0)
