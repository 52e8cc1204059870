"""GPU: each layer of the VAE alone -- the implicit-GEMM convolutions (3x3, temporal (3,1,1), stride-2 Downsample2D), the
"+ shortcut" epilogue, GroupNorm (+ SiLU) and the mid-block attention -- through its C-ABI entry point, against the torch op
in fp64 on the same 16-bit-rounded inputs and weights, with the weights packed by the product's own packers (latte_b200/vae.py).

Random-data cases allow one 16-bit rounding of the output (fp16 4e-3, bf16 3e-2, abs + rel, as in test_gpu_ops.py).  The
"delta" cases use small integers, exact in 16 bits and in fp32 sums, on images that are zero except for single pixels at the
corners, edge midpoints, tile seams and one interior point: the result must equal the reference bit for bit, and a wrong tap
offset or a missing zero-fill at a border names the pixels it changes.  The end-to-end test_gpu_vae.py cannot see such errors:
they touch under 1 % of a feature map."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]
TOL = {torch.float16: 4e-3, torch.bfloat16: 3e-2}
DEV = torch.device("cuda:0")


def _close(got, ref, tol, what):
    """|got - ref| <= tol * (1 + |ref|) everywhere; ref is fp64.  Prints the worst error for the record."""
    assert got.shape == ref.shape, (got.shape, ref.shape)
    assert not torch.isnan(got).any(), f"{what}: NaN in the output"
    err = (got.double() - ref).abs()
    ratio = (err / (tol * (1 + ref.abs()))).max().item()
    print(f"[vae-ops] {what}: max abs err {err.max().item():.3e}, worst err / tol(1 + |ref|) = {ratio:.3f}")
    bad = (err > tol + tol * ref.abs()).nonzero()
    assert bad.shape[0] == 0, (f"{what}: {bad.shape[0]} elements outside tol {tol}, max err {err.max().item():.3e}; "
                               f"first (index..., channel): {bad[:6].tolist()}")


def _equal(got, ref, what):
    """Bit-exact comparison of an NHWC 16-bit output with an fp64 reference that is exactly representable; on failure the
    message names the (image, y, x) pixels that differ."""
    want = ref.to(got.dtype)
    assert torch.equal(ref, want.double()), f"{what}: the reference is not exact in 16 bits (test data too large)"
    diff = (got != want).any(dim=-1).nonzero().tolist()
    assert not diff, f"{what}: {len(diff)} pixels differ from the reference, (image, y, x): {diff[:12]}"


def _randn(gen, *shape, scale=1.0):
    return torch.randn(*shape, generator=gen) * scale


def _ints(gen, lo, hi, *shape):
    return torch.randint(lo, hi + 1, shape, generator=gen).float()


def _edge_points(h, w):
    """Corners, edge midpoints, one interior pixel, and the pixels on both sides of the 128-pixel tile seams."""
    pts = {(0, 0), (0, w - 1), (h - 1, 0), (h - 1, w - 1), (0, w // 2), (h - 1, w // 2), (h // 2, 0), (h // 2, w - 1), (h // 2, w // 2 + 1)}
    if w >= 128:
        for x0 in range(128, w, 128):                      # seams inside a row
            pts |= {(h // 2, x0 - 1), (h // 2, x0)}
    else:
        bh = 128 // w                                      # packed-row tiles: seams between rows bh-1 and bh
        for y0 in range(bh, h, bh):
            pts |= {(y0 - 1, w // 3), (y0, w // 3)}
    return sorted(pts)


def _delta_input(gen, n, h, w, c, points, images=None):
    """Zero NHWC image except at `points` of `images`, each with 3 channels set to a small nonzero integer."""
    x = torch.zeros(n, h, w, c)
    for img in (range(n) if images is None else images):
        for (y, xx) in points:
            ch = torch.randperm(c, generator=gen)[:3]
            x[img, y, xx, ch] = _ints(gen, 1, 2, 3) * (1 - 2 * _ints(gen, 0, 1, 3))
    return x


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


def _nchw(t):
    return t.permute(0, 3, 1, 2)


# ------------------------------------------------------------------------------------------------------ 3x3 convolution
def _conv3x3_ref(x16, w16, bias, add16):
    ref = _nhwc(F.conv2d(_nchw(x16.double()), w16.double(), bias.double(), padding=1))
    return ref + add16.double() if add16 is not None else ref


def _conv3x3(x16, w16, bias, add16):
    from latte_b200 import ops, vae
    return ops.vae_conv(x16.contiguous(), vae.pack_conv3x3(w16).contiguous(), bias, "3x3", add16)


CONV_CASES = [
    # n, h, w, cin, cout, add16      conv_bh = 128 / w for w < 128; w >= 128: one row per 128-pixel tile
    (1, 16, 8, 64, 32, False),       # a single 128-row tile: the second CTA of the pair lies wholly past M; padded conv_out
    (3, 16, 8, 128, 64, True),
    (1, 16, 16, 512, 128, False),
    (3, 8, 16, 64, 256, True),       # 3 tiles (odd)
    (1, 8, 32, 128, 512, True),
    (3, 12, 32, 64, 64, False),
    (1, 6, 64, 512, 256, True),
    (3, 4, 64, 128, 32, False),
    (1, 7, 128, 64, 128, True),      # 7 tiles (odd)
    (3, 3, 128, 512, 512, False),
    (1, 5, 256, 128, 256, False),
    (3, 3, 256, 64, 512, True),
    (1, 2, 64, 256, 192, True),      # cout = 192: not a multiple of a 128- or 256-wide tile
]


@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("case", CONV_CASES, ids=lambda c: "n{}_{}x{}_ci{}_co{}{}".format(*c[:5], "_add" if c[5] else ""))
def test_conv3x3(dt, case):
    n, h, w, cin, cout, add = case
    g = torch.Generator().manual_seed(n * 7 + h * 131 + w * 17 + cin + cout)
    x = _randn(g, n, h, w, cin).to(DEV, dt)
    wt = _randn(g, cout, cin, 3, 3, scale=(9 * cin) ** -0.5).to(DEV, dt)
    bias = _randn(g, cout, scale=0.1).to(DEV)
    add16 = _randn(g, n, h, w, cout).to(DEV, dt) if add else None
    _close(_conv3x3(x, wt, bias, add16), _conv3x3_ref(x, wt, bias, add16), TOL[dt], f"conv3x3 {case} {dt}")


@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("case", [(2, 32, 8, 64, 32), (2, 16, 16, 128, 64), (2, 8, 32, 64, 64), (2, 4, 64, 64, 128),
                                  (2, 4, 128, 64, 32), (2, 3, 256, 128, 64)], ids=lambda c: "n{}_{}x{}_ci{}_co{}".format(*c))
def test_conv3x3_delta(dt, case):
    """Exact: single integer pixels at the borders and tile seams of two stacked images, integer weights, bias and shortcut."""
    n, h, w, cin, cout = case
    g = torch.Generator().manual_seed(h * 1000 + w)
    x = _delta_input(g, n, h, w, cin, _edge_points(h, w)).to(DEV, dt)
    wt = _ints(g, -3, 3, cout, cin, 3, 3).to(DEV, dt)
    bias = _ints(g, -2, 2, cout).to(DEV)
    add16 = _ints(g, -4, 4, n, h, w, cout).to(DEV, dt)
    _equal(_conv3x3(x, wt, bias, None), _conv3x3_ref(x, wt, bias, None), f"conv3x3 delta {case} {dt}")
    _equal(_conv3x3(x, wt, bias, add16), _conv3x3_ref(x, wt, bias, add16), f"conv3x3 delta + shortcut {case} {dt}")


# ------------------------------------------------------------------------------------------- temporal Conv3d (3,1,1)
def _conv_t3_ref(x16, w5, bias, add16):
    v = x16.double().permute(3, 0, 1, 2)[None]                        # [1, C, frames, h, w]
    ref = F.conv3d(v, w5.double(), bias.double(), padding=(1, 0, 0))[0].permute(1, 2, 3, 0)
    return ref + add16.double() if add16 is not None else ref


def _conv_t3(x16, w5, bias, add16):
    from latte_b200 import ops, vae
    return ops.vae_conv(x16.contiguous(), vae.pack_conv_t3(w5).to(x16.dtype).contiguous(), bias, "t3", add16)


@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("case", [(1, 16, 8, 128, True), (2, 8, 16, 64, False), (14, 16, 16, 128, True), (14, 4, 64, 512, False),
                                  (2, 2, 128, 256, True)], ids=lambda c: "f{}_{}x{}_c{}{}".format(*c[:4], "_add" if c[4] else ""))
def test_conv_t3(dt, case):
    frames, h, w, c, add = case
    g = torch.Generator().manual_seed(frames * 100 + h + w + c)
    x = _randn(g, frames, h, w, c).to(DEV, dt)
    w5 = _randn(g, c, c, 3, 1, 1, scale=(3 * c) ** -0.5).to(DEV, dt)
    bias = _randn(g, c, scale=0.1).to(DEV)
    add16 = _randn(g, frames, h, w, c).to(DEV, dt) if add else None
    _close(_conv_t3(x, w5, bias, add16), _conv_t3_ref(x, w5, bias, add16), TOL[dt], f"conv_t3 {case} {dt}")


@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("frames", [1, 2, 14])
def test_conv_t3_delta(dt, frames):
    """Exact: pixels only on the first and last frame (and one in the middle): the clip ends are zero-padded and nothing
    wraps from frame n-1 into frame 0 or from one image's pixel into another's."""
    h, w, c = 16, 8, 64
    g = torch.Generator().manual_seed(frames)
    ends = sorted({0, frames - 1})
    x = _delta_input(g, frames, h, w, c, _edge_points(h, w), images=ends)
    if frames > 2:
        x[frames // 2] = _delta_input(g, 1, h, w, c, [(h // 2, w // 2)])[0]
    x = x.to(DEV, dt)
    w5 = _ints(g, -3, 3, c, c, 3, 1, 1).to(DEV, dt)
    bias = _ints(g, -2, 2, c).to(DEV)
    add16 = _ints(g, -4, 4, frames, h, w, c).to(DEV, dt)
    _equal(_conv_t3(x, w5, bias, None), _conv_t3_ref(x, w5, bias, None), f"conv_t3 delta frames={frames} {dt}")
    _equal(_conv_t3(x, w5, bias, add16), _conv_t3_ref(x, w5, bias, add16), f"conv_t3 delta + shortcut frames={frames} {dt}")


# ----------------------------------------------------------------------------------------------- stride-2 Downsample2D
def _down2_ref(x16, wt, bias):
    return _nhwc(F.conv2d(F.pad(_nchw(x16.double()), (0, 1, 0, 1)), wt.double(), bias.double(), stride=2))


def _down2(x16, wt, bias):
    from latte_b200 import ops, vae
    return ops.vae_conv(x16.contiguous(), vae.pack_down2(wt).to(x16.dtype).contiguous(), bias, "down2")


@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("case", [(1, 32, 64), (3, 32, 512), (2, 64, 128), (1, 64, 512), (1, 128, 64), (2, 128, 128),
                                  (1, 256, 128), (1, 256, 64)], ids=lambda c: "n{}_{}px_c{}".format(*c))
def test_downsample(dt, case):
    n, s, c = case
    g = torch.Generator().manual_seed(n + s + c)
    x = _randn(g, n, s, s, c).to(DEV, dt)
    wt = _randn(g, c, c, 3, 3, scale=(9 * c) ** -0.5).to(DEV, dt)
    bias = _randn(g, c, scale=0.1).to(DEV)
    _close(_down2(x, wt, bias), _down2_ref(x, wt, bias), TOL[dt], f"downsample {case} {dt}")


@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("s", [32, 64, 256])
def test_downsample_delta(dt, s):
    """Exact: pixels on the bottom row and right column (read by the last output row / column through the zero padding of
    F.pad (0,1,0,1)), on odd and even rows and columns, in two stacked images."""
    n, c = 2, 64
    g = torch.Generator().manual_seed(s)
    pts = _edge_points(s, s) + [(s - 1, s // 2 + 1), (s // 2 + 1, s - 1), (s - 2, s - 2), (s - 3, s - 1), (1, 1), (3, 2)]
    x = _delta_input(g, n, s, s, c, sorted(set(pts))).to(DEV, dt)
    wt = _ints(g, -3, 3, c, c, 3, 3).to(DEV, dt)
    bias = _ints(g, -2, 2, c).to(DEV)
    _equal(_down2(x, wt, bias), _down2_ref(x, wt, bias), f"downsample delta {s}px {dt}")


# ----------------------------------------------------------------------------------------------------------- GroupNorm
def _gn_ref(x16, groups, gamma, beta, eps, silu):
    n, C = x16.shape[0], x16.shape[-1]
    xd = x16.double().reshape(n, -1, C).transpose(1, 2)                # [n, C, pixels]
    y = F.group_norm(xd, groups, gamma.double(), beta.double(), eps).transpose(1, 2).reshape(x16.shape)
    return F.silu(y) if silu else y


def _affine(g, C):
    return (1 + _randn(g, C, scale=0.3)).to(DEV), _randn(g, C, scale=0.3).to(DEV)


GN_CASES = [
    # C, groups, hw, n_img, eps, silu     cpg = C / groups: 4 (one thread's 8 channels straddle two groups), 8, 16
    (64, 16, 128, 1, 1e-6, True),
    (64, 16, 65536, 3, 1e-5, False),
    (64, 16, 384, 3, 1e-6, False),       # 384 = a partial 256-pixel block
    (128, 32, 384, 3, 1e-6, True),
    (128, 32, 4096, 1, 1e-5, True),
    (128, 32, 65536, 1, 1e-6, False),
    (256, 32, 128, 3, 1e-5, True),
    (256, 32, 65536, 1, 1e-6, True),
    (256, 32, 4096, 3, 1e-6, False),
    (512, 32, 384, 1, 1e-5, True),
    (512, 32, 4096, 3, 1e-6, False),
    (512, 32, 65536, 1, 1e-5, True),
]


@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("case", GN_CASES, ids=lambda c: "C{}_g{}_hw{}_n{}_eps{:g}{}".format(*c[:5], "_silu" if c[5] else ""))
def test_group_norm(dt, case):
    from latte_b200 import ops
    C, groups, hw, n, eps, silu = case
    g = torch.Generator().manual_seed(C + hw + n)
    # per-channel offsets and scales, so every group has its own statistics
    x = (_randn(g, n, hw, C) * (0.5 + _randn(g, C).abs()) + _randn(g, C)).to(DEV, dt)
    gamma, beta = _affine(g, C)
    _close(ops.group_norm(x, gamma, beta, groups, eps, silu), _gn_ref(x, groups, gamma, beta, eps, silu), TOL[dt],
           f"group_norm {case} {dt}")


@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("C,groups", [(128, 32), (512, 32)])
@pytest.mark.parametrize("clips", [1, 2])
def test_group_norm_temporal(dt, C, groups, clips):
    """The temporal decoder's GroupNorm: statistics over all 14 frames of a clip, i.e. one image of 14 * h * w pixels,
    against F.group_norm on the [clips, C, frames, h, w] tensor (eps 1e-5, + SiLU)."""
    from latte_b200 import ops
    frames, h, w = 14, 16, 16
    g = torch.Generator().manual_seed(C + clips)
    x = (_randn(g, clips, frames, h, w, C) * 2 + _randn(g, C)).to(DEV, dt)
    gamma, beta = _affine(g, C)
    got = ops.group_norm(x, gamma, beta, groups, 1e-5, True)
    ref = F.silu(F.group_norm(x.double().permute(0, 4, 1, 2, 3), groups, gamma.double(), beta.double(), 1e-5)).permute(0, 2, 3, 4, 1)
    _close(got, ref, TOL[dt], f"group_norm temporal C{C} clips{clips} {dt}")


@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("C,groups", [(128, 32), (512, 32)])
@pytest.mark.parametrize("silu", [False, True])
def test_group_norm_constant_group(dt, C, groups, silu):
    """A group whose pixels are all equal has zero variance: its output is silu?(beta), finite."""
    from latte_b200 import ops
    hw, cpg = 65536, C // groups
    g = torch.Generator().manual_seed(C)
    x = _randn(g, 1, hw, C)
    x[..., :cpg] = 0.7                          # group 0: a constant that is not a power of two
    x[..., cpg:2 * cpg] = 0.0                   # group 1: all zero
    x = x.to(DEV, dt)
    gamma, beta = _affine(g, C)
    got = ops.group_norm(x, gamma, beta, groups, 1e-6, silu)
    assert torch.isfinite(got).all()
    want = beta.double()[: 2 * cpg].expand(1, hw, 2 * cpg)
    _close(got[..., : 2 * cpg], F.silu(want) if silu else want, TOL[dt], f"group_norm constant group C{C} silu={silu} {dt}")
    _close(got, _gn_ref(x, groups, gamma, beta, 1e-6, silu), TOL[dt], f"group_norm with constant groups C{C} silu={silu} {dt}")


@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("C,groups", [(128, 32), (512, 32)])
@pytest.mark.parametrize("mean_over_std", [16, 64])
def test_group_norm_large_mean(dt, C, groups, mean_over_std):
    """Groups whose mean is 16 or 64 times their standard deviation over 65536 pixels: the variance must not be lost to
    cancellation in the statistics.  Ordinary inputs land within one rounding of the output, and so must these: the bound
    here is two roundings (2^-10 fp16, 2^-7 bf16, abs + rel).  One-pass sums of the raw values missed it at 64x by up to
    7 fp16 roundings."""
    from latte_b200 import ops
    hw, cpg = 65536, C // groups
    g = torch.Generator().manual_seed(mean_over_std + C)
    std = 0.5 + torch.rand(groups, generator=g)                         # per group
    sign = 1 - 2 * _ints(g, 0, 1, groups)
    mean = (sign * mean_over_std * std).repeat_interleave(cpg)
    x = (_randn(g, 1, hw, C) * std.repeat_interleave(cpg) + mean).to(DEV, dt)
    gamma, beta = _affine(g, C)
    two_roundings = {torch.float16: 2.0 ** -10, torch.bfloat16: 2.0 ** -7}[dt]
    _close(ops.group_norm(x, gamma, beta, groups, 1e-6, False), _gn_ref(x, groups, gamma, beta, 1e-6, False), two_roundings,
           f"group_norm mean/std={mean_over_std} C{C} {dt}")


# ------------------------------------------------------------------------------------------------- mid-block attention
def _attn_weights(g, C, dt, qk_scale):
    from latte_b200 import vae
    w = {k: _randn(g, C, C, scale=C ** -0.5 * (qk_scale if k in "qk" else 1.0)).to(DEV, dt) for k in "qkvo"}
    b = {k: _randn(g, C, scale=0.05).to(DEV) for k in "qkvo"}
    gn_g, gn_b = (1 + _randn(g, C, scale=0.1)).to(DEV), _randn(g, C, scale=0.05).to(DEV)
    packed = dict(gn_g=gn_g, gn_b=gn_b, q_w16=vae.pack_linear(w["q"]).contiguous(), q_b=b["q"], k_w16=vae.pack_linear(w["k"]).contiguous(),
                  k_b=b["k"], v_w16=vae.pack_linear(w["v"]).contiguous(), o_w16=vae.pack_linear(w["o"]).contiguous(),
                  o_b=vae.fold_v_bias(w["o"], b["o"], b["v"]).contiguous())
    return w, b, gn_g, gn_b, packed


def _attn_ref(x16, w, b, gn_g, gn_b, groups, eps):
    """oracle/vae_oracle.py mid_attention in fp64: x + to_out(softmax(q k^T / sqrt(C)) v), q/k/v of GroupNorm(x).  The
    GroupNorm output and q, k are rounded to the 16-bit type, as the product stores them: with peaked scores the
    logits' error from that rounding alone exceeds one rounding of the output.
    Also returns, per query, the gap between its two largest logits and the spread (max - min per channel) of the outputs
    x + to_out(v_j) of its three best keys j: near a tie the result may move anywhere between those."""
    n, h, w_, C = x16.shape
    dt = x16.dtype
    xd = x16.double().reshape(n, h * w_, C)
    xg = F.group_norm(xd.transpose(1, 2), groups, gn_g.double(), gn_b.double(), eps).transpose(1, 2).to(dt).double()
    q = F.linear(xg, w["q"].double(), b["q"].double()).to(dt).double()
    k = F.linear(xg, w["k"].double(), b["k"].double()).to(dt).double()
    v = F.linear(xg, w["v"].double(), b["v"].double())
    s = q @ k.transpose(1, 2) * C ** -0.5
    o = F.linear(torch.softmax(s, dim=-1) @ v, w["o"].double(), b["o"].double())
    top = s.topk(3, dim=-1)
    per_key = F.linear(v, w["o"].double(), b["o"].double())                        # [n, keys, C]
    best = torch.stack([torch.gather(per_key, 1, top.indices[..., j:j + 1].expand(n, h * w_, C)) for j in range(3)])
    spread = (best.amax(0) - best.amin(0)).reshape(n, h, w_, C)
    gap = (top.values[..., 0] - top.values[..., 1]).reshape(n, h, w_)
    return (o + xd).reshape(n, h, w_, C), gap, spread


@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("case", [
    # n, h, w, C, scale of the q and k weights
    (1, 8, 16, 128, 1.0), (2, 8, 16, 512, 1.0), (1, 32, 32, 512, 1.0), (2, 32, 32, 128, 1.0),
    (1, 64, 64, 128, 1.0), (2, 64, 64, 512, 1.0),
    (1, 32, 32, 128, 8.0),               # scores 64x larger: the softmax in its peaked regime
], ids=lambda c: "n{}_{}x{}_C{}_qk{:g}".format(*c))
def test_mid_attention(dt, case):
    from latte_b200 import ops
    n, h, w, C, qk = case
    groups = 32
    g = torch.Generator().manual_seed(n + h * w + C + int(qk))
    x = _randn(g, n, h, w, C).to(DEV, dt)
    wts, bs, gn_g, gn_b, packed = _attn_weights(g, C, dt, qk)
    got = ops.vae_mid_attention(x, groups=groups, eps=1e-6, **packed)
    ref, gap, spread = _attn_ref(x, wts, bs, gn_g, gn_b, groups, 1e-6)
    if qk == 1.0:
        _close(got, ref, TOL[dt], f"mid_attention {case} {dt}")
        return
    # Peaked: a query whose two best logits lie within a few units of each other weighs them by exp(gap), and a one-ulp
    # difference in the 16-bit q or k moves its output along the segment between them.  Queries with a clear winner
    # (gap >= 4: the runner-up's weight < 2 %) get the one-rounding tolerance; near-tie queries must stay finite and
    # within the spread of their best keys' outputs.
    clear = gap >= 4.0
    assert clear.float().mean() > 0.5, f"only {clear.float().mean().item():.2f} of the queries are peaked"
    _close(got[clear], ref[clear], TOL[dt], f"mid_attention {case} {dt}, {int(clear.sum())} peaked queries")
    near = ~clear
    err = (got[near].double() - ref[near]).abs()
    assert torch.isfinite(got).all() and (err <= TOL[dt] * (1 + ref[near].abs()) + spread[near]).all(), \
        f"mid_attention {case} {dt}: a near-tie query leaves the spread of its best keys, max err {err.max().item():.3e}"
