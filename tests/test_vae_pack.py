"""CPU: the weight layouts of latte_b200/vae.py, read back the way the native convolutions read them (csrc/vae.cu: the tap
tables of conv3x3 / conv_t3 / conv_down2 and the space_to_depth regrouping), reproduce the torch ops exactly in fp64."""
import torch
import torch.nn.functional as F

from latte_b200 import vae


def _shift(x, dy, dx):
    """x [n, h, w, c] -> x[n, y + dy, x + dx, c], zero outside the image (TMA zero-fill)."""
    n, h, w, c = x.shape
    out = torch.zeros_like(x)
    ys, xs = slice(max(0, -dy), min(h, h - dy)), slice(max(0, -dx), min(w, w - dx))
    out[:, ys, xs] = x[:, max(0, dy):min(h, h + dy), max(0, dx):min(w, w + dx)]
    return out


def _implicit_gemm(x, wp, taps):
    """sum over taps t of shift(x, dy_t, dx_t) @ wp[:, t*C:(t+1)*C]^T -- the k-block order of the GEMM's conv mode."""
    c = x.shape[-1]
    return sum(_shift(x, dy, dx) @ wp[:, t * c:(t + 1) * c].t() for t, (dy, dx) in enumerate(taps))


def test_conv3x3_layout():
    g = torch.Generator().manual_seed(0)
    x, wt = torch.randn(2, 5, 7, 16, generator=g, dtype=torch.float64), torch.randn(8, 16, 3, 3, generator=g, dtype=torch.float64)
    taps = [(t // 3 - 1, t % 3 - 1) for t in range(9)]
    got = _implicit_gemm(x, vae.pack_conv3x3(wt), taps)
    ref = F.conv2d(x.permute(0, 3, 1, 2), wt, padding=1).permute(0, 2, 3, 1)
    assert torch.allclose(got, ref, atol=1e-12)


def test_conv_t3_layout():
    """Conv3d (3,1,1) over the frames of one clip: the taps move along the image index (frames), zero beyond both ends."""
    g = torch.Generator().manual_seed(1)
    frames, h, w, c = 5, 3, 4, 8
    x, wt = torch.randn(frames, h, w, c, generator=g, dtype=torch.float64), torch.randn(c, c, 3, 1, 1, generator=g, dtype=torch.float64)
    wp = vae.pack_conv_t3(wt, 0.5).double()
    xs = x.reshape(1, frames, h * w, c)
    got = sum(_shift(xs, kt - 1, 0) @ wp[:, kt * c:(kt + 1) * c].t() for kt in range(3)).reshape(frames, h, w, c)
    ref = F.conv3d(x.permute(3, 0, 1, 2)[None], wt * 0.5, padding=(1, 0, 0))[0].permute(1, 2, 3, 0)
    assert torch.allclose(got, ref, atol=1e-12)


def test_down2_layout():
    """Downsample2D (pad (0,1,0,1), stride 2) = space_to_depth + 2x2 taps over 4C channels; the (phase 1, offset 1) weights,
    which would read input row / column 2y + 3, are zero."""
    g = torch.Generator().manual_seed(2)
    n, h, w, c = 2, 8, 6, 4
    x, wt = torch.randn(n, h, w, c, generator=g, dtype=torch.float64), torch.randn(5, c, 3, 3, generator=g, dtype=torch.float64)
    s2d = x.reshape(n, h // 2, 2, w // 2, 2, c).permute(0, 1, 3, 2, 4, 5).reshape(n, h // 2, w // 2, 4 * c)   # [.., py*2+px, c]
    wp = vae.pack_down2(wt).double()
    got = _implicit_gemm(s2d, wp, [(t >> 1, t & 1) for t in range(4)])
    ref = F.conv2d(F.pad(x.permute(0, 3, 1, 2), (0, 1, 0, 1)), wt, stride=2).permute(0, 2, 3, 1)
    assert torch.allclose(got, ref, atol=1e-12)
    five = wp.reshape(5, 2, 2, 2, 2, c)                       # [O][oy][ox][py][px][I]
    assert five[:, 1, :, 1].abs().sum() == 0 and five[:, :, 1, :, 1].abs().sum() == 0


def test_fold_v_bias():
    """P (V + 1 b_v^T) W_o^T + b_o == P V W_o^T + fold_v_bias(W_o, b_o, b_v) for row-stochastic P."""
    g = torch.Generator().manual_seed(3)
    C, n = 16, 10
    p = torch.softmax(torch.randn(n, n, generator=g, dtype=torch.float64), -1)
    v, wo = torch.randn(n, C, generator=g, dtype=torch.float64), torch.randn(C, C, generator=g, dtype=torch.float64)
    bo, bv = torch.randn(C, generator=g, dtype=torch.float64), torch.randn(C, generator=g, dtype=torch.float64)
    ref = (p @ (v + bv)) @ wo.t() + bo
    assert torch.allclose(p @ v @ wo.t() + vae.fold_v_bias(wo, bo, bv).double(), ref, atol=1e-4)
