"""The workspace layouts of `b200_t5_encode` and `b200_t2v_forward` (t5_carve / t2v_carve in latte_b200/csrc/api.cu): every
buffer in declaration order, each starting on a 1024-byte boundary.  The caller owns the workspace, so after one call the
fp64 tests read the exact 16-bit and fp32 tensors each stage read and wrote.  tests/test_text_workspace.py holds the totals
to the library's own size queries."""
import torch

ALIGN = 1024
GEMM_SK_FLAGS = 1024          # u64 words (B200_GEMM_SK_FLAGS)


def _up(n):
    return (n + ALIGN - 1) // ALIGN * ALIGN


def t5_layout(d_model, heads, d_ff, batch, dt=torch.float16):
    """[(name, dtype, shape)] of t5_carve: sequences padded to 128 rows."""
    R, D, I, FF = batch * 128, d_model, heads * 64, d_ff
    return [("x", torch.float32, (R, D)), ("h", dt, (R, D)), ("qkv", dt, (R, 3 * I)), ("att", dt, (R, I)),
            ("g0", dt, (R, FF)), ("g", dt, (R, FF)), ("ones", torch.float32, (D,)), ("sk_flags", torch.int64, (GEMM_SK_FLAGS,))]


def t2v_layout(layers, hidden, mlp_hidden, patch, out_channels, input_size, frames, caption_channels, batch, text_len,
               dt=torch.float16):
    """[(name, dtype, shape)] of t2v_carve.  `head` is the fp32 [T, n_out] head output followed by its n_out ones, sized for
    at least 32 columns (head_floats)."""
    grid = input_size // patch
    T, D, R, L = batch * frames * grid * grid, hidden, batch * text_len, layers
    n_out = max(patch * patch * out_channels, 32)
    return [("x", torch.float32, (T, D)), ("h", dt, (T, D)), ("qkv", dt, (T, 3 * D)), ("g", dt, (T, mlp_hidden)),
            ("text16", dt, (R, caption_channels)), ("cap_h", dt, (R, D)), ("cap_o", dt, (R, D)),
            ("kv_all", dt, (R, L * 2 * D)), ("ones", torch.float32, (D,)), ("tfreq", torch.float32, (batch, 256)),
            ("th", torch.float32, (batch, D)), ("emb", torch.float32, (batch, D)), ("ts", torch.float32, (batch, 6 * D)),
            ("mod", torch.float32, (batch, L * 2 * 6 * D + 2 * D)), ("sk_flags", torch.int64, (GEMM_SK_FLAGS,)),
            ("head", torch.float32, ((T + 1) * n_out,))]


def _nbytes(dtype, shape):
    n = dtype.itemsize
    for s in shape:
        n *= s
    return n


def total_bytes(layout):
    return sum(_up(_nbytes(dt, shape)) for _, dt, shape in layout)


class Workspace:
    """A device workspace for one layout, every byte 0xFF before each call (a NaN in fp32, fp16 and bf16), so a stage that
    reads memory no earlier stage wrote yields non-finite values.  `ptr` is 1024-byte aligned; `views[name]` are tensors over
    the buffers."""

    def __init__(self, layout, device):
        self.nbytes = total_bytes(layout)
        self._raw = torch.empty(self.nbytes + ALIGN, dtype=torch.uint8, device=device)
        base = (-self._raw.data_ptr()) % ALIGN
        self._buf = self._raw[base:base + self.nbytes]
        self.ptr = self._buf.data_ptr()
        self.views, off = {}, 0
        for name, dt, shape in layout:
            n = _nbytes(dt, shape)
            self.views[name] = self._buf[off:off + n].view(dt).view(shape)
            off += _up(n)

    def poison(self):
        self._buf.fill_(0xFF)

    def __getitem__(self, name):
        return self.views[name]
