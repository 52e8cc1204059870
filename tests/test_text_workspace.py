"""CPU: tests/text_workspace.py's mirror of the T5 and LatteT2V workspace layouts has the library's total size, so the
fp64 GPU tests (test_gpu_t5_fp64.py, test_gpu_t2v_glue_fp64.py) read each stage's buffer where the kernels wrote it.  The size
queries run before anything is launched, so no GPU is needed."""
import ctypes as C

import pytest
import torch

import text_workspace as TW
from latte_b200 import _lib

T5_SHAPES = [(256, 4, 512, 100), (512, 8, 1024, 32128), (4096, 64, 10240, 512), (4096, 64, 10240, 32128), (768, 12, 2048, 7)]


@pytest.mark.parametrize("d_model,heads,d_ff,vocab", T5_SHAPES)
@pytest.mark.parametrize("batch", [1, 2, 3, 8])
def test_t5_layout_matches_library(d_model, heads, d_ff, vocab, batch):
    lib = _lib.load()
    for dtype in (_lib.FP16, _lib.BF16):
        s = _lib.T5Shape(layers=1, d_model=d_model, heads=heads, d_ff=d_ff, vocab=vocab, dtype=dtype, eps=1e-6)
        want = lib.b200_t5_workspace_bytes(C.byref(s), batch)
        assert want > 0, _lib.last_error()
        assert TW.total_bytes(TW.t5_layout(d_model, heads, d_ff, batch)) == want
        s.layers = 24                    # the layout does not depend on the depth
        assert lib.b200_t5_workspace_bytes(C.byref(s), batch) == want


T2V_SHAPES = [  # (layers, heads, head_dim, caption_channels, input_size, out_channels)
    (28, 16, 72, 4096, 64, 8), (28, 16, 72, 4096, 16, 8), (2, 16, 72, 4096, 32, 8), (2, 2, 64, 256, 16, 8),
    (1, 8, 72, 512, 32, 4), (3, 6, 64, 1024, 16, 8),
]


@pytest.mark.parametrize("layers,heads,hd,cap,size,out_ch", T2V_SHAPES)
@pytest.mark.parametrize("frames", [1, 4, 16])
def test_t2v_layout_matches_library(layers, heads, hd, cap, size, out_ch, frames):
    lib = _lib.load()
    D = heads * hd
    for batch in (1, 2, 3):
        for text_len in (1, 9, 120, 128):
            s = _lib.T2VShape(layers=layers, hidden=D, heads=heads, mlp_hidden=4 * D, patch=2, in_channels=4,
                              out_channels=out_ch, input_size=size, frames=frames, caption_channels=cap, dtype=_lib.BF16)
            want = lib.b200_t2v_workspace_bytes(C.byref(s), batch, text_len)
            if frames * (size // 2) ** 2 % 128:      # not a whole number of 128-row tiles per sample: refused
                assert want == 0 and "multiple of 128" in _lib.last_error()
                continue
            assert want > 0, _lib.last_error()
            got = TW.total_bytes(TW.t2v_layout(layers, D, 4 * D, 2, out_ch, size, frames, cap, batch, text_len))
            assert got == want, (batch, text_len, got, want)


def test_workspace_views_tile_the_buffer():
    """The views start on 1024-byte boundaries in declaration order and end inside the buffer."""
    layout = TW.t2v_layout(2, 1152, 4608, 2, 8, 16, 4, 4096, 2, 9, torch.bfloat16)
    ws = TW.Workspace(layout, torch.device("cpu"))
    assert ws.ptr % 1024 == 0 and ws.nbytes == TW.total_bytes(layout)
    prev_end = ws.ptr
    for name, dt, shape in layout:
        v = ws[name]
        assert v.dtype == dt and tuple(v.shape) == shape
        assert v.data_ptr() % 1024 == 0 and v.data_ptr() >= prev_end
        prev_end = v.data_ptr() + v.numel() * v.element_size()
    assert prev_end <= ws.ptr + ws.nbytes
    ws.poison()
    assert torch.isnan(ws["x"]).all() and torch.isnan(ws["kv_all"].float()).all()
