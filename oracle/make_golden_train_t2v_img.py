"""tests/golden/train_t2v_img_*.npz: the vector-Jacobian product of one training-mode forward of the UNMODIFIED reference
LatteT2V with video + image joint training (`use_image_num` > 0; /root/reference/models/latte_t2v.py through oracle/ref_shim,
loaded as make_golden_t2v.py loads it).

TEST INFRASTRUCTURE.  Runs only where the reference checkout exists; outputs are committed.
    python oracle/make_golden_train_t2v_img.py

As make_golden_train_t2v.py in every other respect: the module in `.train()` (not checkpointed) on seeded weights and inputs
(oracle/t2v_oracle.make_weights, oracle/t2v_img_oracle.make_img_inputs: x (B, C, F + I, H, W), captions (B, 1 + I, L, caption_channels)), an optional
3-D caption keep-mask (B, 1 + I, L) whose rows keep different numbers of leading tokens (0 = a fully masked caption), and
`loss = (out * g).sum()` back-propagated for a seeded cotangent g = randn(out.shape, Generator(gseed)).  Stored: the output,
every parameter's gradient norm (float64) and the full gradient of the same ten parameters; gradients above 16 Ki elements keep
every s-th row, the output every 4th latent row (`<key>_sample` = [axis, s], as make_golden.strided_sample records it).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(HERE, "ref_shim"))

from oracle import t2v_img_oracle as TI  # noqa: E402
from oracle import t2v_oracle as T  # noqa: E402
from oracle.make_golden import strided_sample  # noqa: E402
from oracle.make_golden_t2v import HD72, TINY, build_ref_model, load_reference  # noqa: E402
from oracle.make_golden_train_t2v import FULL  # noqa: E402

TINY256 = dict(TINY, sample_size=32, video_length=4)        # 256 tokens per frame: the images' cross-attention takes 128-row tiles
HD72_F8 = dict(HD72, video_length=8)
F1 = dict(TINY, sample_size=32, video_length=1)
# tag: (config, batch, images, text_len, weight seed, input seed, cotangent seed, kept tokens per (sample, caption) or None)
CASES = {
    "tiny_f4_i3_b2_l20": (TINY256, 2, 3, 20, 3, 4, 11, None),
    "tiny_f4_i3_b2_l20_masked": (TINY256, 2, 3, 20, 3, 4, 11, [[5, 20, 0, 12], [20, 7, 3, 1]]),
    "hd72_f8_i2_b1_l120_masked": (HD72_F8, 1, 2, 120, 5, 6, 12, [[12, 120, 40]]),
    "f1_i2_b2_l20": (F1, 2, 2, 20, 8, 9, 13, [[7, 20, 3], [20, 11, 20]]),
}


def make_mask3(kept, text_len):
    """(B, 1 + I, L) 0/1 keep-mask, kept[b][k] leading ones in caption k of sample b (T5 pads at the end)."""
    m = torch.zeros(len(kept), len(kept[0]), text_len, dtype=torch.int64)
    for b, row in enumerate(kept):
        for k, n in enumerate(row):
            m[b, k, :n] = 1
    return m


def make(ref, tag, cfg_kw, batch, images, text_len, wseed, iseed, gseed, kept):
    cfg = T.T2VConfig(**cfg_kw)
    sd = T.make_weights(cfg, wseed)
    x, t, text = TI.make_img_inputs(cfg, batch, images, text_len, iseed)
    m = build_ref_model(ref, cfg, sd).train()
    mask = make_mask3(kept, text_len) if kept is not None else None
    out = m(x, t, encoder_hidden_states=text, encoder_attention_mask=mask, use_image_num=images, return_dict=False)[0]
    assert out.shape == (batch, cfg.out_channels, cfg.video_length + images, cfg.sample_size, cfg.sample_size)
    g = torch.randn(out.shape, generator=torch.Generator().manual_seed(gseed))
    (out * g).sum().backward()
    res = dict(out=out.detach().numpy(), cfg=np.array(repr(cfg_kw)), batch=np.int64(batch), images=np.int64(images),
               text_len=np.int64(text_len), wseed=np.int64(wseed), iseed=np.int64(iseed), gseed=np.int64(gseed),
               meta=np.array("reference LatteT2V in .train(), use_image_num = images, "
                             "loss = (out * randn(out.shape, Generator(gseed))).sum()"))
    if mask is not None:
        res["mask"] = mask.numpy()
    names, norms = [], []
    for k, p in m.named_parameters():
        assert p.grad is not None, k
        names.append(k)
        norms.append(p.grad.double().norm().item())
        if k in FULL:
            res["grad::" + k] = p.grad.numpy()
            if p.grad.numel() > 1 << 14:
                strided_sample(res, "grad::" + k, 0, min(-(-p.grad.numel() // (1 << 14)), p.grad.shape[0]))
    res["grad_names"] = np.array(names)
    res["grad_norms"] = np.array(norms, dtype=np.float64)
    if res["out"].size > 1 << 15:
        strided_sample(res, "out", 3, 4)         # every frame, video and image ones alike
    path = os.path.join(ROOT, "tests", "golden", f"train_t2v_img_{tag}.npz")
    np.savez_compressed(path, **res)
    print("wrote", path, f"({os.path.getsize(path) / 1e3:.0f} kB)", "params", len(names))


def main():
    torch.manual_seed(0)
    ref = load_reference()
    for tag, case in CASES.items():
        make(ref, tag, *case)


if __name__ == "__main__":
    main()
