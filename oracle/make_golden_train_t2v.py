"""tests/golden/train_t2v_*.npz: the vector-Jacobian product of one training-mode forward of the UNMODIFIED reference
LatteT2V (/root/reference/models/latte_t2v.py through oracle/ref_shim, loaded as make_golden_t2v.py loads it).

TEST INFRASTRUCTURE.  Runs only where the reference checkout exists; outputs are committed.
    python oracle/make_golden_train_t2v.py

The reference ships no text-to-video training objective, so none is invented: the module is put in `.train()`, run on seeded
weights and inputs (oracle/t2v_oracle.make_weights / make_inputs, padded-prompt mask as in make_golden_t2v.py), and
`loss = (out * g).sum()` is back-propagated for a seeded cotangent g = randn(out.shape, Generator(gseed)).  Stored: the output,
every parameter's gradient norm (float64) and the full gradient of a representative subset; gradients above 16 Ki elements keep
every s-th row (the output: every 4th frame) (`<key>_sample` = [axis, s], as make_golden.strided_sample records it).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(HERE, "ref_shim"))

from oracle import t2v_oracle as T  # noqa: E402
from oracle.make_golden import strided_sample  # noqa: E402
from oracle.make_golden_t2v import HD72, TINY, build_ref_model, load_reference, make_mask  # noqa: E402

F1 = dict(TINY, sample_size=32, video_length=1)     # text-to-image: 256 tokens, one frame
FULL = ["caption_projection.linear_1.weight", "transformer_blocks.1.attn2.to_q.weight", "transformer_blocks.1.attn2.to_k.weight",
        "transformer_blocks.1.attn2.to_v.weight", "transformer_blocks.0.scale_shift_table",
        "temporal_transformer_blocks.1.scale_shift_table", "adaln_single.linear.weight",
        "adaln_single.emb.timestep_embedder.linear_1.weight", "proj_out.weight", "temporal_transformer_blocks.0.attn1.to_q.weight"]
# tag: (config, batch, text_len, weight seed, input seed, cotangent seed, valid prompt tokens per sample or None)
CASES = {
    "tiny_b2_l20": (TINY, 2, 20, 3, 4, 11, None),
    "tiny_b2_l20_masked": (TINY, 2, 20, 3, 4, 11, [5, 20]),
    "hd72_b2_l120_masked": (HD72, 2, 120, 5, 6, 12, [12, 120]),
    "f1_b2_l20": (F1, 2, 20, 8, 9, 13, [7, 20]),
}


def make(ref, tag, cfg_kw, batch, text_len, wseed, iseed, gseed, valid):
    cfg = T.T2VConfig(**cfg_kw)
    sd = T.make_weights(cfg, wseed)
    x, t, text = T.make_inputs(cfg, batch, text_len, iseed)
    m = build_ref_model(ref, cfg, sd).train()
    mask = make_mask(batch, text_len, valid) if valid is not None else None
    out = m(x, t, encoder_hidden_states=text, encoder_attention_mask=mask, return_dict=False)[0]
    g = torch.randn(out.shape, generator=torch.Generator().manual_seed(gseed))
    (out * g).sum().backward()
    res = dict(out=out.detach().numpy(), cfg=np.array(repr(cfg_kw)), batch=np.int64(batch), text_len=np.int64(text_len),
               wseed=np.int64(wseed), iseed=np.int64(iseed), gseed=np.int64(gseed),
               meta=np.array("reference LatteT2V in .train(), loss = (out * randn(out.shape, Generator(gseed))).sum()"))
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
        strided_sample(res, "out", 2, 4)
    path = os.path.join(ROOT, "tests", "golden", f"train_t2v_{tag}.npz")
    np.savez_compressed(path, **res)
    print("wrote", path, f"({os.path.getsize(path) / 1e3:.0f} kB)", "params", len(names))


def main():
    torch.manual_seed(0)
    ref = load_reference()
    for tag, case in CASES.items():
        make(ref, tag, *case)


if __name__ == "__main__":
    main()
