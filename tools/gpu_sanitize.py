"""Small invocations of every kernel family through the C ABI, to be run under compute-sanitizer (tools/gpu_sanitize.sh):
a tiny72 Latte forward (+cfg), a stream-K residual GEMM, both attention kernels in every mode, a LatteT2V forward with a
padded-prompt mask, the VAE decoder conv stack and the fused sampler step.  Shapes are small: the sanitizers slow kernels
by 10-100x.  Usage: python tools/gpu_sanitize.py [latte] [gemm] [attn] [t2v] [vae] [sampler]"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from latte_b200 import Latte, LatteT2V, ops  # noqa: E402
from oracle import latte_oracle as O  # noqa: E402

dev = torch.device("cuda:0")


def latte():
    cfg = O.make_config("Latte-tiny72/2", input_size=16, num_frames=16)
    sd = O.make_weights(cfg, 5)
    x, t, y = O.make_inputs(cfg, 2, 6)
    net = Latte(input_size=cfg.input_size, hidden_size=cfg.hidden_size, depth=cfg.depth, num_heads=cfg.num_heads,
                num_frames=cfg.num_frames, num_classes=cfg.num_classes, learn_sigma=True, extras=2)
    net.load_state_dict(sd, strict=True)
    net = net.to(dev).eval()
    net.use_cuda_graphs = False
    with torch.no_grad():
        out = net.forward_with_cfg(x.to(dev), t.to(dev), y=y.to(dev), cfg_scale=7.0)
    torch.cuda.synchronize()
    ref = O.latte_forward_with_cfg(sd, cfg, x, t, y, cfg_scale=7.0)
    print("latte tiny72 forward_with_cfg: max err", (out.cpu() - ref).abs().max().item(), flush=True)


def gemm():
    g = torch.Generator().manual_seed(0)
    for (M, N, K) in [(148 * 128 + 256, 256, 2048), (640, 384, 1152)]:   # the first one streams its last waves along K
        A = torch.randn(M, K, generator=g).to(dev).half()
        W = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev).half()
        bias = torch.randn(N, generator=g).to(dev)
        gate = torch.randn(2, N, generator=g).to(dev)
        x0 = torch.randn(M, N, generator=g).to(dev)
        rpb = (M + 1) // 2
        want = x0 + gate[torch.arange(M, device=dev) // rpb] * (A.float() @ W.float().t() + bias)
        x = x0.clone()
        ops.linear_gate_residual_(x, A, W, bias, gate, rpb)
        torch.cuda.synchronize()
        print(f"gemm resid {M}x{N}x{K}: max err", (x - want).abs().max().item(), "flags clean:", int(ops._sk_flags(dev).abs().sum()) == 0, flush=True)
        o = ops.linear(A, W, bias, gelu=True)
        torch.cuda.synchronize()
        print(f"gemm gelu  {M}x{N}x{K}: ok", tuple(o.shape), flush=True)


def attn():
    g = torch.Generator().manual_seed(1)
    for (b, f, n, h, hd, temporal) in [(1, 2, 256, 2, 72, False), (1, 16, 16, 2, 72, True), (1, 8, 32, 2, 64, True), (1, 2, 64, 2, 80, False),
                                       (1, 1, 128, 1, 64, False)]:
        qkv = torch.randn(b * f * n, 3 * h * hd, generator=g).to(dev).half()
        o = ops.attention(qkv, b, f, n, h, temporal)
        torch.cuda.synchronize()
        print(f"attn b{b} f{f} n{n} h{h} hd{hd} temporal={temporal}: finite", bool(torch.isfinite(o.float()).all()), flush=True)
    q = torch.randn(2 * 128, 2 * 72, generator=g).to(dev).half()
    kv = torch.randn(2 * 20, 2 * 2 * 72, generator=g).to(dev).half()
    bias = torch.zeros(2, 128)
    bias[0, 5:] = -10000.0
    o = ops.cross_attention(q, kv, 2, 128, 20, 2, key_bias=bias.to(dev))
    torch.cuda.synchronize()
    print("cross attn with key bias: finite", bool(torch.isfinite(o.float()).all()), flush=True)
    qkv = torch.randn(1 * 1 * 512, 3 * 1 * 72, generator=g).to(dev).half()     # N = 512: the online-softmax kernel
    o = ops.attention(qkv, 1, 1, 512, 1, False)
    torch.cuda.synchronize()
    print("attn long N=512: finite", bool(torch.isfinite(o.float()).all()), flush=True)


def t2v():
    from oracle import t2v_oracle as T
    kw = dict(num_attention_heads=2, attention_head_dim=64, num_layers=1, sample_size=16, video_length=8, caption_channels=256)
    cfg = T.T2VConfig(**kw)
    sd = T.make_weights(cfg, 3)
    x, t, text = T.make_inputs(cfg, 2, 20, 4)
    mask = torch.zeros(2, 20, dtype=torch.int64)
    mask[0, :5] = 1
    mask[1] = 1
    net = LatteT2V(**kw)
    net.load_state_dict(sd, strict=True)
    net = net.to(dev).eval()
    with torch.no_grad():
        out = net(x.to(dev), t.to(dev), encoder_hidden_states=text.to(dev), encoder_attention_mask=mask.to(dev), return_dict=False)[0]
    torch.cuda.synchronize()
    ref = T.t2v_forward(sd, cfg, x, t, text, text_mask=mask)
    print("t2v tiny masked forward: max err", (out.cpu() - ref).abs().max().item(), flush=True)


def vae():
    from latte_b200 import AutoencoderKL
    net = AutoencoderKL(block_out_channels=(64, 128, 128), norm_num_groups=16).to(dev).half().eval()
    with torch.no_grad():
        out = net.decode(torch.randn(2, 4, 16, 16, device=dev)).sample
    torch.cuda.synchronize()
    print("vae decode (2 blocks):", tuple(out.shape), "finite", bool(torch.isfinite(out.float()).all()), flush=True)


def sampler():
    from latte_b200.diffusion import create_diffusion
    d = create_diffusion("8")
    g = torch.Generator().manual_seed(2)
    x = torch.randn(2, 4, 4, 8, 8, generator=g).to(dev)
    fake = lambda xx, tt, **kw: torch.cat([xx, xx * 0.1], dim=2)   # noqa: E731
    out = d.ddim_sample_loop(fake, x.shape, x, clip_denoised=False, device=dev)
    torch.cuda.synchronize()
    print("sampler ddim 8 steps: finite", bool(torch.isfinite(out).all()), flush=True)


def train():
    """One training step of the tiny64 model (every kernel of csrc/train.cu, dgrad / wgrad in the GEMM's MN-major modes, the
    multi-tensor passes) checked against the reference's golden gradients."""
    import numpy as np
    from latte_b200 import utils as U
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    gold = np.load(os.path.join(root, "tests", "golden", "train_tiny64.npz"))
    cfg = O.make_config("Latte-tiny64/2", input_size=16, num_frames=8)
    m = Latte(input_size=16, hidden_size=128, depth=2, num_heads=2, num_frames=8, num_classes=101, extras=2)
    m.load_state_dict(O.make_weights(cfg, 21), strict=True)
    m = m.to(dev).train()
    m.y_embedder.dropout_prob = 0.0
    from latte_b200.diffusion import create_diffusion
    d = create_diffusion(timestep_respacing="")
    x0, noise = torch.from_numpy(gold["x0"]).to(dev), torch.from_numpy(gold["noise"]).to(dev)
    t, y = torch.from_numpy(gold["t"]).to(dev), torch.from_numpy(gold["y"]).to(dev)
    loss = d.training_losses(m, x0, t, dict(y=y), noise=noise)["loss"].mean()
    loss.backward()
    torch.cuda.synchronize()
    named = dict(m.named_parameters())
    worst = max(abs(named[str(k)].grad.double().norm().item() - w) / w for k, w in zip(gold["grad_names"], gold["grad_norms"]))
    print("train tiny64 step: loss", loss.item(), "golden", float(gold["loss"]), "max err of grad norms (relative)", worst, flush=True)
    ema = Latte(input_size=16, hidden_size=128, depth=2, num_heads=2, num_frames=8, num_classes=101, extras=2).to(dev)
    n = U.clip_grad_norm_(m.parameters(), 1.0)
    U.update_ema(ema, m, 0.99)
    torch.cuda.synchronize()
    print("clip / ema: finite", bool(torch.isfinite(n)), flush=True)


def train72():
    """head_dim 72 kernels of the attention backward (spatial 64-token tiles, temporal warp kernel) and the transposing fallbacks."""
    from latte_b200.train_ops import NativeOps
    ops_ = NativeOps(torch.bfloat16)
    g = torch.Generator().manual_seed(4)
    for (b, f, n, h, hd, temporal) in [(1, 2, 128, 2, 72, False), (1, 16, 64, 3, 72, True), (1, 8, 64, 2, 64, True)]:
        T, D = b * f * n, h * hd
        qkv = torch.randn(T, 3 * D, generator=g).to(dev).bfloat16()
        do = torch.randn(T, D, generator=g).to(dev).bfloat16()
        o = ops_.attention(qkv, b, f, n, h, temporal)
        dq = ops_.attention_bwd(qkv, o, do, b, f, n, h, temporal)
        torch.cuda.synchronize()
        print(f"attn_bwd {'temporal' if temporal else 'spatial'} hd {hd}: finite", bool(torch.isfinite(dq.float()).all()), flush=True)
    dy = torch.randn(512, 192, generator=g).to(dev).bfloat16()
    x = torch.randn(512, 576, generator=g).to(dev).bfloat16()
    w = torch.randn(192, 576, generator=g).to(dev).bfloat16()
    gw = ops_.wgrad(torch.zeros(192, 576, device=dev), dy, x)             # n_in = 576: transposing fallback
    gx = ops_.dgrad(dy, w)
    torch.cuda.synchronize()
    print("fallback wgrad / dgrad: max err", (gw - dy.float().t() @ x.float()).abs().max().item(), (gx.float() - dy.float() @ w.float()).abs().max().item(), flush=True)


def vae_enc():
    from latte_b200 import AutoencoderKL
    from oracle import vae_oracle as V
    cfg = V.VaeConfig(block_out_channels=(64, 128, 128), norm_num_groups=16)
    sd = V.make_weights(cfg, 9)
    vae = AutoencoderKL(block_out_channels=(64, 128, 128), norm_num_groups=16)
    vae.load_state_dict(sd, strict=True)
    vae = vae.to(dev).eval()
    x = torch.rand(1, 3, 128, 128, generator=torch.Generator().manual_seed(1)) * 2 - 1
    with torch.no_grad():
        got = vae.encode(x.to(dev)).latent_dist.parameters.cpu()
    print("vae encode: max err", (got - V.vae_encode(sd, cfg, x)).abs().max().item(), flush=True)


if __name__ == "__main__":
    which = sys.argv[1:] or ["latte", "gemm", "attn", "t2v", "vae", "sampler", "train", "train72", "vae_enc"]
    for w in which:
        {"latte": latte, "gemm": gemm, "attn": attn, "t2v": t2v, "vae": vae, "sampler": sampler, "train": train, "train72": train72,
         "vae_enc": vae_enc}[w]()
