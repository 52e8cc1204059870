"""`Latte` — the reference's denoiser module surface, backed by hand-written sm_90a CUDA.

Mirrors the public interface of Vchitect/Latte `models/latte.py`:
  * constructor signature and attribute names                       (latte.py:208-232)
  * parameter names / shapes, so reference checkpoints load unchanged (SURVEY.md App. B;
    `sample/sample.py:62-64` -> `load_state_dict`, `train.py:121,263` deepcopy / state_dict)
  * `forward(x, t, y=None, text_embedding=None, use_fp16=False)`      (latte.py:314-377)
  * `forward_with_cfg(x, t, y=None, cfg_scale=7.0, use_fp16=False)`   (latte.py:379-398)
  * `unpatchify`, the `Latte_models` table and `Latte_XL_2` ... builders (latte.py:297-310, 464-506)

Nothing is computed with torch ops: the nn.Linear / Conv2d / Embedding children are parameter
containers only.  `forward` repacks parameters once (16-bit tensor-core operands, stacked over
blocks) and makes ONE call into the C ABI (`b200_latte_forward`), which enqueues every kernel of the
step on the current CUDA stream.  There is no CPU path: a CPU tensor raises.
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import torch
import torch.nn as nn

from . import _lib
from .ops import quantize_rows_e4m3
from ._cache import DeviceCacheMixin
from .training import GradientCheckpointingMixin


# ------------------------------------------------------------------------------------------------
# parameter containers (names must match the reference state_dict)
# ------------------------------------------------------------------------------------------------
class _PatchEmbedParams(nn.Module):
    """Holds `proj.weight (D,C,p,p)` / `proj.bias` like timm's PatchEmbed (latte.py:233)."""

    def __init__(self, img_size, patch_size, in_chans, embed_dim):
        super().__init__()
        self.patch_size = (patch_size, patch_size)
        self.num_patches = (img_size // patch_size) ** 2
        self.proj = nn.Conv2d(in_chans, embed_dim, kernel_size=patch_size, stride=patch_size, bias=True)


class _TimestepParams(nn.Module):
    """`mlp.0` Linear(256,D), `mlp.2` Linear(D,D) (latte.py:88-96)."""

    def __init__(self, hidden_size, frequency_embedding_size=256):
        super().__init__()
        self.mlp = nn.Sequential(nn.Linear(frequency_embedding_size, hidden_size), nn.SiLU(),
                                 nn.Linear(hidden_size, hidden_size))
        self.frequency_embedding_size = frequency_embedding_size


class _LabelParams(nn.Module):
    """`embedding_table` with one extra row for the null class when dropout > 0 (latte.py:130-135)."""

    def __init__(self, num_classes, hidden_size, dropout_prob):
        super().__init__()
        self.embedding_table = nn.Embedding(num_classes + int(dropout_prob > 0), hidden_size)
        self.num_classes = num_classes
        self.dropout_prob = dropout_prob


class _AttnParams(nn.Module):
    def __init__(self, dim, num_heads):
        super().__init__()
        self.num_heads = num_heads
        self.qkv = nn.Linear(dim, dim * 3, bias=True)
        self.proj = nn.Linear(dim, dim)


class _MlpParams(nn.Module):
    def __init__(self, dim, hidden):
        super().__init__()
        self.fc1 = nn.Linear(dim, hidden)
        self.fc2 = nn.Linear(hidden, dim)


class _BlockParams(nn.Module):
    """attn.qkv / attn.proj / mlp.fc1 / mlp.fc2 / adaLN_modulation.1 (latte.py:164-175)."""

    def __init__(self, hidden_size, num_heads, mlp_ratio):
        super().__init__()
        self.attn = _AttnParams(hidden_size, num_heads)
        self.mlp = _MlpParams(hidden_size, int(hidden_size * mlp_ratio))
        self.adaLN_modulation = nn.Sequential(nn.SiLU(), nn.Linear(hidden_size, 6 * hidden_size))


class _FinalParams(nn.Module):
    def __init__(self, hidden_size, patch_size, out_channels):
        super().__init__()
        self.linear = nn.Linear(hidden_size, patch_size * patch_size * out_channels)
        self.adaLN_modulation = nn.Sequential(nn.SiLU(), nn.Linear(hidden_size, 2 * hidden_size))


def _sincos_1d(dim: int, pos: np.ndarray) -> np.ndarray:
    """[sin | cos] table with fp64 frequencies 10000^(-k/(dim/2)) (latte.py:440-457)."""
    k = np.arange(dim // 2, dtype=np.float64) / (dim / 2.0)
    ang = pos.reshape(-1).astype(np.float64)[:, None] * (1.0 / 10000 ** k)[None, :]
    return np.concatenate([np.sin(ang), np.cos(ang)], axis=1)


def _sincos_2d(dim: int, grid: int) -> np.ndarray:
    """2-D table: first half of the channels encodes the column index, second half the row index
    (the reference's meshgrid puts w first — latte.py:416-419,433-437)."""
    coords = np.arange(grid, dtype=np.float32)
    ww, hh = np.meshgrid(coords, coords)
    return np.concatenate([_sincos_1d(dim // 2, ww), _sincos_1d(dim // 2, hh)], axis=1)


class Latte(GradientCheckpointingMixin, DeviceCacheMixin, nn.Module):
    """Diffusion transformer with alternating spatial / temporal blocks (reference latte.py:204-398)."""

    def __init__(self, input_size=32, patch_size=2, in_channels=4, hidden_size=1152, depth=28, num_heads=16,
                 mlp_ratio=4.0, num_frames=16, class_dropout_prob=0.1, num_classes=1000, learn_sigma=True,
                 extras=1, attention_mode="math"):
        super().__init__()
        if attention_mode != "math":
            # 'flash' is numerically wrong in the reference and 'xformers' needs an absent lib (SURVEY.md F4)
            raise NotImplementedError("latte_b200 implements the reference's default 'math' attention semantics only")
        if extras not in (1, 2):
            raise NotImplementedError("extras=78 (legacy CLIP text conditioning) is outside the built hot path")
        self.learn_sigma = learn_sigma
        self.in_channels = in_channels
        self.out_channels = in_channels * 2 if learn_sigma else in_channels
        self.patch_size = patch_size
        self.num_heads = num_heads
        self.extras = extras
        self.num_frames = num_frames
        self.hidden_size = hidden_size
        self.input_size = input_size
        self.depth = depth
        self.mlp_hidden = int(hidden_size * mlp_ratio)
        self.attention_mode = attention_mode
        #: tensor-core operand type used when the parameters are fp32 (fp16 = the reference's `use_fp16` path)
        self.compute_dtype = torch.float16
        #: operand type of the training step with fp32 parameters outside autocast (train.py runs under bf16 autocast)
        self.train_dtype = torch.bfloat16

        self.x_embedder = _PatchEmbedParams(input_size, patch_size, in_channels, hidden_size)
        self.t_embedder = _TimestepParams(hidden_size)
        if extras == 2:
            self.y_embedder = _LabelParams(num_classes, hidden_size, class_dropout_prob)
        n = self.x_embedder.num_patches
        self.pos_embed = nn.Parameter(torch.zeros(1, n, hidden_size), requires_grad=False)
        self.temp_embed = nn.Parameter(torch.zeros(1, num_frames, hidden_size), requires_grad=False)
        self.blocks = nn.ModuleList([_BlockParams(hidden_size, num_heads, mlp_ratio) for _ in range(depth)])
        self.final_layer = _FinalParams(hidden_size, patch_size, self.out_channels)
        self.initialize_weights()
        self._packed = None
        self._packed_key = None
        self._trajectory = None
        self._workspace = None
        self._graphs = None
        self._frozen = None
        self._train_backend = None
        self._train_operands = None
        #: eval-mode calls replay a CUDA graph of the whole forward (captured per (batch, cfg) signature on its second
        #: use; results are bit-identical to the eager launch sequence).  Set False to always launch eagerly.
        self.use_cuda_graphs = True
        #: sampling runs QKV and fc1 -- the two GEMMs fed by LayerNorm + modulate -- with FP8 (e4m3) tensor-core operands:
        #: per-token activation scales, per-output-channel weight scales, fp32 accumulation.  Every other operand keeps the
        #: 16-bit type.  Eval / no-grad calls only; a training forward raises.  Toggling it repacks the weights.
        self.use_fp8 = False
        #: training steps keep each block's input only and rerun the block in the backward (`enable_gradient_checkpointing`)
        self.gradient_checkpointing = False

    # -------------------------------------------------------------------------------------------
    def initialize_weights(self):
        """Same initial distribution as the reference (latte.py:257-295): xavier-uniform Linears with
        zero bias, fixed sin-cos tables, N(0, 0.02) label / timestep MLP weights, adaLN-Zero."""
        for m in self.modules():
            if isinstance(m, nn.Linear):
                nn.init.xavier_uniform_(m.weight)
                nn.init.zeros_(m.bias)
        grid = int(self.x_embedder.num_patches ** 0.5)
        self.pos_embed.data.copy_(torch.from_numpy(_sincos_2d(self.hidden_size, grid)).float()[None])
        self.temp_embed.data.copy_(torch.from_numpy(
            _sincos_1d(self.hidden_size, np.arange(self.num_frames))).float()[None])
        w = self.x_embedder.proj.weight.data
        nn.init.xavier_uniform_(w.view(w.shape[0], -1))
        nn.init.zeros_(self.x_embedder.proj.bias)
        if self.extras == 2:
            nn.init.normal_(self.y_embedder.embedding_table.weight, std=0.02)
        nn.init.normal_(self.t_embedder.mlp[0].weight, std=0.02)
        nn.init.normal_(self.t_embedder.mlp[2].weight, std=0.02)
        for blk in self.blocks:
            nn.init.zeros_(blk.adaLN_modulation[-1].weight)
            nn.init.zeros_(blk.adaLN_modulation[-1].bias)
        for p in (self.final_layer.adaLN_modulation[-1].weight, self.final_layer.adaLN_modulation[-1].bias,
                  self.final_layer.linear.weight, self.final_layer.linear.bias):
            nn.init.zeros_(p)

    def unpatchify(self, x):
        """(n, T, p*p*c) -> (n, c, h*p, w*p) (latte.py:297-310).  Host-side utility kept for API parity;
        the CUDA final-layer kernel scatters directly into this layout."""
        c, p = self.out_channels, self.patch_size
        h = w = int(x.shape[1] ** 0.5)
        assert h * w == x.shape[1]
        return x.reshape(x.shape[0], h, w, p, p, c).permute(0, 5, 1, 3, 2, 4).reshape(x.shape[0], c, h * p, w * p)

    # -------------------------------------------------------------------------------------------
    def _operand_dtype(self) -> torch.dtype:
        pd = self.blocks[0].attn.qkv.weight.dtype
        if pd in (torch.float16, torch.bfloat16):
            return pd
        return self.compute_dtype

    def _pack_key(self):
        w0 = self.blocks[0].attn.qkv.weight
        ver = 0
        for p in self.parameters():
            ver += p._version
        return (ver, w0.data_ptr(), w0.device, w0.dtype, self.compute_dtype, bool(self.use_fp8))

    def repack(self):
        """Drop the packed operand cache (call after mutating parameters through `.data`)."""
        self._packed = None
        self._packed_key = None
        self._graphs = None
        self._frozen = None

    @torch.no_grad()
    def _pack(self):
        if self._frozen is not None:          # inside a sampling loop (precompute_conditioning .. clear_conditioning)
            if (self._frozen[2].get("qkv_w8") is not None) == bool(self.use_fp8):
                return self._frozen
            # use_fp8 was toggled inside the loop: pack in the new mode (the precomputed conditioning rows do not depend on
            # it) and keep that packing for the rest of the loop
            self._frozen = None
            self._frozen = self._pack()
            return self._frozen
        key = self._pack_key()
        if self._packed is not None and key == self._packed_key:
            return self._packed
        self._graphs = None                   # captured graphs hold pointers into the previous packing
        dev = self.pos_embed.device
        od = self._operand_dtype()
        f32 = lambda t: t.detach().to(device=dev, dtype=torch.float32).contiguous()
        D = self.hidden_size
        blocks = list(self.blocks)
        T = {}
        T["patch_w"] = f32(self.x_embedder.proj.weight).reshape(D, -1).contiguous()
        T["patch_b"] = f32(self.x_embedder.proj.bias)
        T["pos_embed"] = f32(self.pos_embed).reshape(-1, D).contiguous()
        T["temp_embed"] = f32(self.temp_embed).reshape(-1, D).contiguous()
        T["t_w0"] = f32(self.t_embedder.mlp[0].weight)
        T["t_b0"] = f32(self.t_embedder.mlp[0].bias)
        T["t_w2"] = f32(self.t_embedder.mlp[2].weight)
        T["t_b2"] = f32(self.t_embedder.mlp[2].bias)
        T["y_table"] = f32(self.y_embedder.embedding_table.weight) if self.extras == 2 else None
        stack16 = lambda ts: torch.stack([t.detach() for t in ts]).to(device=dev, dtype=od).contiguous()
        cat32 = lambda ts: torch.cat([t.detach().reshape(-1) for t in ts]).to(device=dev, dtype=torch.float32).contiguous()
        T["ada_w16"] = torch.cat([b.adaLN_modulation[1].weight.detach() for b in blocks] +
                                 [self.final_layer.adaLN_modulation[1].weight.detach()]).to(device=dev, dtype=od).contiguous()
        T["ada_b"] = cat32([b.adaLN_modulation[1].bias for b in blocks] + [self.final_layer.adaLN_modulation[1].bias])
        # with use_fp8 the forward reads only the e4m3 copies of QKV and fc1 (below), so no 16-bit ones are made
        T["qkv_w16"] = None if self.use_fp8 else stack16([b.attn.qkv.weight for b in blocks])
        T["qkv_b"] = cat32([b.attn.qkv.bias for b in blocks])
        T["proj_w16"] = stack16([b.attn.proj.weight for b in blocks])
        T["proj_b"] = cat32([b.attn.proj.bias for b in blocks])
        T["fc1_w16"] = None if self.use_fp8 else stack16([b.mlp.fc1.weight for b in blocks])
        T["fc1_b"] = cat32([b.mlp.fc1.bias for b in blocks])
        T["fc2_w16"] = stack16([b.mlp.fc2.weight for b in blocks])
        T["fc2_b"] = cat32([b.mlp.fc2.bias for b in blocks])
        T["final_w"] = f32(self.final_layer.linear.weight)
        T["final_b"] = f32(self.final_layer.linear.bias)
        T["final_w16"] = self.final_layer.linear.weight.detach().to(device=dev, dtype=od).contiguous()
        for name in ("qkv_w8", "qkv_ws", "fc1_w8", "fc1_ws"):
            T[name] = None
        if self.use_fp8:
            # ONE quantization call for every QKV and fc1 weight (the same width D): rows [0, depth*3D) are QKV, stacked over
            # blocks like the 16-bit copies, then fc1; one scale per output channel (b200_quantize_rows_e4m3)
            w32 = torch.cat([b.attn.qkv.weight.detach() for b in blocks] + [b.mlp.fc1.weight.detach() for b in blocks]).to(
                device=dev, dtype=torch.float32).contiguous()
            q8, ws8 = quantize_rows_e4m3(w32)
            q8, nq = q8.view(torch.uint8), self.depth * 3 * D
            T["qkv_w8"], T["fc1_w8"] = q8[:nq], q8[nq:]
            T["qkv_ws"], T["fc1_ws"] = ws8[:nq], ws8[nq:]

        w = _lib.LatteWeights()
        for name in _lib.WEIGHT_FIELDS:
            t = T[name]
            setattr(w, name, t.data_ptr() if t is not None else None)
        shape = _lib.LatteShape(
            depth=self.depth, hidden=D, heads=self.num_heads, mlp_hidden=self.mlp_hidden, patch=self.patch_size,
            in_channels=self.in_channels, out_channels=self.out_channels, input_size=self.input_size,
            frames=self.num_frames,
            num_embed=(self.y_embedder.embedding_table.weight.shape[0] if self.extras == 2 else 0),
            dtype=_lib.BF16 if od == torch.bfloat16 else _lib.FP16, wide_patch=1)
        self._packed = (shape, w, T, od)  # T keeps the device tensors alive
        self._packed_key = key
        return self._packed

    def _check_input(self, x):
        if x.dim() != 5 or x.shape[1] != self.num_frames or x.shape[2] != self.in_channels \
                or x.shape[3] != self.input_size or x.shape[4] != self.input_size:
            raise ValueError(f"x must be (B, {self.num_frames}, {self.in_channels}, {self.input_size}, {self.input_size}), got {tuple(x.shape)}")
        if self.pos_embed.device != x.device:
            raise RuntimeError(f"model is on {self.pos_embed.device}, input on {x.device}")

    def _labels(self, y, B, dev):
        """Class labels as int64 on `dev` (None unless extras == 2), with the reference's label dropout in training mode."""
        if self.extras != 2:
            return None
        if y is None:
            raise ValueError("class-conditional model (extras=2) needs labels y")
        yy = y.detach().to(device=dev, dtype=torch.int64).contiguous()
        if self.training and self.y_embedder.dropout_prob > 0:  # token_drop, latte.py:137-146
            drop = torch.rand(B, device=dev) < self.y_embedder.dropout_prob
            yy = torch.where(drop, torch.full_like(yy, self.y_embedder.num_classes), yy)
        return yy

    def _run(self, x, t, y, use_cfg, cfg_scale, trajectory_step=None):
        if not x.is_cuda:
            raise RuntimeError("latte_b200.Latte runs on CUDA (sm_90a) only; there is no CPU fallback "
                               "(the CPU truth lives in oracle/, which is test infrastructure)")
        if torch.is_grad_enabled() and self.training and any(p.requires_grad for p in self.parameters()):
            if use_cfg or trajectory_step is not None:
                raise NotImplementedError("latte_b200: forward_with_cfg / trajectory conditioning are sampling-only; train through forward()")
            return self._run_train(x, t, y)
        self._check_input(x)
        lib = _lib.load()
        dev = x.device
        B = x.shape[0]
        with torch.cuda.device(dev):
            shape, w, _, od = self._pack()
            xf = x.detach().to(torch.float32).contiguous()
            tt = t.detach().to(device=dev, dtype=torch.int64).contiguous()
            if tt.numel() != B:
                raise ValueError("t must have one entry per batch row")
            yy = self._labels(y, B, dev)
            traj = self._trajectory
            mod = None
            if trajectory_step is not None and traj is not None:
                mod = traj[int(trajectory_step)]                    # [B, depth*6D + 2D] rows precomputed for this step
                if mod.shape[0] != B or mod.device != dev:
                    raise ValueError("precomputed conditioning does not match this batch")
            need = lib.b200_latte_workspace_bytes(C.byref(shape), B)
            if need == 0:
                raise RuntimeError("latte_b200: unsupported configuration: " + _lib.last_error())
            if (self.use_cuda_graphs and not torch.is_grad_enabled() and not torch.cuda.is_current_stream_capturing()
                    and not _lib.profiling_enabled()):
                out = self._run_graphed(lib, shape, w, xf, tt, yy, mod, B, use_cfg, cfg_scale, need, dev)
            else:
                out = torch.empty(B, self.num_frames, self.out_channels, self.input_size, self.input_size,
                                  dtype=torch.float32, device=dev)
                self._launch(lib, shape, w, xf, tt, yy, mod, B, use_cfg, cfg_scale, out, self._aligned_workspace(need, dev), need,
                             torch.cuda.current_stream(dev).cuda_stream)
        pd = self.blocks[0].attn.qkv.weight.dtype
        return out if pd == torch.float32 else out.to(pd)

    def _run_train(self, x, t, y):
        """Training-mode forward (`model.train()` with grad enabled, train.py:206-222): the native forward that keeps its
        activations, with the hand-written backward attached as one autograd node (latte_b200/training.py), so the reference's
        `loss.backward()`, optimizer, `clip_grad_norm_` and DistributedDataParallel work unchanged.  Operands are bf16 under
        `torch.autocast(bfloat16)` / fp32 parameters (the reference's mixed-precision recipe) or the parameter dtype if that is
        16-bit; accumulation, the residual stream, LayerNorm statistics and every gradient buffer are fp32."""
        from . import training
        if self.use_fp8:
            raise NotImplementedError("latte_b200: FP8 is a sampling path; clear use_fp8 to train")
        self._check_input(x)
        dev = x.device
        _lib.load()
        od, ops = training.native_backend(self, self.blocks[0].attn.qkv.weight.dtype)
        B = x.shape[0]
        tt = t.to(device=dev, dtype=torch.int64)
        yy = self._labels(y, B, dev)
        with torch.autocast("cuda", enabled=False):
            c = training.conditioning(self, tt, yy)
            return training.train_forward(self, ops, od, x.float(), c)

    def _launch(self, lib, shape, w, xf, tt, yy, mod, B, use_cfg, cfg_scale, out, base, need, stream):
        """ONE C-ABI call = the whole forward (206 kernel launches for XL/2 with CFG) enqueued on `stream`."""
        if mod is not None:
            rc = lib.b200_latte_forward_conditioned(C.byref(shape), C.byref(w), xf.data_ptr(), mod.data_ptr(), B, int(use_cfg),
                                                    float(cfg_scale), out.data_ptr(), base, need, stream)
            _lib.check(rc, "b200_latte_forward_conditioned")
        else:
            rc = lib.b200_latte_forward(C.byref(shape), C.byref(w), xf.data_ptr(), tt.data_ptr(),
                                        yy.data_ptr() if yy is not None else None, B, int(use_cfg), float(cfg_scale),
                                        out.data_ptr(), base, need, stream)
            _lib.check(rc, "b200_latte_forward")

    def _run_graphed(self, lib, shape, w, xf, tt, yy, mod, B, use_cfg, cfg_scale, need, dev):
        """CUDA-graph replay of the forward.  The C-ABI call neither allocates nor synchronises and keeps no host-side launch
        state, so its launch sequence can be captured once per call signature and replayed with the inputs copied into
        fixed buffers: the per-step host cost drops from ~200 launches to three small copies and one graph launch.
        First use of a signature runs eagerly (it also sets per-device kernel attributes), the second captures."""
        key = (B, bool(use_cfg), float(cfg_scale), yy is not None, mod is not None, dev, bool(self.use_fp8))
        if self._graphs is None:
            self._graphs = {}
        st = self._graphs.get(key)
        if st is None:
            self._graphs[key] = {"graph": None}
            out = torch.empty(B, self.num_frames, self.out_channels, self.input_size, self.input_size,
                              dtype=torch.float32, device=dev)
            self._launch(lib, shape, w, xf, tt, yy, mod, B, use_cfg, cfg_scale, out, self._aligned_workspace(need, dev), need,
                         torch.cuda.current_stream(dev).cuda_stream)
            return out
        if st["graph"] is None:
            st["ws"] = torch.empty(need + 1024, dtype=torch.uint8, device=dev)     # this graph's own scratch
            st["x"], st["t"] = torch.empty_like(xf), torch.empty_like(tt)
            st["y"] = torch.empty_like(yy) if yy is not None else None
            st["mod"] = torch.empty_like(mod) if mod is not None else None
            st["out"] = torch.empty(B, self.num_frames, self.out_channels, self.input_size, self.input_size,
                                    dtype=torch.float32, device=dev)
            base = (st["ws"].data_ptr() + 1023) // 1024 * 1024
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._launch(lib, shape, w, st["x"], st["t"], st["y"], st["mod"], B, use_cfg, cfg_scale, st["out"], base, need,
                             torch.cuda.current_stream(dev).cuda_stream)
            st["graph"] = g
        st["x"].copy_(xf)
        st["t"].copy_(tt)
        if yy is not None:
            st["y"].copy_(yy)
        if mod is not None:
            st["mod"].copy_(mod)
        st["graph"].replay()
        return st["out"].clone()

    def forward(self, x, t, y=None, text_embedding=None, use_fp16=False, trajectory_step=None):
        """x (N,F,C,H,W), t (N,), y (N,) -> (N,F,out_channels,H,W) (latte.py:314-377).  `use_fp16` is accepted for
        call compatibility; the operand precision follows the parameter dtype (`.half()` as in sample.py:72-75).
        `trajectory_step` (not in the reference): use row `trajectory_step` of `precompute_conditioning` instead of (t, y)."""
        if text_embedding is not None:
            raise NotImplementedError("text_embedding (extras=78) is outside the built hot path")
        return self._run(x, t, y, False, 0.0, trajectory_step)

    def forward_with_cfg(self, x, t, y=None, cfg_scale=7.0, use_fp16=False, text_embedding=None, trajectory_step=None):
        """Classifier-free guidance variant (latte.py:379-398): the first half of `x` is run with (t, y) of both
        halves; eps channels [:in_channels] of both halves become uncond + s * (cond - uncond)."""
        if text_embedding is not None:
            raise NotImplementedError("text_embedding (extras=78) is outside the built hot path")
        return self._run(x, t, y, True, float(cfg_scale), trajectory_step)

    # ------------------------------------------------------------------ whole-trajectory conditioning (SURVEY.md 8f rank 2)
    def precompute_conditioning(self, timesteps, y=None):
        """The conditioning path (t_embedder + y_embedder, latte.py:332-339; every adaLN_modulation, :160-163,192-195) depends
        only on (t, y).  `timesteps` (steps, B) int64 = the ORIGINAL timesteps the sampler will feed, step by step; `y` (B,).
        Evaluates all steps * B rows once (same kernels and arithmetic as inside forward -> bit-identical outputs) and keeps
        them on the device; `forward*(…, trajectory_step=i)` then skips the 446 MB/step adaLN weight stream.  Used by
        latte_b200.diffusion's loops; `clear_conditioning()` drops the cache."""
        lib = _lib.load()
        dev = self.pos_embed.device
        if dev.type != "cuda":
            raise RuntimeError("latte_b200.Latte runs on CUDA (sm_90a) only; there is no CPU fallback")
        steps, B = timesteps.shape
        with torch.cuda.device(dev):
            shape, w, _, _ = self._pack()
            tt = timesteps.detach().to(device=dev, dtype=torch.int64).contiguous().view(-1)
            yy = None
            if self.extras == 2:
                if y is None:
                    raise ValueError("class-conditional model (extras=2) needs labels y")
                yy = y.detach().to(device=dev, dtype=torch.int64).view(1, B).expand(steps, B).contiguous().view(-1)
            n = steps * B
            row = lib.b200_latte_conditioning_bytes(C.byref(shape), 1) // 4
            if row == 0:
                raise RuntimeError("latte_b200: unsupported configuration: " + _lib.last_error())
            mod = torch.empty(n * row + 256, dtype=torch.float32, device=dev)
            off = (-(mod.data_ptr() // 4)) % 256                      # 1024-byte aligned start
            mod = mod[off:off + n * row]
            need = lib.b200_latte_conditioning_workspace_bytes(C.byref(shape), n)
            ws = torch.empty(need + 1024, dtype=torch.uint8, device=dev)
            base = (ws.data_ptr() + 1023) // 1024 * 1024
            rc = lib.b200_latte_conditioning(C.byref(shape), C.byref(w), tt.data_ptr(), yy.data_ptr() if yy is not None else None,
                                             n, mod.data_ptr(), base, need, torch.cuda.current_stream(dev).cuda_stream)
            _lib.check(rc, "b200_latte_conditioning")
            ws.record_stream(torch.cuda.current_stream(dev))
        self._trajectory = mod.view(steps, B, row)
        self._frozen = self._packed      # the loop's steps reuse this packing without re-walking the 293 parameters
        return self._trajectory

    def conditioning_row_bytes(self) -> int:
        """Bytes of precomputed conditioning per (step, sample): (depth*6 + 2) * hidden fp32."""
        return (self.depth * 6 + 2) * self.hidden_size * 4

    def clear_conditioning(self):
        self._trajectory = None
        self._frozen = None


# ------------------------------------------------------------------------------------------------
# size table (latte.py:464-506)
# ------------------------------------------------------------------------------------------------
def _mk(depth, hidden, patch, heads):
    def build(**kwargs):
        return Latte(depth=depth, hidden_size=hidden, patch_size=patch, num_heads=heads, **kwargs)
    return build


Latte_XL_2, Latte_XL_4, Latte_XL_8 = _mk(28, 1152, 2, 16), _mk(28, 1152, 4, 16), _mk(28, 1152, 8, 16)
Latte_L_2, Latte_L_4, Latte_L_8 = _mk(24, 1024, 2, 16), _mk(24, 1024, 4, 16), _mk(24, 1024, 8, 16)
Latte_B_2, Latte_B_4, Latte_B_8 = _mk(12, 768, 2, 12), _mk(12, 768, 4, 12), _mk(12, 768, 8, 12)
Latte_S_2, Latte_S_4, Latte_S_8 = _mk(12, 384, 2, 6), _mk(12, 384, 4, 6), _mk(12, 384, 8, 6)

Latte_models = {
    "Latte-XL/2": Latte_XL_2, "Latte-XL/4": Latte_XL_4, "Latte-XL/8": Latte_XL_8,
    "Latte-L/2": Latte_L_2, "Latte-L/4": Latte_L_4, "Latte-L/8": Latte_L_8,
    "Latte-B/2": Latte_B_2, "Latte-B/4": Latte_B_4, "Latte-B/8": Latte_B_8,
    "Latte-S/2": Latte_S_2, "Latte-S/4": Latte_S_4, "Latte-S/8": Latte_S_8,
}
