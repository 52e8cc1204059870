"""`LatteIMG` — video + image joint training (reference models/latte_img.py, trained by train_with_img.py).

Same parameters as `Latte` (checkpoints are interchangeable); `forward(x, t, y=None, use_fp16=False, y_image=None,
use_image_num=0)` takes x (B, F + I, C, H, W): F = num_frames video frames, then I = use_image_num still images per sample.
Spatial blocks and the final layer run over all F + I frames, each conditioned on t_b + its own label (the video label y_b for
video frames, y_image[b][i] for image i when extras == 2); temporal blocks and temp_embed see the video frames only
(latte_img.py:316-399).

With use_image_num == 0 every call is `Latte`'s, unchanged (sampling, forward_with_cfg, CUDA graphs, trajectory conditioning,
the training step).  With images, a training-mode call with grad enabled is one native step of latte_b200/training.py behind one
autograd node; other calls run the same engine's forward without keeping activations.
"""
from __future__ import annotations

from collections.abc import Sequence

import torch

from . import _lib
from .latte import Latte


class LatteIMG(Latte):
    def __init__(self, input_size=32, patch_size=2, in_channels=4, hidden_size=1152, depth=28, num_heads=16,
                 mlp_ratio=4.0, num_frames=16, class_dropout_prob=0.1, num_classes=1000, learn_sigma=True,
                 extras=2, attention_mode="math"):
        super().__init__(input_size=input_size, patch_size=patch_size, in_channels=in_channels, hidden_size=hidden_size,
                         depth=depth, num_heads=num_heads, mlp_ratio=mlp_ratio, num_frames=num_frames,
                         class_dropout_prob=class_dropout_prob, num_classes=num_classes, learn_sigma=learn_sigma,
                         extras=extras, attention_mode=attention_mode)

    def forward(self, x, t, y=None, use_fp16=False, y_image=None, use_image_num=0, text_embedding=None, trajectory_step=None):
        """x (B, F + I, C, H, W), t (B,), y (B,), y_image: B label tensors of I entries (train_with_img.py) or a (B, I) tensor
        -> (B, F + I, out_channels, H, W) (latte_img.py:316-399)."""
        I = int(use_image_num)
        if I == 0:
            return super().forward(x, t, y, text_embedding=text_embedding, use_fp16=use_fp16, trajectory_step=trajectory_step)
        if text_embedding is not None:
            raise NotImplementedError("text_embedding (extras=78) is outside the built hot path")
        if self.use_fp8:
            # frames with images run the training engine's 16-bit forward (training and eval alike): no silent fallback
            raise NotImplementedError("latte_b200: FP8 is a sampling path of the video forward; LatteIMG with images "
                                      "(use_image_num > 0) has none -- clear use_fp8")
        if trajectory_step is not None:
            raise ValueError("latte_b200: trajectory conditioning is a sampling path; it takes no images (use_image_num = 0)")
        if I < 0:
            raise ValueError(f"use_image_num must be >= 0, got {use_image_num}")
        train_step = torch.is_grad_enabled() and self.training and any(p.requires_grad for p in self.parameters())
        if self.extras == 2 and not self.training:
            raise ValueError("LatteIMG with extras=2 has no image labels in eval mode: the reference conditions image frames on "
                             "y_image only in training mode (latte_img.py:336-348); call with use_image_num=0 or model.train()")
        want = (self.num_frames + I, self.in_channels, self.input_size, self.input_size)
        if x.dim() != 5 or tuple(x.shape[1:]) != want:
            raise ValueError(f"x must be (B, num_frames + use_image_num = {self.num_frames} + {I}, {self.in_channels}, "
                             f"{self.input_size}, {self.input_size}), got {tuple(x.shape)}")
        dev = x.device
        B = x.shape[0]
        tt = torch.as_tensor(t).to(device=dev, dtype=torch.int64).reshape(-1)
        if tt.numel() != B:
            raise ValueError("t must have one entry per batch row")
        yy = yi = None
        if self.extras == 2:
            if y is None:
                raise ValueError("class-conditional model (extras=2) needs labels y")
            yy = torch.as_tensor(y).to(device=dev, dtype=torch.int64).reshape(-1)
            if yy.numel() != B:
                raise ValueError("y must have one label per batch row")
            yi = self._image_labels(y_image, B, I, dev)
            if self.y_embedder.dropout_prob > 0:
                # token_drop (latte_img.py:140-149): one draw per video, one per sample's image set (all I labels together)
                p, null = self.y_embedder.dropout_prob, self.y_embedder.num_classes
                yy = torch.where(torch.rand(B, device=dev) < p, torch.full_like(yy, null), yy)
                yi = torch.where((torch.rand(B, device=dev) < p)[:, None], torch.full_like(yi, null), yi)
        if not x.is_cuda:
            raise RuntimeError("latte_b200.LatteIMG runs on CUDA (sm_90a) only; there is no CPU fallback")
        if self.pos_embed.device != dev:
            raise RuntimeError(f"model is on {self.pos_embed.device}, input on {dev}")
        from . import training
        _lib.load()
        od, ops = training.native_backend(self, self.blocks[0].attn.qkv.weight.dtype)
        with torch.autocast("cuda", enabled=False):
            if train_step:
                c = training.frame_conditioning(self, tt, yy, yi, I)
                return training.train_forward(self, ops, od, x.float(), c, images=I)
            with torch.no_grad():
                c = training.frame_conditioning(self, tt, yy, yi, I)
                out = training.image_forward(self, ops, od, x, c, I)
        pd = self.blocks[0].attn.qkv.weight.dtype
        return out if pd == torch.float32 else out.to(pd)

    @staticmethod
    def _image_labels(y_image, B, I, dev):
        """B label tensors of I entries each (train_with_img.py:216-220) or a (B, I) tensor -> (B, I) int64 on `dev`."""
        if y_image is None:
            raise ValueError("LatteIMG with extras=2 in training mode needs y_image: I labels per sample")
        if isinstance(y_image, torch.Tensor):
            yi = y_image
        elif isinstance(y_image, Sequence) and len(y_image) == B:
            rows = [torch.as_tensor(r).reshape(-1) for r in y_image]
            if any(r.numel() != I for r in rows):
                raise ValueError(f"every entry of y_image must hold use_image_num = {I} labels, got {[r.numel() for r in rows]}")
            yi = torch.stack([r.to(dev) for r in rows])
        else:
            raise ValueError(f"y_image must be a sequence of B = {B} label tensors or a (B, I) tensor")
        if tuple(yi.shape) != (B, I):
            raise ValueError(f"y_image must be (B, use_image_num) = ({B}, {I}), got {tuple(yi.shape)}")
        if yi.dtype.is_floating_point or yi.dtype == torch.bool:
            raise ValueError(f"y_image holds class labels (an integer type), got {yi.dtype}")
        return yi.to(device=dev, dtype=torch.int64)


def _mk(depth, hidden, patch, heads):
    def build(**kwargs):
        return LatteIMG(depth=depth, hidden_size=hidden, patch_size=patch, num_heads=heads, **kwargs)
    return build


LatteIMG_XL_2, LatteIMG_XL_4, LatteIMG_XL_8 = _mk(28, 1152, 2, 16), _mk(28, 1152, 4, 16), _mk(28, 1152, 8, 16)
LatteIMG_L_2, LatteIMG_L_4, LatteIMG_L_8 = _mk(24, 1024, 2, 16), _mk(24, 1024, 4, 16), _mk(24, 1024, 8, 16)
LatteIMG_B_2, LatteIMG_B_4, LatteIMG_B_8 = _mk(12, 768, 2, 12), _mk(12, 768, 4, 12), _mk(12, 768, 8, 12)
LatteIMG_S_2, LatteIMG_S_4, LatteIMG_S_8 = _mk(12, 384, 2, 6), _mk(12, 384, 4, 6), _mk(12, 384, 8, 6)

# latte_img.py:524-529
LatteIMG_models = {
    "LatteIMG-XL/2": LatteIMG_XL_2, "LatteIMG-XL/4": LatteIMG_XL_4, "LatteIMG-XL/8": LatteIMG_XL_8,
    "LatteIMG-L/2": LatteIMG_L_2, "LatteIMG-L/4": LatteIMG_L_4, "LatteIMG-L/8": LatteIMG_L_8,
    "LatteIMG-B/2": LatteIMG_B_2, "LatteIMG-B/4": LatteIMG_B_4, "LatteIMG-B/8": LatteIMG_B_8,
    "LatteIMG-S/2": LatteIMG_S_2, "LatteIMG-S/4": LatteIMG_S_4, "LatteIMG-S/8": LatteIMG_S_8,
}
