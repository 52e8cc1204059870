"""`clip_grad_norm_` and `update_ema` with the reference's signatures (utils.py:72-125, 190-200; called at train.py:226-235,163).

The reference walks the parameter list in python -- two small kernels per tensor, ~1200 launches per optimisation step for
Latte-XL/2's 293 tensors.  Here each function is one or two launches of a multi-tensor kernel (csrc/train.cu:
`multi_tensor_kernel`) over a device-resident pointer table that is cached for as long as the tensors stay where they are; the
clip coefficient is computed and applied on the device, so neither function synchronises the host.  CUDA tensors only."""
from __future__ import annotations

from collections import OrderedDict

import torch

from . import ops

MT_SUMSQ, MT_SCALE, MT_AXPBY = 1, 2, 3


def get_grad_norm(parameters, norm_type: float = 2.0) -> torch.Tensor:
    """utils.py:45-70: the 2-norm of all gradients viewed as one vector.  Each thread of the multi-tensor kernel sums its
    squares in fp32 and each warp sums its threads in fp32; one thread per block adds the block's 8 warp sums in float64 and
    adds that to the total with one float64 atomic.  The relative error therefore grows linearly with the elements per
    thread (tests/test_gpu_train_gemm_fp64.py)."""
    if isinstance(parameters, torch.Tensor):
        parameters = [parameters]
    grads = [p.grad.detach() for p in parameters if p.grad is not None]
    if float(norm_type) != 2.0:
        raise NotImplementedError("latte_b200.utils: only the 2-norm is built (what train.py uses)")
    if len(grads) == 0:
        return torch.tensor(0.)
    accum = torch.zeros(1, dtype=torch.float64, device=grads[0].device)
    ops.multi_tensor(MT_SUMSQ, grads, [None] * len(grads), accum=accum)
    return accum.sqrt().float().reshape(())


def clip_grad_norm_(parameters, max_norm: float, norm_type: float = 2.0, error_if_nonfinite: bool = False, clip_grad=True) -> torch.Tensor:
    """utils.py:72-125: returns the total norm; with `clip_grad` scales every gradient in place by min(1, max_norm / (norm + 1e-6))."""
    if isinstance(parameters, torch.Tensor):
        parameters = [parameters]
    parameters = list(parameters)
    total_norm = get_grad_norm(parameters, norm_type)
    grads = [p.grad.detach() for p in parameters if p.grad is not None]
    if clip_grad and grads:
        if error_if_nonfinite and not bool(torch.isfinite(total_norm)):
            raise RuntimeError(f"The total norm of order {norm_type} for gradients from `parameters` is non-finite, so it cannot be clipped.")
        coef = torch.clamp(float(max_norm) / (total_norm + 1e-6), max=1.0).reshape(1).contiguous()
        ops.multi_tensor(MT_SCALE, [None] * len(grads), grads, scalar=coef)
    return total_norm


@torch.no_grad()
def update_ema(ema_model, model, decay: float = 0.9999) -> None:
    """utils.py:190-200: ema = decay * ema + (1 - decay) * param for every named parameter, one launch."""
    ema_params = OrderedDict(ema_model.named_parameters())
    srcs, dsts = [], []
    for name, param in model.named_parameters():
        srcs.append(param.detach())
        dsts.append(ema_params[name].detach())
    if srcs:
        ops.multi_tensor(MT_AXPBY, srcs, dsts, a=decay, b=1.0 - decay)


def requires_grad(model, flag: bool = True) -> None:
    """utils.py:202-207."""
    for p in model.parameters():
        p.requires_grad = flag
