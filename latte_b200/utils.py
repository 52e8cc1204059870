"""`clip_grad_norm_` and `update_ema` with the reference's signatures (utils.py:72-125, 190-200; called at train.py:226-235,163).

The reference walks the parameter list in python -- two small kernels per tensor, ~1200 launches per optimisation step for
Latte-XL/2's 293 tensors.  Here each function is one or two launches of a multi-tensor kernel (csrc/train.cu:
`multi_tensor_kernel`) over a device-resident pointer table that is cached for as long as the tensors stay where they are; the
clip coefficient is computed and applied on the device, so neither function synchronises the host.  CUDA tensors only."""
from __future__ import annotations

from collections import OrderedDict

import torch

from . import _lib

MT_SUMSQ, MT_SCALE, MT_AXPBY = 1, 2, 3
_CHUNK = 4096
_tables: "OrderedDict[tuple, tuple]" = OrderedDict()


def _table(srcs, dsts):
    key = tuple(t.data_ptr() if t is not None else 0 for t in srcs) + tuple(t.data_ptr() if t is not None else 0 for t in dsts) + \
        tuple(t.numel() for t in (srcs if srcs[0] is not None else dsts))
    hit = _tables.get(key)
    if hit is not None:
        _tables.move_to_end(key)
        return hit
    rows, first, dev = [], 0, None
    for a, b in zip(srcs, dsts):
        t = a if a is not None else b
        if not t.is_cuda:
            raise RuntimeError("latte_b200.utils runs on CUDA tensors only; there is no CPU fallback")
        if t.dtype != torch.float32 or not t.is_contiguous() or (a is not None and b is not None and (a.shape != b.shape or b.dtype != torch.float32
                                                                                                     or not b.is_contiguous())):
            raise TypeError("latte_b200.utils: contiguous float32 tensors of matching shapes expected")
        dev = t.device
        n = t.numel()
        rows.append([a.data_ptr() if a is not None else 0, b.data_ptr() if b is not None else 0, n, first])
        first += (n + _CHUNK - 1) // _CHUNK
    host = torch.tensor(rows, dtype=torch.int64).pin_memory()        # async upload: building a table never stalls the host on the GPU
    out = (host.to(dev, non_blocking=True), len(rows), first, dev, host)
    _tables[key] = out
    while len(_tables) > 8:
        _tables.popitem(last=False)
    return out


def _run(op, srcs, dsts, a=0.0, b=0.0, scalar=None, accum=None):
    table, n, total, dev, _ = _table(srcs, dsts)
    with torch.cuda.device(dev):
        rc = _lib.load().b200_multi_tensor(table.data_ptr(), n, total, op, float(a), float(b),
                                           scalar.data_ptr() if scalar is not None else None,
                                           accum.data_ptr() if accum is not None else None, torch.cuda.current_stream(dev).cuda_stream)
    _lib.check(rc, "b200_multi_tensor")


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
    _run(MT_SUMSQ, grads, [None] * len(grads), accum=accum)
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
        _run(MT_SCALE, [None] * len(grads), grads, scalar=coef)
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
        _run(MT_AXPBY, srcs, dsts, a=decay, b=1.0 - decay)


def requires_grad(model, flag: bool = True) -> None:
    """utils.py:202-207."""
    for p in model.parameters():
        p.requires_grad = flag
