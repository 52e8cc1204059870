"""Host-side mirror of the reference's `diffusion` package for the SAMPLING path (SURVEY.md §8 row a20 / §8f rank 1):
`create_diffusion(str(steps))` returns an object with the reference's `ddim_sample_loop`, `p_sample_loop`, their
`*_progressive` generators, `ddim_sample`, `p_sample` and `p_mean_variance` (same names, arguments and return dicts:
diffusion/__init__.py:10-47, diffusion/gaussian_diffusion.py:254-336, 380-516, 517-689, diffusion/respace.py:65-130), so
`sample/sample.py:67,100-107` and `sample/sample_ddp.py:87,149-156` run on it unchanged.

What differs from the reference is only HOW a step is computed: the schedule tables are built once in float64 numpy (the
reference's formulas), cast to fp32 exactly as `_extract_into_tensor` does, and kept on the device; the ~40 elementwise
launches and ~12 pageable H2D copies the reference issues around every model call become ONE kernel
(`b200_sampler_step`, latte_b200/csrc/sampler.cu) and the timestep tensors are slices of device-resident tables, so a
sampling loop never synchronises the host with the GPU.  The per-step `randn_like` is still drawn in BOTH methods (the
reference consumes RNG at eta = 0 too, gaussian_diffusion.py:555).

CUDA tensors only -- there is no CPU path (the CPU truth is oracle/sampler_oracle.py, test infrastructure).
`training_losses` (MSE + learned-range VB, the objective train.py uses) is torch elementwise math with autograd around the
native forward/backward of the denoiser.  Not built (raise NotImplementedError): cond_fn / denoised_fn hooks, predict_xstart,
fixed-variance models.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import torch

from latte_b200 import _lib, ops   # absolute: this package is also importable as top-level `diffusion` through a symlink (INTEGRATION.md)

DDPM, DDIM = 0, 1


def _space_timesteps(num_timesteps: int, section_counts) -> set:
    """respace.py:12-62 ("ddimN" integer stride, or per-section fractional strides with python `round`)."""
    if isinstance(section_counts, str):
        if section_counts.startswith("ddim"):
            want = int(section_counts[len("ddim"):])
            for stride in range(1, num_timesteps):
                if len(range(0, num_timesteps, stride)) == want:
                    return set(range(0, num_timesteps, stride))
            raise ValueError(f"cannot create exactly {num_timesteps} steps with an integer stride")
        section_counts = [int(v) for v in section_counts.split(",")]
    size_per, extra = divmod(num_timesteps, len(section_counts))
    start, steps = 0, []
    for i, count in enumerate(section_counts):
        size = size_per + (1 if i < extra else 0)
        if size < count:
            raise ValueError(f"cannot divide section of {size} steps into {count}")
        frac = 1 if count <= 1 else (size - 1) / (count - 1)
        cur = 0.0
        for _ in range(count):
            steps.append(start + round(cur))
            cur += frac
        start += size
    return set(steps)


class SpacedDiffusion:
    """The sampling half of respace.SpacedDiffusion(GaussianDiffusion): eps-prediction, learned-range variance."""

    def __init__(self, use_timesteps, betas):
        base = np.array(betas, dtype=np.float64)
        self.original_num_steps = len(base)
        self.use_timesteps = set(use_timesteps)
        base_ac = np.cumprod(1.0 - base, axis=0)
        last, new_betas, self.timestep_map = 1.0, [], []
        for i, ac in enumerate(base_ac):                       # respace.py:77-86
            if i in self.use_timesteps:
                new_betas.append(1 - ac / last)
                last = ac
                self.timestep_map.append(i)
        b = self.betas = np.array(new_betas, dtype=np.float64)  # gaussian_diffusion.py:171-208
        assert b.ndim == 1 and (b > 0).all() and (b <= 1).all()
        self.num_timesteps = int(b.shape[0])
        alphas = 1.0 - b
        self.alphas_cumprod = np.cumprod(alphas, axis=0)
        self.alphas_cumprod_prev = np.append(1.0, self.alphas_cumprod[:-1])
        self.alphas_cumprod_next = np.append(self.alphas_cumprod[1:], 0.0)
        self.sqrt_alphas_cumprod = np.sqrt(self.alphas_cumprod)
        self.sqrt_one_minus_alphas_cumprod = np.sqrt(1.0 - self.alphas_cumprod)
        self.sqrt_recip_alphas_cumprod = np.sqrt(1.0 / self.alphas_cumprod)
        self.sqrt_recipm1_alphas_cumprod = np.sqrt(1.0 / self.alphas_cumprod - 1)
        self.posterior_variance = b * (1.0 - self.alphas_cumprod_prev) / (1.0 - self.alphas_cumprod)
        self.posterior_log_variance_clipped = (np.log(np.append(self.posterior_variance[1], self.posterior_variance[1:]))
                                               if len(b) > 1 else np.array([]))
        self.posterior_mean_coef1 = b * np.sqrt(self.alphas_cumprod_prev) / (1.0 - self.alphas_cumprod)
        self.posterior_mean_coef2 = (1.0 - self.alphas_cumprod_prev) * np.sqrt(alphas) / (1.0 - self.alphas_cumprod)
        self._dev = {}   # (device, batch, eta) -> (SamplerTables, keep-alive tensor, t table, mapped-t table)

    def __getstate__(self):
        """The device tables (ctypes structs with raw pointers) are a cache, not state: copies / pickles start empty."""
        state = dict(self.__dict__)
        state["_dev"] = {}
        return state

    # ------------------------------------------------------------------ device-resident state
    _BASE = ["sqrt_recip_alphas_cumprod", "sqrt_recipm1_alphas_cumprod", "posterior_mean_coef1", "posterior_mean_coef2",
             "posterior_log_variance_clipped"]

    def _state(self, device: torch.device, batch: int, eta: float = 0.0):
        """(tables, keep-alive tensor, t table, mapped-t table) for this device / batch size / DDIM eta, built once."""
        key = (device, batch, float(eta))
        st = self._dev.get(key)
        if st is None:
            f32 = lambda a: torch.from_numpy(np.asarray(a, dtype=np.float64)).float()   # noqa: E731  float64 table -> .float()
            base = [f32(getattr(self, n)) for n in self._BASE] + [f32(np.log(self.betas))]
            # DDIM scalars in fp32 with the reference's expressions (gaussian_diffusion.py:544-556), evaluated on the host
            ab, abp = f32(self.alphas_cumprod), f32(self.alphas_cumprod_prev)
            sigma = float(eta) * torch.sqrt((1 - abp) / (1 - ab)) * torch.sqrt(1 - ab / abp)
            ddim = [torch.sqrt(abp), sigma, torch.sqrt(1 - abp - sigma ** 2)]
            flat = torch.stack(base + ddim).to(device)
            tab = _lib.SamplerTables()
            tab.num_timesteps = self.num_timesteps
            for i, n in enumerate(self._BASE + ["log_betas", "ddim_sqrt_alpha_prev", "ddim_sigma", "ddim_dir"]):
                setattr(tab, n, flat[i].data_ptr())
            t_table = torch.arange(self.num_timesteps, device=device, dtype=torch.int64).unsqueeze(1).repeat(1, batch).contiguous()
            mapped = torch.tensor(self.timestep_map, device=device, dtype=torch.int64)[t_table].contiguous()
            st = self._dev[key] = (tab, flat, t_table, mapped)
        return st

    # ------------------------------------------------------------------ one step
    def _step(self, method, model_output, x, t, noise, clip_denoised, eta, want):
        if not x.is_cuda:
            raise RuntimeError("latte_b200.diffusion runs on CUDA tensors only (no CPU path)")
        if isinstance(model_output, tuple):
            model_output = model_output[0]
        B, F, C_ = x.shape[:3]
        hw = int(np.prod(x.shape[3:]))
        if tuple(model_output.shape) != (B, F, 2 * C_, *x.shape[3:]):
            raise ValueError(f"model output {tuple(model_output.shape)} != {(B, F, 2 * C_, *x.shape[3:])} (learn_sigma layout)")
        x = x.float().contiguous()
        model_output = model_output.contiguous()
        t = t.to(device=x.device, dtype=torch.int64).contiguous()
        if noise is not None:
            noise = noise.float().contiguous()
        tab = self._state(x.device, B, eta)[0]
        outs = {k: torch.empty_like(x) for k in want}
        ptr = lambda k: outs[k].data_ptr() if k in outs else None   # noqa: E731
        ops.call("b200_sampler_step", x.device, C.byref(tab), method, int(bool(clip_denoised)), t.data_ptr(), x.data_ptr(),
                 model_output.data_ptr(), ops._kind(model_output), noise.data_ptr() if noise is not None else None,
                 B, F, C_, hw, ptr("sample"), ptr("pred_xstart"), ptr("mean"), ptr("log_variance"))
        return outs

    def _call_model(self, model, x, t, model_kwargs, mapped=None, traj=None):
        """_WrappedModel.__call__ (respace.py:125-130): the model sees ORIGINAL timesteps.  The loops pass `mapped`, a row of
        the device-resident table; a free-standing call gathers from the cached device copy of timestep_map."""
        if mapped is None:
            key = ("map", x.device)
            mt = self._dev.get(key)
            if mt is None:
                mt = self._dev[key] = torch.tensor(self.timestep_map, device=x.device, dtype=torch.int64)
            mapped = mt[t.to(device=x.device, dtype=torch.int64)]
        kw = dict(model_kwargs or {})
        if traj is not None:
            kw["trajectory_step"] = traj      # latte_b200.Latte: conditioning rows precomputed for the whole loop
        return model(x, mapped, **kw)

    @staticmethod
    def _no_hooks(denoised_fn, cond_fn):
        if denoised_fn is not None or cond_fn is not None:
            raise NotImplementedError("denoised_fn / cond_fn hooks are not built in latte_b200.diffusion")

    def p_mean_variance(self, model, x, t, clip_denoised=True, denoised_fn=None, model_kwargs=None):
        self._no_hooks(denoised_fn, None)
        mo = self._call_model(model, x, t, model_kwargs)
        o = self._step(DDPM, mo, x, t, None, clip_denoised, 0.0, ("mean", "log_variance", "pred_xstart"))
        return {"mean": o["mean"], "variance": torch.exp(o["log_variance"]), "log_variance": o["log_variance"],
                "pred_xstart": o["pred_xstart"], "extra": None}

    def p_sample(self, model, x, t, clip_denoised=True, denoised_fn=None, cond_fn=None, model_kwargs=None, noise=None, _mapped=None,
                 _traj=None):
        self._no_hooks(denoised_fn, cond_fn)
        mo = self._call_model(model, x, t, model_kwargs, _mapped, _traj)
        if noise is None:
            noise = torch.randn_like(x, dtype=torch.float32)
        return self._step(DDPM, mo, x, t, noise, clip_denoised, 0.0, ("sample", "pred_xstart"))

    def ddim_sample(self, model, x, t, clip_denoised=True, denoised_fn=None, cond_fn=None, model_kwargs=None, eta=0.0, noise=None,
                    _mapped=None, _traj=None):
        self._no_hooks(denoised_fn, cond_fn)
        mo = self._call_model(model, x, t, model_kwargs, _mapped, _traj)
        if noise is None:
            noise = torch.randn_like(x, dtype=torch.float32)   # drawn even at eta = 0, as the reference does
        return self._step(DDIM, mo, x, t, noise, clip_denoised, eta, ("sample", "pred_xstart"))

    # ------------------------------------------------------------------ loops
    def _loop(self, step_fn, model, shape, noise, device, progress, **kw):
        if device is None:   # the reference needs `device=` when handed a bound method (sample.py:102); accept both here
            device = next(getattr(model, "__self__", model).parameters()).device
        device = torch.device(device)
        assert isinstance(shape, (tuple, list))
        img = noise if noise is not None else torch.randn(*shape, device=device)
        _, _, t_table, mapped_table = self._state(device, shape[0])
        indices = list(range(self.num_timesteps))[::-1]
        if progress:
            from tqdm.auto import tqdm
            indices = tqdm(indices)
        # SURVEY.md 8f rank 2: this repo's module can evaluate the (t, y)-only conditioning of ALL steps before the loop
        owner = getattr(model, "__self__", None)
        armed = False
        if (owner is not None and hasattr(owner, "precompute_conditioning") and not getattr(owner, "training", False)
                and not os.environ.get("B200_NO_TRAJECTORY_CONDITIONING")):
            # steps x B rows of (depth*6D + 2D) fp32: 0.8 MB per row for XL/2.  Bounded: past the budget (long chains at a
            # large batch) the loop falls back to the per-step conditioning path instead of risking an OOM the reference
            # would not have hit.
            row_bytes = getattr(owner, "conditioning_row_bytes", lambda: 0)()
            need = row_bytes * self.num_timesteps * shape[0]
            free = torch.cuda.mem_get_info(device)[0] if device.type == "cuda" else 0
            if 0 < need <= min(int(os.environ.get("B200_TRAJECTORY_BUDGET_MB", "4096")) << 20, free // 4):
                owner.precompute_conditioning(mapped_table, (kw.get("model_kwargs") or {}).get("y"))
                armed = True
        try:
            for i in indices:
                with torch.no_grad():
                    out = step_fn(model, img, t_table[i], _mapped=mapped_table[i], _traj=i if armed else None, **kw)
                yield out
                img = out["sample"]
        finally:
            if armed:
                owner.clear_conditioning()

    def p_sample_loop_progressive(self, model, shape, noise=None, clip_denoised=True, denoised_fn=None, cond_fn=None,
                                  model_kwargs=None, device=None, progress=False):
        yield from self._loop(self.p_sample, model, shape, noise, device, progress, clip_denoised=clip_denoised,
                              denoised_fn=denoised_fn, cond_fn=cond_fn, model_kwargs=model_kwargs)

    def p_sample_loop(self, model, shape, noise=None, clip_denoised=True, denoised_fn=None, cond_fn=None, model_kwargs=None,
                      device=None, progress=False):
        final = None
        for final in self.p_sample_loop_progressive(model, shape, noise, clip_denoised, denoised_fn, cond_fn, model_kwargs, device, progress):
            pass
        return final["sample"]

    def ddim_sample_loop_progressive(self, model, shape, noise=None, clip_denoised=True, denoised_fn=None, cond_fn=None,
                                     model_kwargs=None, device=None, progress=False, eta=0.0):
        yield from self._loop(self.ddim_sample, model, shape, noise, device, progress, clip_denoised=clip_denoised,
                              denoised_fn=denoised_fn, cond_fn=cond_fn, model_kwargs=model_kwargs, eta=eta)

    def ddim_sample_loop(self, model, shape, noise=None, clip_denoised=True, denoised_fn=None, cond_fn=None, model_kwargs=None,
                         device=None, progress=False, eta=0.0):
        final = None
        for final in self.ddim_sample_loop_progressive(model, shape, noise, clip_denoised, denoised_fn, cond_fn, model_kwargs,
                                                       device, progress, eta):
            pass
        return final["sample"]

    # ------------------------------------------------------------------ training objective (train.py:131,221)
    def _gather(self, name, t, ndim):
        """_extract_into_tensor (gaussian_diffusion.py:869-881): float64 table -> device gather -> .float(), broadcastable."""
        key = ("tab", name, t.device)
        tab = self._dev.get(key)
        if tab is None:
            arr = np.log(self.betas) if name == "log_betas" else getattr(self, name)
            tab = self._dev[key] = torch.from_numpy(np.asarray(arr, dtype=np.float64)).to(t.device)
        return tab[t].float().view(-1, *([1] * (ndim - 1)))

    def q_sample(self, x_start, t, noise=None):
        """x_t = sqrt(abar_t) x_0 + sqrt(1 - abar_t) noise (gaussian_diffusion.py:223-236)."""
        if noise is None:
            noise = torch.randn_like(x_start)
        return (self._gather("sqrt_alphas_cumprod", t, x_start.dim()) * x_start
                + self._gather("sqrt_one_minus_alphas_cumprod", t, x_start.dim()) * noise)

    def training_losses(self, model, x_start, t, model_kwargs=None, noise=None):
        """LossType.MSE with LEARNED_RANGE variance (gaussian_diffusion.py:719-795, the only objective create_diffusion builds):
        loss = mean((noise - eps)^2) + L_vb(eps.detach(), var_values), with L_vb = KL(q(x_{t-1}|x_t,x_0) || p) in bits and the
        discretised decoder NLL at t == 0 (:686-716; diffusion_utils.py:10-88).  The model is called with the ORIGINAL timestep
        (respace.py:125-130).  On CUDA the terms and their gradient with respect to the model output come from ONE kernel
        (`b200_training_loss`, csrc/sampler.cu) behind an autograd node -- the reference spends ~80 elementwise launches here;
        on CPU tensors (tests, toy models) the same expressions run as torch ops with autograd."""
        if noise is None:
            noise = torch.randn_like(x_start)
        if x_start.is_cuda and x_start.dim() == 5:
            x_t = self.q_sample(x_start.float(), t, noise.float())
            mo = self._call_model(model, x_t, t, model_kwargs)
            if isinstance(mo, tuple):
                mo = mo[0]
            Cc = x_t.shape[2]
            if tuple(mo.shape) != (x_t.shape[0], x_t.shape[1], 2 * Cc, *x_t.shape[3:]):
                raise ValueError(f"model output {tuple(mo.shape)} is not the learn_sigma layout of x {tuple(x_t.shape)}")
            mse, vb = _FusedLoss.apply(self, mo.float(), x_start.float(), x_t, noise.float(), t)
            return {"loss": mse + vb, "mse": mse, "vb": vb}
        return self._training_losses_torch(model, x_start, t, model_kwargs, noise)

    def _training_losses_torch(self, model, x_start, t, model_kwargs, noise):
        """The same objective as elementwise torch ops (CPU tensors / non-video shapes); the fused kernel is tested against it."""
        nd = x_start.dim()
        x_t = self.q_sample(x_start, t, noise)
        mo = self._call_model(model, x_t, t, model_kwargs)
        if isinstance(mo, tuple):
            mo = mo[0]
        Cc = x_t.shape[2]
        if tuple(mo.shape) != (x_t.shape[0], x_t.shape[1], 2 * Cc, *x_t.shape[3:]):
            raise ValueError(f"model output {tuple(mo.shape)} is not the learn_sigma layout of x {tuple(x_t.shape)}")
        mo = mo.float()
        eps, var_values = torch.split(mo, Cc, dim=2)
        flat = lambda v: v.mean(dim=list(range(1, v.dim())))   # noqa: E731  mean_flat
        # --- variational bound term on a frozen mean (:757-765)
        eps_f = eps.detach()
        min_log = self._gather("posterior_log_variance_clipped", t, nd)
        max_log = self._gather("log_betas", t, nd)
        frac = (var_values + 1) / 2
        log_var = frac * max_log + (1 - frac) * min_log
        pred_x0 = self._gather("sqrt_recip_alphas_cumprod", t, nd) * x_t - self._gather("sqrt_recipm1_alphas_cumprod", t, nd) * eps_f
        c1, c2 = self._gather("posterior_mean_coef1", t, nd), self._gather("posterior_mean_coef2", t, nd)
        mean = c1 * pred_x0 + c2 * x_t
        true_mean = c1 * x_start + c2 * x_t
        kl = 0.5 * (-1.0 + log_var - min_log + torch.exp(min_log - log_var) + (true_mean - mean) ** 2 * torch.exp(-log_var))
        kl = flat(kl) / np.log(2.0)
        centered = x_start - mean
        inv_std = torch.exp(-0.5 * log_var)
        cdf = lambda v: 0.5 * (1.0 + torch.tanh(np.sqrt(2.0 / np.pi) * (v + 0.044715 * torch.pow(v, 3))))   # noqa: E731
        cdf_plus, cdf_min = cdf(inv_std * (centered + 1.0 / 255.0)), cdf(inv_std * (centered - 1.0 / 255.0))
        log_probs = torch.where(x_start < -0.999, torch.log(cdf_plus.clamp(min=1e-12)),
                                torch.where(x_start > 0.999, torch.log((1.0 - cdf_min).clamp(min=1e-12)),
                                            torch.log((cdf_plus - cdf_min).clamp(min=1e-12))))
        nll = flat(-log_probs) / np.log(2.0)
        vb = torch.where(t.to(kl.device) == 0, nll, kl)
        mse = flat((noise - eps) ** 2)
        return {"loss": mse + vb, "mse": mse, "vb": vb}


class _FusedLoss(torch.autograd.Function):
    """(mse, vb) per sample from `b200_training_loss`, with d mse / d eps and d vb / d var_values kept for the backward."""

    @staticmethod
    def forward(ctx, diff, mo, x0, x_t, noise, t):
        B, F, C2 = mo.shape[:3]
        Cc = C2 // 2
        hw = int(np.prod(mo.shape[3:]))
        dev = mo.device
        mo, x0, x_t, noise = mo.contiguous(), x0.contiguous(), x_t.contiguous(), noise.contiguous()
        tt = t.to(device=dev, dtype=torch.int64).contiguous()
        tab = diff._state(dev, B)[0]
        sums = torch.empty(2, B, dtype=torch.float32, device=dev)
        need_grad = ctx.needs_input_grad[1]
        dmo = torch.empty_like(mo) if need_grad else None
        ops.call("b200_training_loss", dev, C.byref(tab), tt.data_ptr(), x0.data_ptr(), x_t.data_ptr(), noise.data_ptr(),
                 mo.data_ptr(), B, F, Cc, hw, sums.data_ptr(), dmo.data_ptr() if need_grad else None)
        n = float(F * Cc * hw)
        # saved, not kept on ctx: autograd frees it after the first backward, so a second backward through a freed graph
        # raises autograd's own error, and one through a retained graph adds the gradient again, as torch's loss would
        if need_grad:
            ctx.save_for_backward(dmo)
        return sums[0] / n, sums[1] / (n * float(np.log(2.0)))

    @staticmethod
    def backward(ctx, g_mse, g_vb):
        (dmo,) = ctx.saved_tensors
        B, F = dmo.shape[:2]
        scale = torch.stack((g_mse, g_vb), dim=1).reshape(B, 1, 2, 1, 1)
        return None, (dmo.reshape(B, F, 2, -1, dmo.shape[-1]) * scale).reshape(dmo.shape), None, None, None, None


def create_diffusion(timestep_respacing, noise_schedule="linear", use_kl=False, sigma_small=False, predict_xstart=False,
                     learn_sigma=True, rescale_learned_sigmas=False, diffusion_steps=1000):
    """diffusion/__init__.py:10-47 for the configuration every Latte script uses."""
    if noise_schedule != "linear" or predict_xstart or not learn_sigma:
        raise NotImplementedError("only the linear schedule with eps-prediction and learned-range variance is built")
    scale = 1000 / diffusion_steps
    betas = np.linspace(scale * 0.0001, scale * 0.02, diffusion_steps, dtype=np.float64)   # gaussian_diffusion.py:110-118
    if timestep_respacing is None or timestep_respacing == "":
        timestep_respacing = [diffusion_steps]
    return SpacedDiffusion(_space_timesteps(diffusion_steps, timestep_respacing), betas)
