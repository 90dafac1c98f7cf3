"""H100-native DiffusionDDIM: the reference's DDIM sampler interface
(tools/modules/diffusions/diffusion_ddim.py:27-254) with the per-step tensor arithmetic fused into one
kernel (vgen_ddim_step: CFG mix + v->x0 + eps + x_{t-1}).

Host side (kept in fp64 torch / Python exactly like the reference, so it is bit-exact):
  * beta schedules `cosine`, `linear_sd` (+ zero-terminal-SNR rescale)     schedules.py:5-21,62-63,72-79,143-165
  * cumulative-product tables                                             diffusion_ddim.py:46-78
  * the timestep list  (1 + arange(0, T, T // S)).clamp(0, T-1).flip(0)   diffusion_ddim.py:250
Only the sampling entry points used by the inference engines are provided: ddim_sample_loop and ddim_sample, and the
DDIM inversion ddim_reverse_sample_loop / ddim_reverse_sample (DreamVideo), for var_type fixed_small / mean_type v|eps.  The arithmetic of the reference's p_mean_variance (:147-206: two model calls,
CFG mix, v -> x0) has no method of its own here -- it lives inside the fused step kernel; the training losses and PLMS are
out of scope and absent (calling them raises AttributeError, not a fallback).  DiffusionDDIMReward (InstructVideo) samples
like DiffusionDDIM; its reward fine-tuning methods raise NotImplementedError.
"""
from __future__ import annotations

import math
import os

import torch

from . import ops


def _cosine_betas(num_timesteps, cosine_s=0.008, **kw):
    def abar(u):
        return math.cos((u + cosine_s) / (1 + cosine_s) * math.pi / 2) ** 2
    out = []
    for step in range(num_timesteps):
        out.append(min(1.0 - abar((step + 1) / num_timesteps) / abar(step / num_timesteps), 0.999))
    return torch.tensor(out, dtype=torch.float64)


def _linear_sd_betas(num_timesteps, init_beta, last_beta, **kw):
    return torch.linspace(init_beta ** 0.5, last_beta ** 0.5, num_timesteps, dtype=torch.float64) ** 2


def _rescale_zero_terminal_snr(betas):
    abs_ = (1 - betas).cumprod(0).sqrt()
    a0, aT = abs_[0].clone(), abs_[-1].clone()
    abs_ = abs_ - aT
    abs_ = abs_ * (a0 / (a0 - aT))
    ab = abs_ ** 2
    alphas = torch.cat([ab[0:1], ab[1:] / ab[:-1]])
    return 1 - alphas


def beta_schedule(schedule="cosine", num_timesteps=1000, zero_terminal_snr=False, **kwargs):
    fn = {"cosine": _cosine_betas, "linear_sd": _linear_sd_betas}.get(schedule)
    if fn is None:
        raise NotImplementedError(f"vgen_b200: beta schedule '{schedule}' is not used by the supported configs")
    betas = fn(num_timesteps, **kwargs)
    if zero_terminal_snr and abs(betas.max() - 1.0) > 0.0001:
        betas = _rescale_zero_terminal_snr(betas)
    return betas


def _unwrap(model):
    return getattr(model, "module", model)


def cfg_forward(model, xt, ts, model_kwargs, by_keyword=False):
    """The two classifier-free-guidance evaluations of one step (diffusion_ddim.py:157-158, diffusion_gauss.py:204-208).

    A vgen_b200 UNet (`cfg_batch = True`) evaluates both branches as ONE forward of batch 2b -- the same arithmetic
    per sample (batch entries never interact), half the launches, and two tiles per CTA pair on the low-resolution
    layers so their epilogue overlaps a main loop.  Any other callable (e.g. a reference model) gets the reference's
    two separate calls.  VGEN_CFG_BATCH=0 disables the batching.

    Keys a model names in `cfg_per_sample` are per-sample values (a number or a [b] tensor per branch, e.g. DreamVideo's
    ag_strength, or a [b, n] tensor, e.g. UNetSD_LoRA's lora_strength over n LoRA sets): the two branches become one fp32
    [2b] (or [2b, n]) tensor, so branches with different values still run as one forward, and one CUDA graph serves any
    value.  A number or [b] branch next to a [b, n] one is repeated over the n columns."""
    kc, ku = model_kwargs
    m = _unwrap(model)
    call = (lambda x, t, kw: model(x, t=t, **kw)) if by_keyword else (lambda x, t, kw: model(x, t, **kw))
    if getattr(m, "cfg_batch", False) and os.environ.get("VGEN_CFG_BATCH", "1") != "0" and kc.keys() == ku.keys():
        merged = {}
        per_sample = getattr(m, "cfg_per_sample", ())
        for k in kc:
            a, b = kc[k], ku[k]
            if k in per_sample and a is not None and b is not None:
                pa, pb = _per_sample(a, xt), _per_sample(b, xt)
                if pa.dim() != pb.dim():
                    n = (pa if pa.dim() == 2 else pb).size(1)
                    pa, pb = (p if p.dim() == 2 else p[:, None].expand(-1, n) for p in (pa, pb))
                merged[k] = torch.cat([pa, pb])
            elif torch.is_tensor(a) and torch.is_tensor(b) and a.shape == b.shape and a.dtype == b.dtype and a.dim() >= 1 \
                    and a.size(0) == xt.size(0):
                merged[k] = torch.cat([a, b], dim=0)
            elif a is None and b is None:
                merged[k] = None
            else:
                merged = None
                break
        if merged is not None:
            out = call(torch.cat([xt, xt], dim=0), torch.cat([ts, ts], dim=0), merged)
            n = xt.size(0)
            return out[:n], out[n:]
    return call(xt, ts, kc), call(xt, ts, ku)


def _per_sample(v, xt):
    """A number or a 1- / b-entry tensor -> fp32 [b] on xt's device (b = xt.size(0)); a 2-D [1 | b, n] tensor -> fp32
    [b, n]."""
    t = torch.as_tensor(v, dtype=torch.float32).to(xt.device)
    if t.dim() == 2:
        if t.size(0) not in (1, xt.size(0)):
            raise ValueError(f"a per-sample [rows, n] argument must have 1 or {xt.size(0)} rows, got {t.size(0)}")
        return t.expand(xt.size(0), t.size(1))
    t = t.reshape(-1)
    if t.numel() not in (1, xt.size(0)):
        raise ValueError(f"a per-sample argument must be a number or have {xt.size(0)} entries, got {t.numel()}")
    return t.expand(xt.size(0))


class DiffusionDDIM(object):
    def __init__(self, schedule="linear_sd", schedule_param={}, mean_type="eps", var_type="learned_range", loss_type="mse",
                 epsilon=1e-12, rescale_timesteps=False, noise_strength=0.0, **kwargs):
        assert mean_type in ["x0", "x_{t-1}", "eps", "v"]
        assert var_type in ["learned", "learned_range", "fixed_large", "fixed_small"]
        betas = beta_schedule(schedule, **schedule_param)
        assert min(betas) > 0 and max(betas) <= 1
        self.betas = betas
        self.num_timesteps = len(betas)
        self.mean_type, self.var_type, self.loss_type = mean_type, var_type, loss_type
        self.epsilon, self.rescale_timesteps, self.noise_strength = epsilon, rescale_timesteps, noise_strength
        alphas = 1 - self.betas
        self.alphas_cumprod = torch.cumprod(alphas, dim=0)
        self.alphas_cumprod_prev = torch.cat([alphas.new_ones([1]), self.alphas_cumprod[:-1]])
        self.alphas_cumprod_next = torch.cat([self.alphas_cumprod[1:], alphas.new_zeros([1])])
        self.sqrt_alphas_cumprod = torch.sqrt(self.alphas_cumprod)
        self.sqrt_one_minus_alphas_cumprod = torch.sqrt(1.0 - self.alphas_cumprod)
        self.log_one_minus_alphas_cumprod = torch.log(1.0 - self.alphas_cumprod)
        self.sqrt_recip_alphas_cumprod = torch.sqrt(1.0 / self.alphas_cumprod)
        self.sqrt_recipm1_alphas_cumprod = torch.sqrt(1.0 / self.alphas_cumprod - 1)
        self.posterior_variance = betas * (1.0 - self.alphas_cumprod_prev) / (1.0 - self.alphas_cumprod)
        self.posterior_log_variance_clipped = torch.log(self.posterior_variance.clamp(1e-20))
        self.posterior_mean_coef1 = betas * torch.sqrt(self.alphas_cumprod_prev) / (1.0 - self.alphas_cumprod)
        self.posterior_mean_coef2 = (1.0 - self.alphas_cumprod_prev) * torch.sqrt(alphas) / (1.0 - self.alphas_cumprod)

    # ---- timestep / index math (host, integer-exact) --------------------------------------------
    def ddim_steps(self, ddim_timesteps):
        T = self.num_timesteps
        return (1 + torch.arange(0, T, T // ddim_timesteps)).clamp(0, T - 1).flip(0)

    def _scale_timesteps(self, t):
        if self.rescale_timesteps:
            return t.float() * 1000.0 / self.num_timesteps
        return t

    def step_coefficients(self, step, ddim_timesteps, eta=0.0):
        """The seven fp32 scalars of one DDIM update, computed like the reference does: fp64 table
        entries cast to fp32 by _i() (:10-16), then fp32 arithmetic (:230-240)."""
        T = self.num_timesteps
        stride = T // ddim_timesteps
        t = int(step)
        tp = max(t - stride, 0)
        f32 = torch.float32
        a_t = self.alphas_cumprod[t].to(f32)
        a_prev = self.alphas_cumprod[tp].to(f32)
        sigma = eta * torch.sqrt((1 - a_prev) / (1 - a_t) * (1 - a_t / a_prev))
        coef = [self.sqrt_alphas_cumprod[t].to(f32), self.sqrt_one_minus_alphas_cumprod[t].to(f32),
                self.sqrt_recip_alphas_cumprod[t].to(f32), self.sqrt_recipm1_alphas_cumprod[t].to(f32),
                torch.sqrt(a_prev), torch.sqrt(1 - a_prev - sigma ** 2), sigma * (1.0 if t != 0 else 0.0)]
        return [float(c) for c in coef]

    # ---- sampling ----------------------------------------------------------------------------------
    @torch.no_grad()
    def ddim_sample(self, xt, t, model, model_kwargs={}, clamp=None, percentile=None, condition_fn=None, guide_scale=None,
                    ddim_timesteps=20, eta=0.0):
        """One DDIM step (diffusion_ddim.py:209-241); returns (x_{t-1}, x0) like the reference.  All batch entries
        share the timestep (true for every caller on the sampling path)."""
        if clamp is not None or percentile is not None or condition_fn is not None:
            raise NotImplementedError("vgen_b200 DiffusionDDIM: clamp / percentile / condition_fn are not used by the "
                                      "supported inference configs")
        if self.var_type != "fixed_small" or self.mean_type not in ("v", "eps"):
            raise NotImplementedError("vgen_b200 DiffusionDDIM: only var_type fixed_small with mean_type v|eps")
        return self._ddim_step(xt, int(t.flatten()[0]), t, model, model_kwargs, guide_scale, ddim_timesteps, eta, want_x0=True)

    def _ddim_step(self, xt, step, t, model, model_kwargs, guide_scale, ddim_timesteps, eta, want_x0=False):
        if self.var_type != "fixed_small" or self.mean_type not in ("v", "eps"):
            raise NotImplementedError("vgen_b200 DiffusionDDIM: only var_type fixed_small with mean_type v|eps")
        ts = self._scale_timesteps(t)
        if guide_scale is None:
            y_out = model(xt, ts, **model_kwargs)
            u_out = None
        else:
            assert isinstance(model_kwargs, list) and len(model_kwargs) == 2
            y_out, u_out = cfg_forward(model, xt, ts, model_kwargs)
        coef = self.step_coefficients(step, ddim_timesteps, eta)
        # the reference draws the noise in xt's dtype even when eta == 0 (:237) -- keeps the device RNG stream aligned;
        # the kernel reads fp32, so a non-fp32 draw is converted (never reinterpreted)
        noise = torch.randn_like(xt)
        y16 = y_out if y_out.dtype == torch.float16 else y_out.to(torch.float16)
        u16 = None if u_out is None else (u_out if u_out.dtype == torch.float16 else u_out.to(torch.float16))
        xt = xt if (xt.dtype == torch.float32 and xt.is_contiguous()) else xt.float().contiguous()
        xt = xt.clone()
        x0 = torch.empty_like(xt) if want_x0 else None
        ops.ddim_step_(xt, y16.contiguous(), None if u16 is None else u16.contiguous(), coef, guide_scale,
                       mean_type_v=(self.mean_type == "v"),
                       noise=noise.float().contiguous() if coef[6] != 0.0 else None, x0_out=x0)
        return xt, x0

    @torch.no_grad()
    def ddim_sample_loop(self, noise, model, model_kwargs={}, clamp=None, percentile=None, condition_fn=None,
                         guide_scale=None, ddim_timesteps=20, eta=0.0):
        """diffusion_ddim.py:244-254."""
        b = noise.size(0)
        xt = noise
        for step in self.ddim_steps(ddim_timesteps):
            t = torch.full((b,), int(step), dtype=torch.long, device=xt.device)
            if clamp is not None or percentile is not None or condition_fn is not None:
                raise NotImplementedError("vgen_b200 DiffusionDDIM: clamp / percentile / condition_fn are not supported")
            # the step index is known on the host: no device->host read of t inside the loop
            xt, _ = self._ddim_step(xt, int(step), t, model, model_kwargs, guide_scale, ddim_timesteps, eta)
        return xt


    # ---- DDIM inversion (diffusion_ddim.py:256-287) -------------------------------------------------------------
    def ddim_reverse_steps(self, ddim_timesteps):
        """The inversion's timestep list, arange(0, T, T // S) (:282): ascending, no +1 shift."""
        T = self.num_timesteps
        return torch.arange(0, T, T // ddim_timesteps)

    def reverse_step_coefficients(self, step, ddim_timesteps):
        """The seven fp32 scalars of one inversion step x_t -> x_{t+stride}, in vgen_ddim_step's slots: the x0 / eps
        pair of the forward step and then sqrt(a_next), sqrt(1 - a_next) where a_next is the fp64 table
        cat([alphas_cumprod, 0]) at clamp(t + stride, 0, T) cast to fp32 (_i(), :10-16), the square roots in fp32 (:275-279);
        no noise term."""
        T = self.num_timesteps
        t = int(step)
        f32 = torch.float32
        a_next = torch.cat([self.alphas_cumprod, self.alphas_cumprod.new_zeros([1])])[min(max(t + T // ddim_timesteps, 0), T)]
        a_next = a_next.to(f32)
        coef = [self.sqrt_alphas_cumprod[t].to(f32), self.sqrt_one_minus_alphas_cumprod[t].to(f32),
                self.sqrt_recip_alphas_cumprod[t].to(f32), self.sqrt_recipm1_alphas_cumprod[t].to(f32),
                torch.sqrt(a_next), torch.sqrt(1 - a_next), 0.0]
        return [float(c) for c in coef]

    def _reverse_step(self, xt, step, t, model, model_kwargs, guide_scale, ddim_timesteps, want_x0=False):
        if self.var_type != "fixed_small" or self.mean_type not in ("v", "eps"):
            raise NotImplementedError("vgen_b200 DiffusionDDIM: only var_type fixed_small with mean_type v|eps")
        ts = self._scale_timesteps(t)
        if guide_scale is None:
            y_out, u_out = model(xt, ts, **model_kwargs), None
        else:
            assert isinstance(model_kwargs, list) and len(model_kwargs) == 2
            y_out, u_out = cfg_forward(model, xt, ts, model_kwargs)
        coef = self.reverse_step_coefficients(step, ddim_timesteps)
        y16 = y_out if y_out.dtype == torch.float16 else y_out.to(torch.float16)
        u16 = None if u_out is None else (u_out if u_out.dtype == torch.float16 else u_out.to(torch.float16))
        xt = xt if (xt.dtype == torch.float32 and xt.is_contiguous()) else xt.float().contiguous()
        xt = xt.clone()
        x0 = torch.empty_like(xt) if want_x0 else None
        ops.ddim_step_(xt, y16.contiguous(), None if u16 is None else u16.contiguous(), coef, guide_scale,
                       mean_type_v=(self.mean_type == "v"), noise=None, x0_out=x0)
        return xt, x0

    @torch.no_grad()
    def ddim_reverse_sample(self, xt, t, model, model_kwargs={}, clamp=None, percentile=None, guide_scale=None,
                            ddim_timesteps=20):
        """One deterministic inversion step x_t -> x_{t+stride} (diffusion_ddim.py:256-274): the forward step's x0 and
        eps, then mu = sqrt(a_next) x0 + sqrt(1 - a_next) eps in the fused step kernel.  Returns (mu, x0).  All batch
        entries share the timestep; no random numbers are drawn (nor does the reference draw any)."""
        if clamp is not None or percentile is not None:
            raise NotImplementedError("vgen_b200 DiffusionDDIM: clamp / percentile are not used by the supported "
                                      "inference configs")
        return self._reverse_step(xt, int(t.flatten()[0]), t, model, model_kwargs, guide_scale, ddim_timesteps,
                                  want_x0=True)

    @torch.no_grad()
    def ddim_reverse_sample_loop(self, x0, model, model_kwargs={}, clamp=None, percentile=None, guide_scale=None,
                                 ddim_timesteps=20):
        """diffusion_ddim.py:276-287: DDIM inversion of x0 over arange(0, T, T // S) (DreamVideo's inverse_noise_strength,
        inference_dreamvideo_entrance.py:199-209)."""
        if clamp is not None or percentile is not None:
            raise NotImplementedError("vgen_b200 DiffusionDDIM: clamp / percentile are not supported")
        b = x0.size(0)
        xt = x0
        for step in self.ddim_reverse_steps(ddim_timesteps).tolist():
            t = torch.full((b,), step, dtype=torch.long, device=xt.device)
            xt, _ = self._reverse_step(xt, step, t, model, model_kwargs, guide_scale, ddim_timesteps)
        return xt


class DiffusionDDIMReward(DiffusionDDIM):
    """Drop-in for diffusion_ddim.py:516 (DIFFUSION 'DiffusionDDIMReward', every configs/instructvideo Diffusion): the
    reference class inherits ddim_sample_loop unchanged and only adds gradient-carrying methods for InstructVideo's reward
    fine-tuning.  Sampling is DiffusionDDIM's; those methods raise NotImplementedError."""

    def _reward_training(self, name):
        raise NotImplementedError(f"vgen_b200 DiffusionDDIMReward.{name}: reward fine-tuning is not supported (the native "
                                  "path samples without gradients); use the reference class to train")

    def ddim_sample_loop_partial(self, *args, **kwargs):
        self._reward_training("ddim_sample_loop_partial")

    def ddim_sample_gradient(self, *args, **kwargs):
        self._reward_training("ddim_sample_gradient")

    def ddim_sample_with_logprob(self, *args, **kwargs):
        self._reward_training("ddim_sample_with_logprob")

    def ddim_sample_loop_with_logprob(self, *args, **kwargs):
        self._reward_training("ddim_sample_loop_with_logprob")

    def loss(self, *args, **kwargs):
        self._reward_training("loss")
