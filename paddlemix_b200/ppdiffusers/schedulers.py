"""Schedulers on the hot path, mirroring ppdiffusers' interface (set_timesteps / scale_model_input / step).

The index and scalar math runs on the host in numpy float32, operation by operation as the reference does on 0-d
fp32 tensors (ppdiffusers/schedulers/scheduling_ddim.py:205-238, 305-348, 410-457;
scheduling_flow_match_euler_discrete.py:64-83, 140-163, 244-275); the elementwise update of the latent runs in one
fused CUDA kernel (b200mix_ddim_step_ex / b200mix_euler_step) that also folds in the classifier-free-guidance combine.
tests/test_schedulers.py checks the host scalars bit-for-bit against the oracle.
"""
import math
from typing import Optional

import numpy as np

f32 = np.float32


def _betas_for_alpha_bar(n, max_beta=0.999):
    def alpha_bar(t):
        return math.cos((t + 0.008) / 1.008 * math.pi / 2) ** 2
    return np.array([min(1 - alpha_bar((i + 1) / n) / alpha_bar(i / n), max_beta) for i in range(n)], dtype=f32)


def _beta_tables(beta_schedule, beta_start, beta_end, n, owner):
    """betas, alphas = 1 - betas and alphas_cumprod of a training schedule in fp32, as the reference's schedulers build
    them in __init__ (scheduling_ddim.py:205-238); `owner` is the scheduler class named in the error."""
    if beta_schedule == "linear":
        betas = _linspace_f32(beta_start, beta_end, n)
    elif beta_schedule == "scaled_linear":
        betas = _linspace_f32(beta_start ** 0.5, beta_end ** 0.5, n) ** 2
    elif beta_schedule == "squaredcos_cap_v2":
        betas = _betas_for_alpha_bar(n)
    else:
        raise NotImplementedError(f"{beta_schedule} does is not implemented for {owner}")
    alphas = (f32(1.0) - betas).astype(f32)
    return betas, alphas, _cumprod_f32(alphas)


def _train_sigmas(alphas_cumprod):
    """((1 - alphas_cumprod) / alphas_cumprod) ** 0.5 in fp32: the sigmas of the training timesteps."""
    ac = alphas_cumprod
    return np.sqrt(((f32(1.0) - ac) / ac).astype(f32), dtype=f32)


def _karras_sigmas(sigma_min, sigma_max, num_inference_steps, rho=7.0):
    """Karras et al. (2022) noise levels from sigma_max down to sigma_min, in float64."""
    ramp = np.linspace(0, 1, num_inference_steps)
    return (sigma_max ** (1 / rho) + ramp * (sigma_min ** (1 / rho) - sigma_max ** (1 / rho))) ** rho


def _sigma_to_t(sigma, log_sigmas):
    """The (fractional) training timestep of `sigma`, interpolated in log sigma."""
    log_sigma = np.log(np.maximum(sigma, 1e-10))
    dists = log_sigma - log_sigmas[:, np.newaxis]
    low_idx = np.cumsum((dists >= 0), axis=0).argmax(axis=0).clip(max=log_sigmas.shape[0] - 2)
    high_idx = low_idx + 1
    low, high = log_sigmas[low_idx], log_sigmas[high_idx]
    w = np.clip((low - log_sigma) / (low - high), 0, 1)
    return ((1 - w) * low_idx + w * high_idx).reshape(np.shape(sigma))


def _multistep_schedule(ac, num_inference_steps, timestep_spacing, steps_offset, use_karras_sigmas, use_lu_lambdas=False,
                        last_timestep=None):
    """(int64 timesteps, fp32 sigmas with one trailing entry) of the multistep solvers' set_timesteps
    (scheduling_dpmsolver_multistep.py:226-296, scheduling_unipc_multistep.py:210-271) over the training
    alphas_cumprod `ac`; `last_timestep` (default: every training step) is DPM-Solver's lambda_min_clipped bound. The
    Karras / Lu schedules repeat their last sigma as the trailing entry, so their final step has h = 0."""
    N = len(ac)
    last_timestep = N if last_timestep is None else last_timestep
    if timestep_spacing == "linspace":
        timesteps = np.linspace(0, last_timestep - 1, num_inference_steps + 1).round()[::-1][:-1].copy().astype(np.int64)
    elif timestep_spacing == "leading":
        step_ratio = last_timestep // (num_inference_steps + 1)
        timesteps = (np.arange(0, num_inference_steps + 1) * step_ratio).round()[::-1][:-1].copy().astype(np.int64)
        timesteps += steps_offset
    elif timestep_spacing == "trailing":
        step_ratio = N / num_inference_steps
        timesteps = np.arange(last_timestep, 0, -step_ratio).round().copy().astype(np.int64)
        timesteps -= 1
    else:
        raise ValueError(f"{timestep_spacing} is not supported. Please make sure to choose one of 'linspace', "
                         "'leading' or 'trailing'.")
    sigmas = _train_sigmas(ac)
    log_sigmas = np.log(sigmas)
    if use_karras_sigmas:
        sigmas = _karras_sigmas(sigmas[0].item(), sigmas[-1].item(), num_inference_steps)  # training sigmas ascend
        timesteps = np.array([_sigma_to_t(s, log_sigmas) for s in sigmas]).round()
        sigmas = np.concatenate([sigmas, sigmas[-1:]]).astype(f32)
    elif use_lu_lambdas:
        lambdas = np.flip(log_sigmas.copy())
        lmin, lmax = lambdas[-1].item(), lambdas[0].item()
        ramp = np.linspace(0, 1, num_inference_steps)
        sigmas = np.exp(lmax + ramp * (lmin - lmax))
        timesteps = np.array([_sigma_to_t(s, log_sigmas) for s in sigmas]).round()
        sigmas = np.concatenate([sigmas, sigmas[-1:]]).astype(f32)
    else:
        sigmas = np.interp(timesteps, np.arange(0, len(sigmas)), sigmas)
        sigma_last = np.sqrt(f32((f32(1.0) - ac[0]) / ac[0]), dtype=f32)
        sigmas = np.concatenate([sigmas, [sigma_last]]).astype(f32)
    return np.asarray(timesteps).astype(np.int64), sigmas


class DDIMScheduler:
    """ppdiffusers.DDIMScheduler (scheduling_ddim.py:131) without dynamic thresholding. eta = 0 (the deterministic
    sampler) runs b200mix_ddim_step_ex; eta > 0 runs b200mix_ddim_eta_step, which adds std_dev_t * z to the same mean.

    The noise z of a stochastic step is a standard normal per element. `step(..., variance_noise=...)` uses the given
    fp32 tensor; otherwise the first such step after set_timesteps draws one 63-bit seed from `generator` (torch's
    default generator when None), and every step takes counter-based Philox normals keyed by (seed, index of the step
    call since set_timesteps), drawn inside the kernel, exactly as EulerAncestralDiscreteScheduler does. One generator
    state therefore gives one result, on any GPU and with or without CUDA graphs, but not Paddle's draws. In a
    data-parallel run every rank steps its own slice of the batch with its own scheduler: the noise is keyed by that
    rank's generator and by the element's index within the rank's latents, not by the image's global index, so ranks
    given equal generator states draw equal noise for their slices."""

    order = 1
    init_noise_sigma = 1.0
    takes_generator = True  # step(..., generator=) seeds the noise of eta > 0 (see the class docstring)

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.0001, beta_end: float = 0.02,
                 beta_schedule: str = "linear", clip_sample: bool = True, set_alpha_to_one: bool = True,
                 steps_offset: int = 0, prediction_type: str = "epsilon", timestep_spacing: str = "leading",
                 clip_sample_range: float = 1.0, thresholding: bool = False):
        if thresholding:
            raise NotImplementedError("dynamic thresholding (pixel-space models) is outside the latent-diffusion hot path")
        if prediction_type not in ("epsilon", "sample", "v_prediction"):
            raise ValueError(f"prediction_type given as {prediction_type} must be one of `epsilon`, `sample`, or"
                             " `v_prediction`")
        self.clip_sample_range = clip_sample_range
        self.betas, self.alphas, self.alphas_cumprod = _beta_tables(beta_schedule, beta_start, beta_end,
                                                                    num_train_timesteps, type(self))
        self.final_alpha_cumprod = f32(1.0) if set_alpha_to_one else self.alphas_cumprod[0]
        self.num_train_timesteps = num_train_timesteps
        self.clip_sample = clip_sample
        self.steps_offset = steps_offset
        self.prediction_type = prediction_type
        self.timestep_spacing = timestep_spacing
        self.num_inference_steps: Optional[int] = None
        self.timesteps = np.arange(0, num_train_timesteps)[::-1].copy().astype(np.int64)
        self._step, self._seed = 0, None  # the Philox key of the stochastic steps (eta > 0)

    def scale_model_input(self, sample, timestep=None):
        return sample

    def set_timesteps(self, num_inference_steps: int):
        self._step, self._seed = 0, None
        if num_inference_steps > self.num_train_timesteps:
            raise ValueError(
                f"`num_inference_steps`: {num_inference_steps} cannot be larger than `self.config.train_timesteps`:"
                f" {self.num_train_timesteps} as the unet model trained with this scheduler can only handle"
                f" maximal {self.num_train_timesteps} timesteps.")
        self.num_inference_steps = num_inference_steps
        if self.timestep_spacing == "linspace":
            t = np.linspace(0, self.num_train_timesteps - 1, num_inference_steps).round()[::-1].copy().astype(np.int64)
        elif self.timestep_spacing == "leading":
            step_ratio = self.num_train_timesteps // num_inference_steps
            t = (np.arange(0, num_inference_steps) * step_ratio).round()[::-1].copy().astype(np.int64)
            t += self.steps_offset
        elif self.timestep_spacing == "trailing":
            step_ratio = self.num_train_timesteps / num_inference_steps
            t = np.round(np.arange(self.num_train_timesteps, 0, -step_ratio)).astype(np.int64)
            t -= 1
        else:
            raise ValueError(f"{self.timestep_spacing} is not supported. Please make sure to choose one of 'leading' "
                             "or 'trailing'.")
        self.timesteps = t

    def _get_variance(self, timestep, prev_timestep):
        a_t = self.alphas_cumprod[timestep]
        a_p = self.alphas_cumprod[prev_timestep] if prev_timestep >= 0 else self.final_alpha_cumprod
        b_t, b_p = f32(1) - a_t, f32(1) - a_p
        return f32(f32(b_p / b_t) * f32(f32(1) - f32(a_t / a_p)))

    def step_scalars(self, timestep: int):
        """(sqrt(a_t), sqrt(1-a_t), sqrt(a_prev), sqrt(1-a_prev-std^2)) as fp32, eta = 0 (:410-457)."""
        return self.eta_step_scalars(timestep, 0.0)[:4]

    def eta_step_scalars(self, timestep: int, eta: float):
        """(sqrt(a_t), sqrt(1-a_t), sqrt(a_prev), sqrt(1-a_prev-std^2), std) as fp32 with std = eta * variance^0.5
        (:410-457), each computed as the reference computes its 0-d fp32 tensor."""
        if self.num_inference_steps is None:
            raise ValueError("Number of inference steps is 'None', you need to run 'set_timesteps' after creating the "
                             "scheduler")
        timestep = int(timestep)
        prev_timestep = timestep - self.num_train_timesteps // self.num_inference_steps
        a_t = self.alphas_cumprod[timestep]
        a_p = self.alphas_cumprod[prev_timestep] if prev_timestep >= 0 else self.final_alpha_cumprod
        b_t = f32(f32(1) - a_t)
        var = self._get_variance(timestep, prev_timestep)
        std = f32(f32(eta) * np.sqrt(var, dtype=f32))
        dir_coef = np.sqrt(f32(f32(f32(1) - a_p) - f32(std * std)), dtype=f32)
        return (float(np.sqrt(a_t, dtype=f32)), float(np.sqrt(b_t, dtype=f32)), float(np.sqrt(a_p, dtype=f32)),
                float(dir_coef), float(std))

    def step(self, model_output, timestep, sample, eta: float = 0.0, model_output_cond=None, guidance_scale=0.0,
             out=None, use_clipped_model_output: bool = False, generator=None, variance_noise=None):
        """sample, result: fp32 CUDA tensors (out may be sample); model_output: contiguous bf16/fp32 CUDA tensor with
        sample's element count, read in sample's element order. With model_output_cond (same dtype) the CFG combine is
        fused into the same kernel. eta > 0 adds std_dev_t * z (see the class docstring): variance_noise is z as an fp32
        tensor like sample, or None for the Philox stream seeded from `generator`."""
        from .. import ops
        if eta == 0.0 and not use_clipped_model_output:
            sa_t, sb_t, sa_p, sb_p = self.step_scalars(timestep)
            self._step += 1
            return ops.ddim_step(model_output, model_output_cond, guidance_scale, sample, sa_t, sb_t, sa_p, sb_p,
                                 self.prediction_type, self.clip_sample_range if self.clip_sample else 0.0, out=out)
        if eta < 0.0:
            raise ValueError(f"eta must be >= 0, got {eta}")
        if eta > 0.0 and variance_noise is not None and generator is not None:  # :459-464
            raise ValueError("Cannot pass both generator and variance_noise. Please make sure that either `generator` or"
                             " `variance_noise` stays `None`.")
        sa_t, sb_t, sa_p, sb_p, std = self.eta_step_scalars(timestep, eta)
        if eta > 0.0 and variance_noise is None and self._seed is None:
            from ..sampling import seed_from
            self._seed = seed_from(generator)
        self._step += 1
        return ops.ddim_eta_step(model_output, model_output_cond, guidance_scale, sample, variance_noise, sa_t, sb_t, sa_p,
                                 sb_p, std, self.prediction_type, self.clip_sample_range if self.clip_sample else 0.0,
                                 use_clipped_model_output, seed=self._seed or 0, step=self._step - 1, out=out)


class LCMScheduler:
    """ppdiffusers.LCMScheduler (scheduling_lcm.py:133-560) for latent consistency models: host-side fp32 scalars
    (numpy, bit-identical to the reference's 0-d fp32 tensors), one fused device kernel per step
    (b200mix_lcm_step: CFG combine, x0, clip, boundary-condition blend, noise injection)."""

    order = 1
    init_noise_sigma = 1.0

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.00085, beta_end: float = 0.012,
                 beta_schedule: str = "scaled_linear", original_inference_steps: int = 50, clip_sample: bool = False,
                 clip_sample_range: float = 1.0, set_alpha_to_one: bool = True, steps_offset: int = 0,
                 prediction_type: str = "epsilon", thresholding: bool = False, timestep_spacing: str = "leading",
                 timestep_scaling: float = 10.0, rescale_betas_zero_snr: bool = False):
        if thresholding or rescale_betas_zero_snr:
            raise NotImplementedError("LCMScheduler(b200): thresholding / rescale_betas_zero_snr are outside the hot path")
        if prediction_type not in ("epsilon", "sample", "v_prediction"):
            raise ValueError(f"prediction_type given as {prediction_type} must be one of `epsilon`, `sample` or"
                             " `v_prediction` for `LCMScheduler`.")
        self.betas, self.alphas, self.alphas_cumprod = _beta_tables(beta_schedule, beta_start, beta_end,
                                                                    num_train_timesteps, type(self))
        self.final_alpha_cumprod = f32(1.0) if set_alpha_to_one else self.alphas_cumprod[0]
        self.num_train_timesteps, self.original_inference_steps = num_train_timesteps, original_inference_steps
        self.clip_sample, self.clip_sample_range = clip_sample, clip_sample_range
        self.prediction_type, self.timestep_scaling = prediction_type, timestep_scaling
        self.num_inference_steps: Optional[int] = None
        self.timesteps = np.arange(0, num_train_timesteps)[::-1].copy().astype(np.int64)
        self._step_index = None

    @property
    def step_index(self):
        return self._step_index

    def scale_model_input(self, sample, timestep=None):
        return sample

    def set_timesteps(self, num_inference_steps: Optional[int] = None, original_inference_steps: Optional[int] = None,
                      timesteps=None, strength: float = 1.0):
        if num_inference_steps is None and timesteps is None:
            raise ValueError("Must pass exactly one of `num_inference_steps` or `custom_timesteps`.")
        if num_inference_steps is not None and timesteps is not None:
            raise ValueError("Can only pass one of `num_inference_steps` or `custom_timesteps`.")
        original_steps = original_inference_steps if original_inference_steps is not None else self.original_inference_steps
        if original_steps > self.num_train_timesteps:
            raise ValueError(f"`original_steps`: {original_steps} cannot be larger than `self.config.train_timesteps`:"
                             f" {self.num_train_timesteps} as the unet model trained with this scheduler can only handle"
                             f" maximal {self.num_train_timesteps} timesteps.")
        k = self.num_train_timesteps // original_steps
        origin = np.asarray(list(range(1, int(original_steps * strength) + 1))) * k - 1
        if timesteps is not None:
            for i in range(1, len(timesteps)):
                if timesteps[i] >= timesteps[i - 1]:
                    raise ValueError("`custom_timesteps` must be in descending order.")
            if timesteps[0] >= self.num_train_timesteps:
                raise ValueError(f"`timesteps` must start before `self.config.train_timesteps`: {self.num_train_timesteps}.")
            ts = np.array(timesteps, dtype=np.int64)
            self.num_inference_steps = len(ts)
            init_timestep = min(int(self.num_inference_steps * strength), self.num_inference_steps)
            ts = ts[max(self.num_inference_steps - init_timestep, 0) * self.order:]
        else:
            if num_inference_steps > self.num_train_timesteps:
                raise ValueError(f"`num_inference_steps`: {num_inference_steps} cannot be larger than "
                                 f"`self.config.train_timesteps`: {self.num_train_timesteps}")
            if len(origin) // num_inference_steps < 1:
                raise ValueError(f"The combination of `original_steps x strength`: {original_steps} x {strength} is smaller "
                                 f"than `num_inference_steps`: {num_inference_steps}.")
            if num_inference_steps > original_steps:
                raise ValueError(f"`num_inference_steps`: {num_inference_steps} cannot be larger than "
                                 f"`original_inference_steps`: {original_steps}")
            self.num_inference_steps = num_inference_steps
            origin = origin[::-1].copy()
            idx = np.floor(np.linspace(0, len(origin), num=num_inference_steps, endpoint=False)).astype(np.int64)
            ts = origin[idx]
        self.timesteps = ts.astype(np.int64)
        self._step_index = None

    def _init_step_index(self, timestep):
        cand = np.nonzero(self.timesteps == int(timestep))[0]
        self._step_index = int(cand[1] if len(cand) > 1 else cand[0])

    def get_scalings_for_boundary_condition_discrete(self, timestep):
        """scheduling_lcm.py:453-459 in fp32 (an int64 0-d tensor times a Python float is an fp32 tensor in Paddle)."""
        sd2 = f32(0.5 ** 2)
        st = f32(f32(int(timestep)) * f32(self.timestep_scaling))
        den = f32(f32(st * st) + sd2)
        return f32(sd2 / den), f32(st / np.sqrt(den, dtype=f32))

    def step_scalars(self, timestep):
        """(sqrt(a_t), sqrt(1-a_t), c_skip, c_out, sqrt(a_prev), sqrt(1-a_prev), is_last_step) as fp32 values."""
        if self.num_inference_steps is None:
            raise ValueError("Number of inference steps is 'None', you need to run 'set_timesteps' after creating the "
                             "scheduler")
        timestep = int(timestep)
        if self._step_index is None:
            self._init_step_index(timestep)
        nxt = self._step_index + 1
        prev_timestep = int(self.timesteps[nxt]) if nxt < len(self.timesteps) else timestep
        a_t = self.alphas_cumprod[timestep]
        a_p = self.alphas_cumprod[prev_timestep] if prev_timestep >= 0 else self.final_alpha_cumprod
        c_skip, c_out = self.get_scalings_for_boundary_condition_discrete(timestep)
        return (float(np.sqrt(a_t, dtype=f32)), float(np.sqrt(f32(f32(1) - a_t), dtype=f32)), float(c_skip), float(c_out),
                float(np.sqrt(a_p, dtype=f32)), float(np.sqrt(f32(f32(1) - a_p), dtype=f32)),
                self._step_index == self.num_inference_steps - 1)

    def step(self, model_output, timestep, sample, generator=None, model_output_cond=None, guidance_scale=0.0,
             noise=None, out=None, return_denoised=False):
        """sample / result: fp32 CUDA tensors. Multi-step sampling injects z ~ N(0, I) (scheduling_lcm.py:538-545): pass
        `noise` (fp32 CUDA tensor) or a torch `generator` (a CUDA generator of the sample's device); the final step is
        deterministic. With return_denoised also returns LCMSchedulerOutput.denoised."""
        import torch

        from .. import ops
        sa_t, sb_t, c_skip, c_out, sa_p, sb_p, last = self.step_scalars(timestep)
        if not last and noise is None:
            noise = torch.randn(sample.shape, device=sample.device, dtype=torch.float32, generator=generator)
        den = torch.empty_like(sample) if return_denoised else None
        res = ops.lcm_step(model_output, model_output_cond, guidance_scale, sample, None if last else noise, sa_t, sb_t,
                           c_skip, c_out, sa_p, sb_p, self.prediction_type,
                           self.clip_sample_range if self.clip_sample else 0.0, out=out, denoised=den)
        self._step_index += 1
        return (res, den) if return_denoised else res


def _linspace_f32(start, end, n):
    """float32 linspace as the CPU kernels of Paddle / torch define it: start + i*step for the first half,
    end - (n-1-i)*step for the second half, step = (end-start)/(n-1), everything in fp32."""
    start, end = f32(start), f32(end)
    step = f32((end - start) / f32(n - 1))
    i = np.arange(n)
    half = n // 2
    lo = (start + step * i.astype(f32)).astype(f32)
    hi = (end - step * (n - 1 - i).astype(f32)).astype(f32)
    return np.where(i < half, lo, hi).astype(f32)


def _cumprod_f32(a):
    out = np.empty_like(a, dtype=f32)
    acc = f32(1.0)
    for i, v in enumerate(a):
        acc = f32(acc * v)
        out[i] = acc
    return out


class FlowMatchEulerDiscreteScheduler:
    """ppdiffusers.FlowMatchEulerDiscreteScheduler (scheduling_flow_match_euler_discrete.py:44)."""

    order = 1

    def __init__(self, num_train_timesteps: int = 1000, shift: float = 1.0):
        self.num_train_timesteps, self.shift = num_train_timesteps, shift
        t = np.linspace(1, num_train_timesteps, num_train_timesteps, dtype=f32)[::-1].copy()
        sigmas = (t / f32(num_train_timesteps)).astype(f32)
        sigmas = (f32(shift) * sigmas / (f32(1) + f32(shift - 1) * sigmas)).astype(f32)
        self.timesteps = (sigmas * f32(num_train_timesteps)).astype(f32)
        self.sigmas = sigmas
        self.sigma_min, self.sigma_max = float(sigmas[-1]), float(sigmas[0])
        self._step_index = None

    def set_timesteps(self, num_inference_steps: int):
        self.num_inference_steps = num_inference_steps
        t = np.linspace(self.sigma_max * self.num_train_timesteps, self.sigma_min * self.num_train_timesteps,
                        num_inference_steps)
        sigmas = t / self.num_train_timesteps
        sigmas = self.shift * sigmas / (1 + (self.shift - 1) * sigmas)
        sigmas = sigmas.astype(f32)
        self.timesteps = (sigmas * f32(self.num_train_timesteps)).astype(f32)
        self.sigmas = np.concatenate([sigmas, np.zeros(1, dtype=f32)])
        self._step_index = None

    def step_scalars(self, timestep):
        if self._step_index is None:
            idx = np.nonzero(self.timesteps == f32(timestep))[0]
            self._step_index = int(idx[0])
        sigma = self.sigmas[self._step_index]
        dt = f32(self.sigmas[self._step_index + 1] - sigma)
        self._step_index += 1
        return float(sigma), float(dt)

    def step(self, model_output, timestep, sample, model_output_cond=None, guidance_scale=0.0, out=None):
        from .. import ops
        sigma, dt = self.step_scalars(timestep)
        return ops.euler_step(model_output, model_output_cond, guidance_scale, sample, sigma, dt, out=out)


class EulerDiscreteScheduler:
    """ppdiffusers.EulerDiscreteScheduler (scheduling_euler_discrete.py:135-503; SDXL's default sampler) restricted to
    the deterministic path the pipelines use (s_churn = 0 => gamma = 0, sigma_hat = sigma; epsilon prediction). All
    schedule arithmetic runs on the host in numpy with the reference's dtypes (fp32 tensors -> np.float32, its
    np.interp / Karras ramp / _sigma_to_t pieces in float64); the per-step update is the same fp32 expression as the
    reference's (`pred = x - sigma*eps; derivative = (x - pred)/sigma; x + derivative*dt`), which is exactly
    `b200mix_euler_step`; `scale_model_input` is `b200mix_scale_model_input` (x / sqrt(sigma^2 + 1) with an IEEE fp32
    division)."""

    order = 1

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.0001, beta_end: float = 0.02,
                 beta_schedule: str = "linear", prediction_type: str = "epsilon", interpolation_type: str = "linear",
                 use_karras_sigmas: bool = False, sigma_min: Optional[float] = None, sigma_max: Optional[float] = None,
                 timestep_spacing: str = "linspace", timestep_type: str = "discrete", steps_offset: int = 0):
        self.betas, self.alphas, self.alphas_cumprod = _beta_tables(beta_schedule, beta_start, beta_end,
                                                                    num_train_timesteps, type(self))
        if prediction_type != "epsilon":
            raise NotImplementedError("EulerDiscreteScheduler(b200): only prediction_type='epsilon' has a device step")
        if timestep_type != "discrete":
            raise NotImplementedError("EulerDiscreteScheduler(b200): only timestep_type='discrete'")
        self.num_train_timesteps = num_train_timesteps
        self.interpolation_type, self.use_karras_sigmas = interpolation_type, use_karras_sigmas
        self.sigma_min, self.sigma_max = sigma_min, sigma_max
        self.timestep_spacing, self.steps_offset = timestep_spacing, steps_offset
        sig = _train_sigmas(self.alphas_cumprod)
        self.timesteps = np.linspace(0, num_train_timesteps - 1, num_train_timesteps, dtype=float)[::-1].astype(f32)
        self.sigmas = np.concatenate([sig[::-1], np.zeros(1, dtype=f32)]).astype(f32)
        self.num_inference_steps: Optional[int] = None
        self._step_index: Optional[int] = None

    @property
    def init_noise_sigma(self) -> float:
        m = self.sigmas.max()
        if self.timestep_spacing in ("linspace", "trailing"):
            return float(m)
        return float(np.sqrt(f32(f32(m * m) + f32(1.0)), dtype=f32))

    def set_timesteps(self, num_inference_steps: int):
        N = self.num_train_timesteps
        self.num_inference_steps = num_inference_steps
        if self.timestep_spacing == "linspace":
            timesteps = np.linspace(0, N - 1, num_inference_steps, dtype=f32)[::-1].copy()
        elif self.timestep_spacing == "leading":
            step_ratio = N // num_inference_steps
            timesteps = (np.arange(0, num_inference_steps) * step_ratio).round()[::-1].copy().astype(f32)
            timesteps += self.steps_offset
        elif self.timestep_spacing == "trailing":
            step_ratio = N / num_inference_steps
            timesteps = (np.arange(N, 0, -step_ratio)).round().copy().astype(f32)
            timesteps -= 1
        else:
            raise ValueError(f"{self.timestep_spacing} is not supported. Please make sure to choose one of 'linspace', "
                             "'leading' or 'trailing'.")
        sigmas = _train_sigmas(self.alphas_cumprod)
        log_sigmas = np.log(sigmas)
        if self.interpolation_type == "linear":
            sigmas = np.interp(timesteps, np.arange(0, len(sigmas)), sigmas)
        elif self.interpolation_type == "log_linear":
            sigmas = np.exp(np.linspace(np.log(sigmas[-1]), np.log(sigmas[0]), num_inference_steps + 1, dtype=f32))
        else:
            raise ValueError(f"{self.interpolation_type} is not implemented. Please specify interpolation_type to either"
                             " 'linear' or 'log_linear'")
        if self.use_karras_sigmas:
            smin = self.sigma_min if self.sigma_min is not None else sigmas[-1].item()
            smax = self.sigma_max if self.sigma_max is not None else sigmas[0].item()
            sigmas = _karras_sigmas(smin, smax, num_inference_steps)
            timesteps = np.array([_sigma_to_t(s, log_sigmas) for s in sigmas])
        self.timesteps = np.asarray(timesteps).astype(f32)
        self.sigmas = np.concatenate([np.asarray(sigmas).astype(f32), np.zeros(1, dtype=f32)])
        self._step_index = None

    def _init_step_index(self, timestep):
        cand = np.nonzero(self.timesteps == f32(timestep))[0]
        if len(cand) == 0:
            raise ValueError(f"timestep {timestep} is not one of scheduler.timesteps")
        self._step_index = int(cand[1] if len(cand) > 1 else cand[0])

    def input_scale_denominator(self, timestep) -> float:
        """(sigma^2 + 1) ** 0.5 in fp32: what scale_model_input divides the sample by."""
        if self._step_index is None:
            self._init_step_index(timestep)
        s = self.sigmas[self._step_index]
        return float(np.sqrt(f32(f32(s * s) + f32(1.0)), dtype=f32))

    def scale_model_input(self, sample, timestep, out=None):
        from .. import ops
        return ops.scale_model_input(sample, self.input_scale_denominator(timestep), out=out)

    def step_scalars(self, timestep):
        if isinstance(timestep, (int, np.integer)):
            raise ValueError("Passing integer indices (e.g. from `enumerate(timesteps)`) as timesteps to "
                             "`EulerDiscreteScheduler.step()` is not supported. Make sure to pass one of the "
                             "`scheduler.timesteps` as a timestep.")
        if self._step_index is None:
            self._init_step_index(timestep)
        sigma = self.sigmas[self._step_index]
        dt = f32(self.sigmas[self._step_index + 1] - sigma)
        self._step_index += 1
        return float(sigma), float(dt)

    def step(self, model_output, timestep, sample, model_output_cond=None, guidance_scale=0.0, out=None):
        from .. import ops
        sigma, dt = self.step_scalars(timestep)
        return ops.euler_step(model_output, model_output_cond, guidance_scale, sample, sigma, dt, out=out)

    def add_noise_sigma(self, timestep) -> float:
        """sigma of `timestep`: add_noise is original + noise * sigma (scheduling_euler_discrete.py:472-497)."""
        idx = np.nonzero(self.timesteps == f32(timestep))[0]
        return float(self.sigmas[int(idx[0])])


class DPMSolverMultistepScheduler:
    """ppdiffusers.DPMSolverMultistepScheduler (scheduling_dpmsolver_multistep.py:36-919) restricted to what has a device
    step: algorithm "dpmsolver++" (the "DPM-Solver++ 2M" sampler of SD / SDXL) or "sde-dpmsolver++" ("DPM-Solver++ 2M
    SDE"), solver_type "midpoint", order 1 or 2, epsilon prediction, incl. Karras sigmas / Lu lambdas,
    lower_order_final, euler_at_final. The schedule and the per-step scalars are computed on the host in numpy with the
    reference's dtypes; `step` runs ONE fused kernel (`b200mix_dpmpp_2m_step`, `b200mix_dpmpp_2m_sde_step`): CFG
    combine, x0 = (x - sigma_t*eps)/alpha_t, the first / second order update in the reference's operation order, and
    the x0 history for the next step (kept on the device).

    The SDE's noise is a standard normal per element. `step(..., noise=...)` uses the given fp32 tensor; otherwise the
    first step after set_timesteps draws one 63-bit seed from `generator` (torch's default generator when None), and
    every step takes counter-based Philox normals keyed by (seed, step index), drawn inside the kernel, exactly as
    EulerAncestralDiscreteScheduler does. One generator state therefore gives one result, on any GPU and with or
    without CUDA graphs, but not Paddle's draws. In a data-parallel run every rank steps its own slice of the batch with
    its own scheduler: the noise is keyed by that rank's generator and by the element's index within the rank's
    latents, not by the image's global index, so ranks given equal generator states draw equal noise for their
    slices."""

    order = 1
    init_noise_sigma = 1.0
    takes_generator = True  # step(..., generator=) seeds the SDE's noise (see the class docstring)

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.0001, beta_end: float = 0.02,
                 beta_schedule: str = "linear", solver_order: int = 2, prediction_type: str = "epsilon",
                 thresholding: bool = False, sample_max_value: float = 1.0, algorithm_type: str = "dpmsolver++",
                 solver_type: str = "midpoint", lower_order_final: bool = True, euler_at_final: bool = False,
                 use_karras_sigmas: bool = False, use_lu_lambdas: bool = False, lambda_min_clipped: float = -float("inf"),
                 variance_type: Optional[str] = None, timestep_spacing: str = "linspace", steps_offset: int = 0):
        self.betas, self.alphas, self.alphas_cumprod = _beta_tables(beta_schedule, beta_start, beta_end,
                                                                    num_train_timesteps, type(self))
        if (algorithm_type not in ("dpmsolver++", "sde-dpmsolver++") or solver_type != "midpoint" or
                solver_order not in (1, 2) or thresholding or prediction_type != "epsilon" or variance_type):
            raise NotImplementedError("DPMSolverMultistepScheduler(b200): the device step covers dpmsolver++ / "
                                      "sde-dpmsolver++ / midpoint / order 1-2 / epsilon prediction without thresholding")
        self.algorithm_type = algorithm_type
        self.num_train_timesteps, self.solver_order = num_train_timesteps, solver_order
        self.lower_order_final, self.euler_at_final = lower_order_final, euler_at_final
        self.use_karras_sigmas, self.use_lu_lambdas = use_karras_sigmas, use_lu_lambdas
        self.lambda_min_clipped = lambda_min_clipped
        self.timestep_spacing, self.steps_offset = timestep_spacing, steps_offset
        self.num_inference_steps: Optional[int] = None
        self.timesteps = np.linspace(0, num_train_timesteps - 1, num_train_timesteps, dtype=f32)[::-1].copy()
        self.lower_order_nums = 0
        self._step_index: Optional[int] = None
        self._m_prev = None  # x0 prediction of the previous step (device fp32)
        self._seed: Optional[int] = None  # the SDE's Philox key

    def scale_model_input(self, sample, timestep=None):
        return sample

    def set_timesteps(self, num_inference_steps: int):
        N = self.num_train_timesteps
        ac = self.alphas_cumprod
        if np.isinf(self.lambda_min_clipped):
            clipped_idx = 0
        else:
            lam = np.log(np.sqrt(ac, dtype=f32), dtype=f32) - np.log(np.sqrt((f32(1.0) - ac).astype(f32), dtype=f32), dtype=f32)
            clipped_idx = int(np.searchsorted(np.flip(lam), f32(self.lambda_min_clipped)))
        self.timesteps, self.sigmas = _multistep_schedule(ac, num_inference_steps, self.timestep_spacing, self.steps_offset,
                                                          self.use_karras_sigmas, self.use_lu_lambdas, N - clipped_idx)
        self.num_inference_steps = len(self.timesteps)
        self.lower_order_nums = 0
        self._step_index = None
        self._m_prev = None
        self._seed = None

    @staticmethod
    def _alpha_sigma_lambda(sigma):
        """_sigma_to_alpha_sigma_t (:362-366) + lambda = log(alpha) - log(sigma), all fp32."""
        sigma = f32(sigma)
        alpha_t = f32(f32(1.0) / np.sqrt(f32(f32(sigma * sigma) + f32(1.0)), dtype=f32))
        sigma_t = f32(sigma * alpha_t)
        return alpha_t, sigma_t, f32(np.log(alpha_t, dtype=f32) - np.log(sigma_t, dtype=f32))

    def _advance(self, timestep):
        """(first order?, alpha_s0, sigma_s0, alpha_t, sigma_t, h, inv_r0) of this step (the reference's control flow in
        step, :802-880), advancing the step index and the lower-order count."""
        if self.num_inference_steps is None:
            raise ValueError("Number of inference steps is 'None', you need to run 'set_timesteps' after creating the scheduler")
        if self._step_index is None:
            cand = np.nonzero(self.timesteps == int(timestep))[0]
            self._step_index = len(self.timesteps) - 1 if len(cand) == 0 else int(cand[1] if len(cand) > 1 else cand[0])
        i, n = self._step_index, len(self.timesteps)
        lower_order_final = (i == n - 1) and (self.euler_at_final or (self.lower_order_final and n < 15))
        alpha_s0, sigma_s0, lam_s0 = self._alpha_sigma_lambda(self.sigmas[i])
        alpha_t, sigma_t, lam_t = self._alpha_sigma_lambda(self.sigmas[i + 1])
        h = f32(lam_t - lam_s0)
        first = self.solver_order == 1 or self.lower_order_nums < 1 or lower_order_final
        inv_r0 = f32(0.0)
        if not first:
            _, _, lam_s1 = self._alpha_sigma_lambda(self.sigmas[i - 1])
            # Karras / Lu schedules repeat the last sigma: h == 0 there, r0 = inf, 1/r0 = 0 and C = 0 (x' = x), exactly
            # like the reference's 0-d tensor arithmetic
            with np.errstate(divide="ignore", invalid="ignore"):
                r0 = f32(f32(lam_s0 - lam_s1) / h)
                inv_r0 = f32(f32(1.0) / r0)
        if self.lower_order_nums < self.solver_order:
            self.lower_order_nums += 1
        self._step_index += 1
        return first, alpha_s0, sigma_s0, alpha_t, sigma_t, h, inv_r0

    def step_scalars(self, timestep):
        """(order, sigma_cur, alpha_cur, A, C, halfC, inv_r0): x0 = (x - sigma_cur*eps)/alpha_cur;
        order 1: x' = A*x - C*x0; order 2: x' = A*x - C*x0 - halfC*(inv_r0*(x0 - x0_prev))."""
        first, alpha_s0, sigma_s0, alpha_t, sigma_t, h, inv_r0 = self._advance(timestep)
        A = f32(sigma_t / sigma_s0)
        C = f32(alpha_t * f32(np.exp(f32(-h), dtype=f32) - f32(1.0)))
        return (1 if first else 2, float(sigma_s0), float(alpha_s0), float(A), float(C), float(f32(f32(0.5) * C)), float(inv_r0))

    def sde_step_scalars(self, timestep):
        """(order, sigma_cur, alpha_cur, A, B, halfB, inv_r0, N) of an "sde-dpmsolver++" step (:561-567, :666-674):
        x0 = (x - sigma_cur*eps)/alpha_cur; order 1: x' = A*x + B*x0 + N*z; order 2: x' = A*x + B*x0 +
        halfB*(inv_r0*(x0 - x0_prev)) + N*z, with A = sigma_t/sigma_s0*exp(-h), B = alpha_t*(1 - exp(-2h)),
        halfB = 0.5*B and N = sigma_t*sqrt(1 - exp(-2h))."""
        first, alpha_s0, sigma_s0, alpha_t, sigma_t, h, inv_r0 = self._advance(timestep)
        A = f32(f32(sigma_t / sigma_s0) * np.exp(f32(-h), dtype=f32))
        one_minus = f32(f32(1.0) - np.exp(f32(f32(-2.0) * h), dtype=f32))
        B = f32(alpha_t * one_minus)
        N = f32(sigma_t * np.sqrt(one_minus, dtype=f32))
        return (1 if first else 2, float(sigma_s0), float(alpha_s0), float(A), float(B), float(f32(f32(0.5) * B)),
                float(inv_r0), float(N))

    def step(self, model_output, timestep, sample, model_output_cond=None, guidance_scale=0.0, out=None, generator=None,
             noise=None):
        """sample / result: fp32 CUDA tensors (out may be sample); model_output (and model_output_cond, same dtype, for
        the fused CFG combine) bf16 / fp32 with sample's element count. "sde-dpmsolver++" only: noise is fp32 standard
        normals like sample, or None for the Philox stream described in the class docstring."""
        from .. import ops
        sde = self.algorithm_type == "sde-dpmsolver++"
        if noise is not None and not sde:
            raise ValueError("DPMSolverMultistepScheduler: only algorithm_type='sde-dpmsolver++' takes noise")
        if sde:
            order, sigma_cur, alpha_cur, A, B, halfB, inv_r0, N = self.sde_step_scalars(timestep)
        else:
            order, sigma_cur, alpha_cur, A, C, halfC, inv_r0 = self.step_scalars(timestep)
        if self._m_prev is None:
            import torch
            self._m_prev = [torch.empty_like(sample), torch.empty_like(sample)]
            self._m_slot = 0
        m_out, m_prev = self._m_prev[self._m_slot], self._m_prev[self._m_slot ^ 1]
        self._m_slot ^= 1
        if not sde:
            return ops.dpmpp_2m_step(model_output, model_output_cond, guidance_scale, sample,
                                     m_prev if order == 2 else None, m_out, sigma_cur, alpha_cur, A, C, halfC, inv_r0,
                                     out=out)
        if noise is None and self._seed is None:
            from ..sampling import seed_from
            self._seed = seed_from(generator)
        return ops.dpmpp_2m_sde_step(model_output, model_output_cond, guidance_scale, sample, noise,
                                     m_prev if order == 2 else None, m_out, sigma_cur, alpha_cur, A, B, halfB, inv_r0, N,
                                     seed=self._seed or 0, step=self._step_index - 1, out=out)


class EulerAncestralDiscreteScheduler(EulerDiscreteScheduler):
    """ppdiffusers.EulerAncestralDiscreteScheduler ("Euler a", scheduling_euler_ancestral_discrete.py:130-389):
    EulerDiscreteScheduler's schedule, init_noise_sigma and scale_model_input (the reference's set_timesteps :210-250
    is EulerDiscrete's linear-interpolation path), epsilon / v_prediction. sigma_up / sigma_down (:339-347) and the
    v-prediction factors are fp32 host scalars; `step` is one fused kernel (b200mix_euler_ancestral_step): CFG
    combine, x0, the Euler move to sigma_down and the ancestral noise times sigma_up.

    The noise is a standard normal per element. `step(..., noise=...)` uses the given fp32 tensor; otherwise the first
    step after set_timesteps draws one 63-bit seed from `generator` (torch's default generator when None) and every step
    takes counter-based Philox normals keyed by (seed, step index), drawn inside the kernel. One generator state
    therefore gives one result, on any GPU and with or without CUDA graphs; the draws cannot reproduce Paddle's RNG,
    so images differ from the reference's for the same seed, as between any two RNGs. In a data-parallel run every rank
    steps its own slice of the batch with its own scheduler: the noise is keyed by that rank's generator and by the
    element's index within the rank's latents, not by the image's global index."""

    takes_generator = True  # step(..., generator=) seeds the noise

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.0001, beta_end: float = 0.02,
                 beta_schedule: str = "linear", trained_betas=None, prediction_type: str = "epsilon",
                 timestep_spacing: str = "linspace", steps_offset: int = 0):
        if trained_betas is not None:
            raise NotImplementedError("EulerAncestralDiscreteScheduler(b200): trained_betas are not supported")
        if prediction_type == "sample":
            raise NotImplementedError("prediction_type not implemented yet: sample")
        if prediction_type not in ("epsilon", "v_prediction"):
            raise ValueError(f"prediction_type given as {prediction_type} must be one of `epsilon`, or `v_prediction`")
        # the parent's schedule does not depend on prediction_type; its own step covers epsilon only
        super().__init__(num_train_timesteps, beta_start, beta_end, beta_schedule, timestep_spacing=timestep_spacing,
                         steps_offset=steps_offset)
        self.prediction_type = prediction_type
        self._seed: Optional[int] = None

    def set_timesteps(self, num_inference_steps: int):
        super().set_timesteps(num_inference_steps)
        self._seed = None

    def step_scalars(self, timestep):
        """(sigma, c_out, s2p1, dt, sigma_up) of this step as fp32 values, advancing the step index:
        c_out = -sigma/(sigma^2+1)^0.5 and s2p1 = sigma^2+1 (v-prediction), sigma_up, and dt = sigma_down - sigma."""
        if isinstance(timestep, (int, np.integer)):
            raise ValueError("Passing integer indices (e.g. from `enumerate(timesteps)`) as timesteps to "
                             "`EulerDiscreteScheduler.step()` is not supported. Make sure to pass one of the "
                             "`scheduler.timesteps` as a timestep.")
        if self._step_index is None:
            self._init_step_index(timestep)
        s_from, s_to = self.sigmas[self._step_index], self.sigmas[self._step_index + 1]
        f2, t2 = f32(s_from * s_from), f32(s_to * s_to)
        sigma_up = np.sqrt(f32(f32(t2 * f32(f2 - t2)) / f2), dtype=f32)
        sigma_down = np.sqrt(f32(t2 - f32(sigma_up * sigma_up)), dtype=f32)
        s2p1 = f32(f2 + f32(1.0))
        c_out = f32(f32(-s_from) / np.sqrt(s2p1, dtype=f32))
        self._step_index += 1
        return float(s_from), float(c_out), float(s2p1), float(f32(sigma_down - s_from)), float(sigma_up)

    def step(self, model_output, timestep, sample, generator=None, noise=None, model_output_cond=None,
             guidance_scale=0.0, out=None):
        """sample / result: fp32 CUDA tensors (out may be sample); model_output (and model_output_cond, same dtype, for
        the fused CFG combine) bf16 / fp32 with sample's element count. noise: fp32 standard normals like sample, or None
        for the Philox stream described in the class docstring."""
        from .. import ops
        from ..sampling import seed_from
        if self._step_index is None:
            self._init_step_index(timestep)
        index = self._step_index
        if noise is None and self._seed is None:
            self._seed = seed_from(generator)
        sigma, c_out, s2p1, dt, sigma_up = self.step_scalars(timestep)
        return ops.euler_ancestral_step(model_output, model_output_cond, guidance_scale, sample, noise, sigma, c_out, s2p1,
                                        dt, sigma_up, self.prediction_type, seed=self._seed or 0, step=index, out=out)


class UniPCMultistepScheduler:
    """ppdiffusers.UniPCMultistepScheduler (scheduling_unipc_multistep.py:138-843) with predict_x0 = True: solver_type
    bh1 / bh2, solver_order 1-3, lower_order_final, disable_corrector, Karras sigmas, the three spacings,
    epsilon / sample / v_prediction. The schedule is DPM-Solver's (_multistep_schedule); the per-step scalars of
    convert_model_output, UniC and UniP (:368-701, including the order-3 linalg.solve) are computed on the host in
    numpy fp32 like the reference's 0-d tensors, and `step` runs ONE fused kernel (b200mix_unipc_step): CFG combine, x0,
    corrector, predictor. The x0 history (solver_order + 1 device buffers used as a ring) and last_sample live on the
    device, are owned by the scheduler and never alias the caller's tensors; set_timesteps resets them."""

    order = 1
    init_noise_sigma = 1.0

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.0001, beta_end: float = 0.02,
                 beta_schedule: str = "linear", trained_betas=None, solver_order: int = 2,
                 prediction_type: str = "epsilon", thresholding: bool = False,
                 dynamic_thresholding_ratio: float = 0.995, sample_max_value: float = 1.0, predict_x0: bool = True,
                 solver_type: str = "bh2", lower_order_final: bool = True, disable_corrector=(), solver_p=None,
                 use_karras_sigmas: Optional[bool] = False, timestep_spacing: str = "linspace", steps_offset: int = 0):
        if trained_betas is not None or thresholding or not predict_x0 or solver_p is not None:
            raise NotImplementedError("UniPCMultistepScheduler(b200): the device step covers predict_x0 = True without "
                                      "thresholding, solver_p or trained_betas")
        if solver_order not in (1, 2, 3):
            raise NotImplementedError("UniPCMultistepScheduler(b200): the device step covers solver_order 1-3")
        if prediction_type not in ("epsilon", "sample", "v_prediction"):
            raise ValueError(f"prediction_type given as {prediction_type} must be one of `epsilon`, `sample`, or"
                             " `v_prediction` for the UniPCMultistepScheduler.")
        self.betas, self.alphas, self.alphas_cumprod = _beta_tables(beta_schedule, beta_start, beta_end,
                                                                    num_train_timesteps, type(self))
        if solver_type not in ("bh1", "bh2"):
            if solver_type not in ("midpoint", "heun", "logrho"):
                raise NotImplementedError(f"{solver_type} does is not implemented for {type(self)}")
            solver_type = "bh2"  # :184-188
        self.num_train_timesteps, self.solver_order, self.solver_type = num_train_timesteps, solver_order, solver_type
        self.prediction_type, self.lower_order_final = prediction_type, lower_order_final
        self.disable_corrector = list(disable_corrector)
        self.use_karras_sigmas, self.timestep_spacing, self.steps_offset = use_karras_sigmas, timestep_spacing, steps_offset
        self.num_inference_steps: Optional[int] = None
        self.timesteps = np.linspace(0, num_train_timesteps - 1, num_train_timesteps, dtype=f32)[::-1].copy()
        self._reset()

    def _reset(self):
        self.lower_order_nums = 0
        self.this_order = None
        self._step_index: Optional[int] = None
        self._has_last = False  # the reference's `last_sample is not None`
        self._bufs = None       # solver_order + 1 x0 buffers, then last_sample (device fp32)
        self._hist = []         # indices into _bufs of the x0 history, oldest first

    @property
    def step_index(self):
        return self._step_index

    def scale_model_input(self, sample, *args, **kwargs):
        return sample

    def set_timesteps(self, num_inference_steps: int):
        self.timesteps, self.sigmas = _multistep_schedule(self.alphas_cumprod, num_inference_steps, self.timestep_spacing,
                                                          self.steps_offset, self.use_karras_sigmas)
        self.num_inference_steps = len(self.timesteps)
        self._reset()

    def _init_step_index(self, timestep):  # :703-718
        cand = np.nonzero(self.timesteps == int(timestep))[0]
        self._step_index = len(self.timesteps) - 1 if len(cand) == 0 else int(cand[1] if len(cand) > 1 else cand[0])

    def _bh_coefficients(self, i_t, i_s0, hist, order, corrector):
        """(A, K, E, rks, rhos) of multistep_uni_c_bh_update (corrector) / multistep_uni_p_bh_update from sigma index
        i_s0 to i_t with history sigma indices `hist`: A = sigma_t/sigma_s0, K = alpha_t*h_phi_1, E = alpha_t*B_h.
        Karras schedules repeat their last sigma: the final step has h = 0, rk = +-inf and h_phi_k = 0/0 = nan, and
        the order-1 / order-2 updates reduce to x' = x exactly like the reference's 0-d tensor arithmetic (K = E = -0,
        (m_k - m0)/rk = 0); a solve over nan (order 3 without lower_order_final) gives nan there, as in the reference."""
        alpha_t, sigma_t, lam_t = DPMSolverMultistepScheduler._alpha_sigma_lambda(self.sigmas[i_t])
        _, sigma_s0, lam_s0 = DPMSolverMultistepScheduler._alpha_sigma_lambda(self.sigmas[i_s0])
        with np.errstate(divide="ignore", invalid="ignore"):
            h = f32(lam_t - lam_s0)
            rks = [f32(f32(DPMSolverMultistepScheduler._alpha_sigma_lambda(self.sigmas[si])[2] - lam_s0) / h) for si in hist]
            r = np.array(rks + [f32(1.0)], dtype=f32)
            hh = f32(-h)
            h_phi_1 = np.expm1(hh, dtype=f32)
            h_phi_k = f32(f32(h_phi_1 / hh) - f32(1.0))
            B_h = hh if self.solver_type == "bh1" else np.expm1(hh, dtype=f32)
            R, b, fact = [], [], 1
            for k in range(1, order + 1):
                R.append(r ** (k - 1))
                b.append(f32(f32(h_phi_k * f32(fact)) / B_h))
                fact *= k + 1
                h_phi_k = f32(f32(h_phi_k / hh) - f32(1 / fact))
            R, b = np.stack(R).astype(f32), np.array(b, dtype=f32)
            if corrector:
                rhos = [f32(0.5)] if order == 1 else list(np.linalg.solve(R, b).astype(f32))
            else:
                rhos = [] if order == 1 else [f32(0.5)] if order == 2 else list(np.linalg.solve(R[:-1, :-1], b[:-1]).astype(f32))
            return (f32(sigma_t / sigma_s0), f32(alpha_t * h_phi_1), f32(alpha_t * B_h), rks, rhos)

    def step_scalars(self, timestep):
        """The fp32 scalars of this step as a dict (the fields of b200mix_unipc_coeffs, with rc / rk_c / rp / rk_p one
        entry per history term, plus `corrector`, `order_c` and `order_p`), advancing the scheduler's state."""
        if self.num_inference_steps is None:
            raise ValueError("Number of inference steps is 'None', you need to run 'set_timesteps' after creating the "
                             "scheduler")
        if self._step_index is None:
            self._init_step_index(timestep)
        i, n = self._step_index, len(self.timesteps)
        alpha_t, sigma_t, _ = DPMSolverMultistepScheduler._alpha_sigma_lambda(self.sigmas[i])
        c = dict(alpha_t=float(alpha_t), sigma_t=float(sigma_t), corrector=False, order_c=0)
        if i > 0 and (i - 1) not in self.disable_corrector and self._has_last:  # :759-761
            p = self.this_order
            A, K, E, rks, rhos = self._bh_coefficients(i, i - 1, [i - 1 - k for k in range(1, p)], p, True)
            c.update(corrector=True, order_c=p, A_c=float(A), K_c=float(K), E_c=float(E), rc=[float(v) for v in rhos[:-1]],
                     rk_c=[float(v) for v in rks], rc_last=float(rhos[-1]))
        order = min(self.solver_order, n - i) if self.lower_order_final else self.solver_order  # :779-785
        self.this_order = min(order, self.lower_order_nums + 1)
        A, K, E, rks, rhos = self._bh_coefficients(i + 1, i, [i - k for k in range(1, self.this_order)], self.this_order,
                                                   False)
        c.update(order_p=self.this_order, A_p=float(A), K_p=float(K), E_p=float(E), rp=[float(v) for v in rhos],
                 rk_p=[float(v) for v in rks])
        self._has_last = True
        if self.lower_order_nums < self.solver_order:
            self.lower_order_nums += 1
        self._step_index += 1
        return c

    def step(self, model_output, timestep, sample, model_output_cond=None, guidance_scale=0.0, out=None):
        """sample / result: fp32 CUDA tensors (out may be sample); model_output (and model_output_cond, same dtype, for
        the fused CFG combine) bf16 / fp32 with sample's element count."""
        import torch

        from .. import ops
        c = self.step_scalars(timestep)
        if self._bufs is None:
            self._bufs = [torch.empty_like(sample, dtype=torch.float32) for _ in range(self.solver_order + 2)]
        bufs, hist = self._bufs, self._hist
        slot = next(j for j in range(self.solver_order + 1) if j not in hist)
        last = bufs[-1]
        corr = c["corrector"]
        res = ops.unipc_step(model_output, model_output_cond, guidance_scale, sample, c, bufs[slot], last,
                             last_sample=last if corr else None, m_prev=bufs[hist[-1]] if corr else None,
                             hist_c=[bufs[hist[-1 - k]] for k in range(1, c["order_c"])],
                             hist_p=[bufs[hist[-k]] for k in range(1, c["order_p"])],
                             prediction_type=self.prediction_type, out=out)
        hist.append(slot)
        if len(hist) > self.solver_order:
            hist.pop(0)
        return res
