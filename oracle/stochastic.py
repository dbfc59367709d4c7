"""ORACLE (test infrastructure, not product code): CPU fp32 restatements of the two noise-drawing steps that
oracle.samplers does not cover: DDIMScheduler with eta > 0 (ppdiffusers/schedulers/scheduling_ddim.py:350-475,
use_clipped_model_output included) and DPMSolverMultistepScheduler with algorithm_type "sde-dpmsolver++"
(scheduling_dpmsolver_multistep.py:507-880, midpoint, epsilon prediction, orders 1-2), with torch fp32 0-d tensors
standing in for paddle's (the helpers of oracle.schedulers).

Element-wise, each update runs in the reference's operation order, which is also the order of its device kernel, so a
device step can be compared bit for bit. The noise is either a tensor passed in or a seed, which draws
oracle.iddpm.philox_normal(seed, step, n), the device's Philox stream, at the step's index.
"""
import torch

from .iddpm import philox_normal
from .schedulers import DDIMScheduler as _DDIMScheduler
from .schedulers import DPMSolverMultistepScheduler, exp_f32, pow_half


def _noise_or_philox(noise, seed, step, sample):
    return philox_normal(seed, step, sample.numel()).reshape(sample.shape) if noise is None else noise


class DDIMScheduler(_DDIMScheduler):
    """scheduling_ddim.py:350-475 with eta >= 0, use_clipped_model_output and the variance noise given as a tensor or
    as a seed (the device's Philox stream at the index of the step call since set_timesteps)."""

    def set_timesteps(self, num_inference_steps):
        super().set_timesteps(num_inference_steps)
        self._step = 0

    def step(self, model_output, timestep, sample, eta=0.0, use_clipped_model_output=False, variance_noise=None,
             seed=0):  # :350-475
        timestep = int(timestep)
        prev_timestep = timestep - self.num_train_timesteps // self.num_inference_steps
        alpha_prod_t = self.alphas_cumprod[timestep]
        alpha_prod_t_prev = self.alphas_cumprod[prev_timestep] if prev_timestep >= 0 else self.final_alpha_cumprod
        beta_prod_t = 1 - alpha_prod_t
        if self.prediction_type == "epsilon":
            pred_original_sample = (sample - pow_half(beta_prod_t) * model_output) / pow_half(alpha_prod_t)
            pred_epsilon = model_output
        elif self.prediction_type == "sample":
            pred_original_sample = model_output
            pred_epsilon = (sample - pow_half(alpha_prod_t) * pred_original_sample) / pow_half(beta_prod_t)
        elif self.prediction_type == "v_prediction":
            pred_original_sample = (pow_half(alpha_prod_t)) * sample - (pow_half(beta_prod_t)) * model_output
            pred_epsilon = (pow_half(alpha_prod_t)) * model_output + (pow_half(beta_prod_t)) * sample
        else:
            raise ValueError(self.prediction_type)
        if self.clip_sample:
            pred_original_sample = pred_original_sample.clip(-self.clip_sample_range, self.clip_sample_range)
        variance = self._get_variance(timestep, prev_timestep)
        std_dev_t = eta * pow_half(variance)
        if use_clipped_model_output:
            pred_epsilon = (sample - pow_half(alpha_prod_t) * pred_original_sample) / pow_half(beta_prod_t)
        pred_sample_direction = pow_half(1 - alpha_prod_t_prev - std_dev_t ** 2) * pred_epsilon
        prev_sample = pow_half(alpha_prod_t_prev) * pred_original_sample + pred_sample_direction
        if eta > 0:
            prev_sample = prev_sample + std_dev_t * _noise_or_philox(variance_noise, seed, self._step, sample)
        self._step += 1
        return prev_sample

    def eta_step_scalars(self, timestep, eta):
        """(sqrt(a_t), sqrt(1-a_t), sqrt(a_prev), sqrt(1-a_prev-std^2), std) as step() computes them."""
        timestep = int(timestep)
        prev_timestep = timestep - self.num_train_timesteps // self.num_inference_steps
        a_t = self.alphas_cumprod[timestep]
        a_p = self.alphas_cumprod[prev_timestep] if prev_timestep >= 0 else self.final_alpha_cumprod
        std = eta * pow_half(self._get_variance(timestep, prev_timestep))
        return (pow_half(a_t).item(), pow_half(1 - a_t).item(), pow_half(a_p).item(),
                pow_half(1 - a_p - std ** 2).item(), std.item())


class DPMSolverSDEScheduler(DPMSolverMultistepScheduler):
    """DPMSolverMultistepScheduler with algorithm_type "sde-dpmsolver++", solver_type midpoint, epsilon prediction:
    dpm_solver_first_order_update :507-580 (:561-567), multistep_dpm_solver_second_order_update :582-700 (:666-674) and
    step :802-880 with the noise given as a tensor or as a seed (the device's Philox stream at the step index)."""

    def __init__(self, *args, algorithm_type="sde-dpmsolver++", **kw):
        if (algorithm_type != "sde-dpmsolver++" or kw.get("solver_type", "midpoint") != "midpoint" or
                kw.get("prediction_type", "epsilon") != "epsilon"):
            raise NotImplementedError("oracle: sde-dpmsolver++ / midpoint / epsilon prediction only")
        super().__init__(*args, **kw)
        self.config["algorithm_type"] = algorithm_type

    def convert_model_output(self, model_output, sample):  # :446-453 (dpmsolver++ and sde-dpmsolver++, epsilon)
        alpha_t, sigma_t = self._sigma_to_alpha_sigma_t(self.sigmas[self._step_index])
        return (sample - sigma_t * model_output) / alpha_t

    def first_order_update(self, m0, sample):  # :561-567
        (alpha_t, sigma_t, lam_t), (alpha_s, sigma_s, lam_s) = self._lambdas(self._step_index + 1, self._step_index)
        h = lam_t - lam_s
        return ((sigma_t / sigma_s * exp_f32(-h)) * sample + (alpha_t * (1 - exp_f32(-2.0 * h))) * m0
                + sigma_t * pow_half(1.0 - exp_f32(-2 * h)) * self._noise)

    def second_order_update(self, outs, sample):  # :666-674
        (alpha_t, sigma_t, lam_t), (alpha_s0, sigma_s0, lam_s0), (_, _, lam_s1) = self._lambdas(
            self._step_index + 1, self._step_index, self._step_index - 1)
        m0, m1 = outs[-1], outs[-2]
        h, h_0 = lam_t - lam_s0, lam_s0 - lam_s1
        r0 = h_0 / h
        D0, D1 = m0, (1.0 / r0) * (m0 - m1)
        return ((sigma_t / sigma_s0 * exp_f32(-h)) * sample + (alpha_t * (1 - exp_f32(-2.0 * h))) * D0
                + 0.5 * (alpha_t * (1 - exp_f32(-2.0 * h))) * D1 + sigma_t * pow_half(1.0 - exp_f32(-2 * h)) * self._noise)

    def step(self, model_output, timestep, sample, noise=None, seed=0):
        if self._step_index is None:
            self._init_step_index(timestep)
        self._noise = _noise_or_philox(noise, seed, self._step_index, sample)
        return super().step(model_output, timestep, sample)

    def step_scalars(self, timestep):
        """(order, sigma_s0, alpha_s0, A, B, halfB, inv_r0, N) of the next step() in the layout of the product's
        DPMSolverMultistepScheduler.sde_step_scalars, each as step() computes it (advances the scheduler like step())."""
        if self._step_index is None:
            self._init_step_index(timestep)
        c, i, n = self.config, self._step_index, len(self.timesteps)
        lower_order_final = (i == n - 1) and (c["euler_at_final"] or (c["lower_order_final"] and n < 15))
        first = c["solver_order"] == 1 or self.lower_order_nums < 1 or lower_order_final
        (alpha_t, sigma_t, lam_t), (alpha_s0, sigma_s0, lam_s0) = self._lambdas(i + 1, i)
        h = lam_t - lam_s0
        inv_r0 = torch.tensor(0.0)
        if not first:
            lam_s1 = self._lambdas(i - 1)[0][2]
            inv_r0 = 1.0 / ((lam_s0 - lam_s1) / h)
        B = alpha_t * (1 - exp_f32(-2.0 * h))
        if self.lower_order_nums < c["solver_order"]:
            self.lower_order_nums += 1
        self._step_index += 1
        return (1 if first else 2, sigma_s0.item(), alpha_s0.item(), (sigma_t / sigma_s0 * exp_f32(-h)).item(), B.item(),
                (0.5 * B).item(), inv_r0.item(), (sigma_t * pow_half(1.0 - exp_f32(-2 * h))).item())
