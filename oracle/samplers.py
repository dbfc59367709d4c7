"""ORACLE (test infrastructure, not product code): CPU fp32 restatements of the two stochastic / multistep samplers of
the SD pipelines, EulerAncestralDiscreteScheduler (ppdiffusers/schedulers/scheduling_euler_ancestral_discrete.py:130-389)
and UniPCMultistepScheduler (ppdiffusers/schedulers/scheduling_unipc_multistep.py:138-843, predict_x0 = True, no
thresholding / solver_p), with torch fp32 0-d tensors standing in for paddle's (the helpers of oracle.schedulers).

Element-wise, each update runs in the order of its device kernel, which is the reference's order with the einsum over
the history terms written as an ascending sum, so a device step can be compared bit for bit. The ancestral noise is
injected: oracle.iddpm.philox_normal(seed, step, n) is the device's stream.

Pinned: UniPC by every deterministic full-loop golden of ppdiffusers/tests/schedulers/test_scheduler_unipc.py
(tests/golden/unipc_goldens.json). Euler a: its zero-noise step is the pinned EulerDiscreteScheduler step taken to
sigma_down; the reference's own goldens depend on Paddle's RNG and are not transcribed.
"""
import numpy as np
import torch

from .schedulers import DPMSolverMultistepScheduler, EulerDiscreteScheduler, log_f32, pow_half


def expm1_f32(t):
    """fp32 expm1 with numpy's float32 kernel (the definition the product's host scheduler shares)."""
    a = np.expm1(np.asarray(t.detach().numpy(), dtype=np.float32), dtype=np.float32)
    return torch.from_numpy(np.ascontiguousarray(a).reshape(-1)).reshape(t.shape)


def solve_f32(A, b):
    """paddle.linalg.solve on fp32 tensors, as numpy's fp32 LAPACK solve."""
    return torch.from_numpy(np.linalg.solve(A.numpy(), b.numpy()).astype(np.float32))


class EulerAncestralDiscreteScheduler(EulerDiscreteScheduler):
    """scheduling_euler_ancestral_discrete.py: __init__ :130-169 and set_timesteps :210-250 are EulerDiscrete's
    (linear interpolation, no Karras), step :268-363 with the noise passed in."""

    def __init__(self, num_train_timesteps=1000, beta_start=0.0001, beta_end=0.02, beta_schedule="linear",
                 prediction_type="epsilon", timestep_spacing="linspace", steps_offset=0):
        super().__init__(num_train_timesteps, beta_start, beta_end, beta_schedule, prediction_type=prediction_type,
                         timestep_spacing=timestep_spacing, steps_offset=steps_offset)

    def sigmas_up_down(self):  # :339-342 for the next step() call
        sigma_from, sigma_to = self.sigmas[self._step_index], self.sigmas[self._step_index + 1]
        sigma_up = pow_half(sigma_to ** 2 * (sigma_from ** 2 - sigma_to ** 2) / sigma_from ** 2)
        sigma_down = pow_half(sigma_to ** 2 - sigma_up ** 2)
        return sigma_up, sigma_down

    def step(self, model_output, timestep, sample, noise):  # :268-363
        if self._step_index is None:
            self._init_step_index(timestep)
        sigma = self.sigmas[self._step_index]
        pt = self.config["prediction_type"]
        if pt == "epsilon":
            pred_original_sample = sample - sigma * model_output
        elif pt == "v_prediction":
            pred_original_sample = model_output * (-sigma / pow_half(sigma ** 2 + 1)) + (sample / (sigma ** 2 + 1))
        else:
            raise NotImplementedError(f"prediction_type {pt}")
        sigma_up, sigma_down = self.sigmas_up_down()
        derivative = (sample - pred_original_sample) / sigma
        dt = sigma_down - sigma
        prev_sample = sample + derivative * dt
        prev_sample = prev_sample + noise * sigma_up
        self._step_index += 1
        return prev_sample

    def step_scalars(self):
        """(sigma, c_out, s2p1, dt, sigma_up) of the NEXT step() call, each as step() computes it."""
        sigma = self.sigmas[self._step_index]
        sigma_up, sigma_down = self.sigmas_up_down()
        return (sigma.item(), (-sigma / pow_half(sigma ** 2 + 1)).item(), (sigma ** 2 + 1).item(),
                (sigma_down - sigma).item(), sigma_up.item())


class UniPCMultistepScheduler:
    """scheduling_unipc_multistep.py: __init__ :138-201, set_timesteps :210-271 (DPM-Solver's schedule without
    lambda_min_clipped / Lu lambdas, so oracle.schedulers.DPMSolverMultistepScheduler builds it), convert_model_output
    :368-437, UniP :438-565, UniC :567-701, _init_step_index :703-718, step :720-804, add_noise :821-843."""
    order = 1
    init_noise_sigma = 1.0

    def __init__(self, num_train_timesteps=1000, beta_start=0.0001, beta_end=0.02, beta_schedule="linear", solver_order=2,
                 prediction_type="epsilon", solver_type="bh2", lower_order_final=True, disable_corrector=(),
                 use_karras_sigmas=False, timestep_spacing="linspace", steps_offset=0):
        if solver_type not in ("bh1", "bh2"):
            raise NotImplementedError(solver_type)
        self._sched = DPMSolverMultistepScheduler(num_train_timesteps, beta_start, beta_end, beta_schedule,
                                                  use_karras_sigmas=use_karras_sigmas, timestep_spacing=timestep_spacing,
                                                  steps_offset=steps_offset)
        self.alphas_cumprod = self._sched.alphas_cumprod
        self.solver_order, self.prediction_type, self.solver_type = solver_order, prediction_type, solver_type
        self.lower_order_final, self.disable_corrector = lower_order_final, list(disable_corrector)
        self.num_inference_steps = None

    def set_timesteps(self, num_inference_steps):
        self._sched.set_timesteps(num_inference_steps)
        self.timesteps, self.sigmas = self._sched.timesteps, self._sched.sigmas
        self.num_inference_steps = len(self.timesteps)
        self.model_outputs = [None] * self.solver_order
        self.lower_order_nums = 0
        self.this_order = None
        self.last_sample = None
        self._step_index = None

    _a_s = staticmethod(DPMSolverMultistepScheduler._sigma_to_alpha_sigma_t)

    def _lambda(self, i):
        alpha, sigma = self._a_s(self.sigmas[i])
        return log_f32(alpha) - log_f32(sigma)

    def _init_step_index(self, timestep):
        cand = (self.timesteps == timestep).nonzero()
        if len(cand) == 0:
            self._step_index = len(self.timesteps) - 1
        else:
            self._step_index = (cand[1] if len(cand) > 1 else cand[0]).item()

    def _bh(self, i_t, i_s0, hist, order, corrector):
        """The 0-d tensors of one B(h) update from sigma index i_s0 to i_t with history sigma indices `hist`:
        (sigma_t/sigma_s0, alpha_t*h_phi_1, alpha_t*B_h, rks, rhos)."""
        alpha_t, sigma_t = self._a_s(self.sigmas[i_t])
        _, sigma_s0 = self._a_s(self.sigmas[i_s0])
        lambda_s0 = self._lambda(i_s0)
        h = self._lambda(i_t) - lambda_s0
        rks = [(self._lambda(si) - lambda_s0) / h for si in hist]
        r = torch.stack(rks + [torch.tensor(1.0)])
        hh = -h
        h_phi_1 = expm1_f32(hh)
        h_phi_k = h_phi_1 / hh - 1
        factorial_i = 1
        B_h = hh if self.solver_type == "bh1" else expm1_f32(hh)
        R, b = [], []
        for i in range(1, order + 1):
            R.append(torch.pow(r, i - 1))
            b.append(h_phi_k * factorial_i / B_h)
            factorial_i *= i + 1
            h_phi_k = h_phi_k / hh - 1 / factorial_i
        R, b = torch.stack(R), torch.stack(b)
        if corrector:
            rhos = torch.tensor([0.5]) if order == 1 else solve_f32(R, b)
        else:
            rhos = torch.zeros(0) if order == 1 else torch.tensor([0.5]) if order == 2 else solve_f32(R[:-1, :-1], b[:-1])
        return sigma_t / sigma_s0, alpha_t * h_phi_1, alpha_t * B_h, rks, rhos

    def _advance(self, timestep):
        """The plan of the next step (the reference's control flow in step :747-799), advancing the counters."""
        if self._step_index is None:
            self._init_step_index(timestep)
        i, n = self._step_index, len(self.timesteps)
        p = dict(i=i, corrector=i > 0 and (i - 1) not in self.disable_corrector and self.this_order is not None,
                 order_c=self.this_order)
        if p["corrector"]:
            p["c"] = self._bh(i, i - 1, [i - 1 - k for k in range(1, self.this_order)], self.this_order, True)
        order = min(self.solver_order, n - i) if self.lower_order_final else self.solver_order
        self.this_order = min(order, self.lower_order_nums + 1)
        p["order_p"] = self.this_order
        p["p"] = self._bh(i + 1, i, [i - k for k in range(1, self.this_order)], self.this_order, False)
        if self.lower_order_nums < self.solver_order:
            self.lower_order_nums += 1
        self._step_index += 1
        return p

    def convert_model_output(self, model_output, sample, i):
        alpha_t, sigma_t = self._a_s(self.sigmas[i])
        if self.prediction_type == "epsilon":
            return (sample - sigma_t * model_output) / alpha_t
        if self.prediction_type == "sample":
            return model_output
        if self.prediction_type == "v_prediction":
            return alpha_t * sample - sigma_t * model_output
        raise ValueError(self.prediction_type)

    @staticmethod
    def _history_sum(rhos, rks, hist, base):
        """einsum("k,bkc...->bc...", rhos, D1s) with D1s[k] = (hist[k] - base)/rks[k], summed in ascending k."""
        acc = None
        for k, m in enumerate(hist):
            t = rhos[k] * ((m - base) / rks[k])
            acc = t if acc is None else acc + t
        return acc

    def step(self, model_output, timestep, sample):
        p = self._advance(timestep)
        m0 = self.convert_model_output(model_output, sample, p["i"])
        if p["corrector"]:  # UniC :567-701
            A, K, E, rks, rhos = p["c"]
            mp = self.model_outputs[-1]
            x_t_ = A * self.last_sample - K * mp
            res = rhos[-1] * (m0 - mp)
            corr = self._history_sum(rhos, rks, self.model_outputs[::-1][1:p["order_c"]], mp)
            if corr is not None:
                res = corr + res
            sample = x_t_ - E * res
        self.model_outputs = self.model_outputs[1:] + [m0]
        self.last_sample = sample
        A, K, E, rks, rhos = p["p"]  # UniP :438-565
        x_t = A * sample - K * m0
        pred = self._history_sum(rhos, rks, self.model_outputs[::-1][1:p["order_p"]], m0)
        return x_t if pred is None else x_t - E * pred

    def step_scalars(self, timestep):
        """The scalars of the next step() as floats, in the layout of the product's UniPCMultistepScheduler.step_scalars
        (advances the scheduler like step())."""
        p = self._advance(timestep)
        alpha_t, sigma_t = self._a_s(self.sigmas[p["i"]])
        c = dict(alpha_t=alpha_t.item(), sigma_t=sigma_t.item(), corrector=p["corrector"],
                 order_c=p["order_c"] if p["corrector"] else 0, order_p=p["order_p"])
        if p["corrector"]:
            A, K, E, rks, rhos = p["c"]
            c.update(A_c=A.item(), K_c=K.item(), E_c=E.item(), rc=rhos[:-1].tolist(), rk_c=[r.item() for r in rks],
                     rc_last=rhos[-1].item())
        A, K, E, rks, rhos = p["p"]
        c.update(A_p=A.item(), K_p=K.item(), E_p=E.item(), rp=rhos.tolist(), rk_p=[r.item() for r in rks])
        return c

    def add_noise(self, original_samples, noise, timesteps):
        return self._sched.add_noise(original_samples, noise, timesteps)
