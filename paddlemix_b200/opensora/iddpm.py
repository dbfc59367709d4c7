"""IDDPM sampler of Open-Sora (ppdiffusers/examples/Open-Sora/schedulers/iddpm: __init__.py:23-114, respace.py:33-105,
gaussian_diffusion.py:96-224) for the text-to-video loop: linear betas, learned-range variance, epsilon prediction,
clip_denoised = False, respaced from `diffusion_steps` to `num_sampling_steps`.

The tables are fp64 numpy arrays computed in the reference's operation order. step_scalars(i) rounds them to fp32 the
way _extract_into_tensor (gaussian_diffusion.py:937-950) does, and step() hands them to b200mix_iddpm_step, which does
the CFG combine, the variance interpolation, x0, the posterior mean and the noise in one launch. The Paddle port casts
the respaced betas to fp32 before building the tables (respace.py:103); here they stay fp64, as in improved-diffusion
and DiT, from which it was ported.
"""
from typing import Iterable, List, Optional, Sequence, Set, Tuple, Union

import numpy as np


def space_timesteps(num_timesteps: int, section_counts: Union[str, Sequence[int]]) -> Set[int]:
    """respace.py:33-79: the kept steps of `num_timesteps`, `section_counts` steps from each of equal-sized sections
    ("100", "10,15,20" or a list), or the DDIM striding for "ddimN". Python's round (half to even) as written."""
    if isinstance(section_counts, str):
        if section_counts.startswith("ddim"):
            desired = int(section_counts[len("ddim"):])
            for i in range(1, num_timesteps):
                if len(range(0, num_timesteps, i)) == desired:
                    return set(range(0, num_timesteps, i))
            raise ValueError(f"cannot create exactly {desired} steps with an integer stride")
        section_counts = [int(x) for x in section_counts.split(",")]
    size_per, extra = divmod(num_timesteps, len(section_counts))
    start, steps = 0, []
    for i, count in enumerate(section_counts):
        size = size_per + (1 if i < extra else 0)
        if size < count:
            raise ValueError(f"cannot divide section of {size} steps into {count}")
        stride = 1 if count <= 1 else (size - 1) / (count - 1)
        cur = 0.0
        for _ in range(count):
            steps.append(start + round(cur))
            cur += stride
        start += size
    return set(steps)


def linear_betas(diffusion_steps: int) -> np.ndarray:
    """get_named_beta_schedule("linear") (gaussian_diffusion.py:147-164): linspace(1e-4 s, 0.02 s, n) in fp64 with
    s = 1000 / n, evaluated as Paddle's linspace does (start + step i for the first half, stop - step (n-1-i) after)."""
    scale = 1000 / diffusion_steps
    start, stop, n = scale * 0.0001, scale * 0.02, diffusion_steps
    if n == 1:
        return np.array([start])
    step = (stop - start) / (n - 1)
    i = np.arange(n, dtype=np.float64)
    return np.where(i < n // 2, start + step * i, stop - step * (n - 1 - i))


class IDDPM:
    """IDDPM(num_sampling_steps, timestep_respacing, ..., cfg_scale, cfg_channel) as the reference constructs it. Only
    what Open-Sora's sampling uses is supported; the other model types raise NotImplementedError."""

    def __init__(self, num_sampling_steps: Optional[int] = None, timestep_respacing=None, noise_schedule: str = "linear",
                 use_kl: bool = False, sigma_small: bool = False, predict_xstart: bool = False, learn_sigma: bool = True,
                 rescale_learned_sigmas: bool = False, diffusion_steps: int = 1000, cfg_scale: float = 4.0,
                 cfg_channel: Optional[int] = None):
        if noise_schedule != "linear":
            raise NotImplementedError(f"IDDPM(b200): noise_schedule={noise_schedule!r} (only 'linear')")
        for name, val in (("use_kl", use_kl), ("sigma_small", sigma_small), ("predict_xstart", predict_xstart),
                          ("learn_sigma", not learn_sigma), ("rescale_learned_sigmas", rescale_learned_sigmas)):
            if val:
                raise NotImplementedError(f"IDDPM(b200): {name} is not supported (learned-range epsilon model only)")
        if num_sampling_steps is not None:
            if timestep_respacing is not None:
                raise ValueError("give num_sampling_steps or timestep_respacing, not both")
            timestep_respacing = str(num_sampling_steps)
        if timestep_respacing is None or timestep_respacing == "":
            timestep_respacing = [diffusion_steps]
        self.cfg_scale, self.cfg_channel = cfg_scale, cfg_channel
        self.diffusion_steps = diffusion_steps
        base = linear_betas(diffusion_steps)
        self.base_alphas_cumprod = np.cumprod(1.0 - base)
        # SpacedDiffusion (respace.py:90-105): betas of the kept steps from the base alphas_cumprod
        keep = space_timesteps(diffusion_steps, timestep_respacing)
        self.timestep_map: List[int] = []
        betas, last = [], 1.0
        for i, ac in enumerate(self.base_alphas_cumprod):
            if i in keep:
                betas.append(1 - ac / last)
                last = ac
                self.timestep_map.append(i)
        self._tables(np.array(betas, dtype=np.float64))

    def _tables(self, betas: np.ndarray):
        """GaussianDiffusion.__init__ (gaussian_diffusion.py:178-224), fp64."""
        self.betas = betas
        self.num_timesteps = len(betas)
        alphas = 1.0 - betas
        self.alphas_cumprod = np.cumprod(alphas)
        self.alphas_cumprod_prev = np.concatenate([[1.0], self.alphas_cumprod[:-1]])
        self.sqrt_recip_alphas_cumprod = np.sqrt(1.0 / self.alphas_cumprod)
        self.sqrt_recipm1_alphas_cumprod = np.sqrt(1.0 / self.alphas_cumprod - 1)
        self.posterior_variance = betas * (1.0 - self.alphas_cumprod_prev) / (1.0 - self.alphas_cumprod)
        self.posterior_log_variance_clipped = (
            np.log(np.concatenate([self.posterior_variance[1:2], self.posterior_variance[1:]]))
            if self.num_timesteps > 1 else np.array([], dtype=np.float64))
        self.posterior_mean_coef1 = betas * np.sqrt(self.alphas_cumprod_prev) / (1.0 - self.alphas_cumprod)
        self.posterior_mean_coef2 = (1.0 - self.alphas_cumprod_prev) * np.sqrt(alphas) / (1.0 - self.alphas_cumprod)
        self.log_betas = np.log(betas)

    def step_scalars(self, i: int) -> Tuple[float, float, float, float, float, float]:
        """(sqrt_recip_ac, sqrt_recipm1_ac, coef1, coef2, max_log = log(beta), min_log) at respaced index i, each
        rounded to fp32 as _extract_into_tensor does."""
        return tuple(float(np.float32(t[i])) for t in (
            self.sqrt_recip_alphas_cumprod, self.sqrt_recipm1_alphas_cumprod, self.posterior_mean_coef1,
            self.posterior_mean_coef2, self.log_betas, self.posterior_log_variance_clipped))

    def indices(self) -> Iterable[int]:
        """The respaced indices in sampling order (p_sample_loop_progressive: num_timesteps - 1 down to 0)."""
        return range(self.num_timesteps - 1, -1, -1)

    def step(self, model_output, i: int, x, seed: int = 0, out=None, out_dup=None, noise=None):
        """p_sample at respaced index i on the [2B, 2C, ...] output of forward_with_cfg's model call; x fp32 [B, C, ...].
        Noise is `noise` when given, else Philox keyed by (seed, i); none is added at i = 0. out may be x."""
        from .. import ops
        C = x.shape[1]
        cfg_channel = C if self.cfg_channel is None else self.cfg_channel
        return ops.iddpm_step(model_output, x, self.cfg_scale, cfg_channel, self.step_scalars(i), add_noise=i != 0,
                              seed=seed, step=i, noise=noise, out=out, out_dup=out_dup)
