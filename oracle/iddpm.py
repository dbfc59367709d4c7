"""ORACLE (test infrastructure, not product code): CPU restatement of Open-Sora's IDDPM sampling,
ppdiffusers/examples/Open-Sora/schedulers/iddpm (IDDPM.sample and forward_with_cfg __init__.py:66-114, space_timesteps
and SpacedDiffusion respace.py:33-140, the tables gaussian_diffusion.py:178-224, p_mean_variance :278-365, p_sample
:409-485, _extract_into_tensor :937-950), in torch: fp64 tables, fp32 arithmetic after the per-step fp32 cast, one
rounding per operation in the reference's order. Pinned where the reference leaves it open:
  - the respaced betas stay fp64 (the Paddle port rounds them to fp32 first, respace.py:103);
  - exp(0.5 * log_variance) is the fp64 exp rounded to fp32;
  - paddle.randn is replaced by injectable noise, or by philox_normal(): the transform of b200mix_iddpm_step.
sample_2b() keeps the reference's 2B-row form (the state is duplicated, both halves are updated, the first half is
returned); sample_b() carries B rows only.

PARITY UNPINNED: the reference has no IDDPM test and no goldens.
"""
import math
from typing import Callable, Optional

import numpy as np
import torch

from .generation import philox4x32_10

f32, f64 = torch.float32, torch.float64


def space_timesteps(num_timesteps, section_counts):
    """respace.py:33-79."""
    if isinstance(section_counts, str):
        if section_counts.startswith("ddim"):
            desired_count = int(section_counts[len("ddim"):])
            for i in range(1, num_timesteps):
                if len(range(0, num_timesteps, i)) == desired_count:
                    return set(range(0, num_timesteps, i))
            raise ValueError(f"cannot create exactly {num_timesteps} steps with an integer stride")
        section_counts = [int(x) for x in section_counts.split(",")]
    size_per = num_timesteps // len(section_counts)
    extra = num_timesteps % len(section_counts)
    start_idx = 0
    all_steps = []
    for i, section_count in enumerate(section_counts):
        size = size_per + (1 if i < extra else 0)
        if size < section_count:
            raise ValueError(f"cannot divide section of {size} steps into {section_count}")
        frac_stride = 1 if section_count <= 1 else (size - 1) / (section_count - 1)
        cur_idx = 0.0
        for _ in range(section_count):
            all_steps.append(start_idx + round(cur_idx))
            cur_idx += frac_stride
        start_idx += size
    return set(all_steps)


def linspace_paddle(start, stop, num):
    """paddle.linspace in fp64: start + step*i below num//2, stop - step*(num-1-i) from there."""
    step = (stop - start) / (num - 1)
    return torch.tensor([start + step * i if i < num // 2 else stop - step * (num - 1 - i) for i in range(num)], dtype=f64)


class Diffusion:
    """GaussianDiffusion.__init__ (:178-224) on the betas of SpacedDiffusion (respace.py:90-105)."""

    def __init__(self, diffusion_steps=1000, respacing="100"):
        scale = 1000 / diffusion_steps
        base = linspace_paddle(scale * 0.0001, scale * 0.02, diffusion_steps)
        self.base_alphas_cumprod = torch.cumprod(1.0 - base, dim=0)
        use = space_timesteps(diffusion_steps, respacing)
        self.timestep_map, new_betas, last = [], [], 1.0
        for i, ac in enumerate(self.base_alphas_cumprod.tolist()):
            if i in use:
                new_betas.append(1 - ac / last)
                last = ac
                self.timestep_map.append(i)
        b = torch.tensor(new_betas, dtype=f64)
        self.betas = b
        self.num_timesteps = len(b)
        alphas = 1.0 - b
        self.alphas_cumprod = torch.cumprod(alphas, dim=0)
        self.alphas_cumprod_prev = torch.cat([torch.tensor([1.0], dtype=f64), self.alphas_cumprod[:-1]])
        self.sqrt_recip_alphas_cumprod = torch.sqrt(1.0 / self.alphas_cumprod)
        self.sqrt_recipm1_alphas_cumprod = torch.sqrt(1.0 / self.alphas_cumprod - 1)
        self.posterior_variance = b * (1.0 - self.alphas_cumprod_prev) / (1.0 - self.alphas_cumprod)
        self.posterior_log_variance_clipped = torch.log(torch.cat([self.posterior_variance[1:2], self.posterior_variance[1:]]))
        self.posterior_mean_coef1 = b * torch.sqrt(self.alphas_cumprod_prev) / (1.0 - self.alphas_cumprod)
        self.posterior_mean_coef2 = (1.0 - self.alphas_cumprod_prev) * torch.sqrt(alphas) / (1.0 - self.alphas_cumprod)
        self.log_betas = torch.log(b)

    def extract(self, arr, i, device=None):
        """_extract_into_tensor: the fp64 table entry rounded to fp32 (a 0-d tensor broadcasts like the reference's)."""
        return arr[i].to(f32).to(device)

    def p_sample(self, model_output, x, i, noise, cfg_channel_out=None):
        """p_mean_variance + p_sample for rows that share respaced index i. model_output [N, 2C, ...] (already the
        forward_with_cfg result), x fp32 [N, C, ...], noise like x."""
        C = x.shape[1]
        dev = x.device
        eps, v = model_output[:, :C].to(f32), model_output[:, C:].to(f32)
        min_log = self.extract(self.posterior_log_variance_clipped, i, dev)
        max_log = self.extract(self.log_betas, i, dev)
        frac = (v + 1) / 2
        log_var = frac * max_log + (1 - frac) * min_log
        x0 = self.extract(self.sqrt_recip_alphas_cumprod, i, dev) * x - self.extract(self.sqrt_recipm1_alphas_cumprod, i, dev) * eps
        mean = self.extract(self.posterior_mean_coef1, i, dev) * x0 + self.extract(self.posterior_mean_coef2, i, dev) * x
        if i == 0:  # nonzero_mask = 0
            return mean
        sd = torch.exp((0.5 * log_var).to(f64)).to(f32)
        return mean + sd * noise


def forward_with_cfg(model, x, t, y, cfg_scale, cfg_channel=None, **kw):
    """__init__.py:97-114: the model sees [half, half]; eps channels [0, cfg_channel) are guided."""
    half = x[: len(x) // 2]
    combined = torch.cat([half, half], 0)
    out = model(combined, t, y, **kw)
    if cfg_channel is None:
        cfg_channel = out.shape[1] // 2
    eps, rest = out[:, :cfg_channel], out[:, cfg_channel:]
    cond_eps, uncond_eps = torch.split(eps, len(eps) // 2, dim=0)
    half_eps = uncond_eps + cfg_scale * (cond_eps - uncond_eps)
    eps = torch.cat([half_eps, half_eps], 0)
    return torch.cat([eps, rest], 1)


def philox_normal(seed: int, step: int, n: int) -> torch.Tensor:
    """The first n normals of b200mix_iddpm_step's Philox stream at (seed, step): group g = elements 4g..4g+3,
    counter (step, g mod 2^32, g div 2^32, 0), key (seed mod 2^32, seed div 2^32), u = (r + 0.5) 2^-32,
    fp64 Box-Muller pairs (u0, u1), (u2, u3), each result rounded to fp32. Returns fp32 [n]."""
    g = np.arange((n + 3) // 4, dtype=np.uint64)
    r = philox4x32_10((np.full_like(g, step), g & np.uint64(0xFFFFFFFF), g >> np.uint64(32), np.zeros_like(g)),
                      (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF))
    u = [(w.astype(np.float64) + 0.5) * 2.0 ** -32 for w in r]
    z = np.empty((len(g), 4), dtype=np.float32)
    for p in range(2):
        rad = np.sqrt(-2.0 * np.log(u[2 * p]))
        ang = 6.283185307179586 * u[2 * p + 1]
        z[:, 2 * p] = (rad * np.cos(ang)).astype(np.float32)
        z[:, 2 * p + 1] = (rad * np.sin(ang)).astype(np.float32)
    return torch.from_numpy(z.reshape(-1)[:n].copy())


def philox_noise_fn(seed: int) -> Callable:
    """noise_fn(i, shape) for the loops below: the kernel's Philox normals for a [B, ...] state."""
    return lambda i, shape: philox_normal(seed, i, math.prod(shape)).reshape(shape)


def sample_2b(diff: Diffusion, model, z, y_cond, y_null, cfg_scale, cfg_channel=None, noise_fn=None, model_kwargs=None):
    """IDDPM.sample (__init__.py:66-94) with p_sample_loop: z [B, C, ...]; y = cat([y_cond, y_null]); the 2B-row state
    is updated whole. noise_fn(i, shape) gives the step's noise for `shape` ([2B, ...] here); returns the first half."""
    kw = dict(model_kwargs or {})
    x = torch.cat([z, z], 0)
    y = torch.cat([y_cond, y_null], 0)
    for i in range(diff.num_timesteps - 1, -1, -1):
        t = torch.full((x.shape[0],), diff.timestep_map[i], dtype=torch.int64, device=x.device)  # _WrappedModel
        out = forward_with_cfg(model, x, t, y, cfg_scale, cfg_channel, **kw)
        x = diff.p_sample(out, x, i, noise_fn(i, tuple(x.shape)))
    return x[: len(x) // 2]


def sample_b(diff: Diffusion, model, z, y_cond, y_null, cfg_scale, cfg_channel=None, noise_fn=None, model_kwargs=None):
    """The same loop on a B-row state: the model still sees [x, x] and cat([y_cond, y_null]); only the conditional rows
    of the combined output are stepped. noise_fn(i, shape) is called with the B-row shape."""
    kw = dict(model_kwargs or {})
    x = z
    y = torch.cat([y_cond, y_null], 0)
    B = x.shape[0]
    for i in range(diff.num_timesteps - 1, -1, -1):
        t = torch.full((2 * B,), diff.timestep_map[i], dtype=torch.int64, device=x.device)
        out = model(torch.cat([x, x], 0), t, y, **kw)
        cc = out.shape[1] // 2 if cfg_channel is None else cfg_channel
        g = out[:B].clone()
        g[:, :cc] = out[B:, :cc] + cfg_scale * (out[:B, :cc] - out[B:, :cc])
        x = diff.p_sample(g, x, i, noise_fn(i, tuple(x.shape)))
    return x
