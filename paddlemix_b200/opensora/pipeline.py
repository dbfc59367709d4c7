"""Open-Sora 1.1 text-to-video sampling (ppdiffusers/examples/Open-Sora/scripts/inference.py:62-159 with IDDPM.sample,
schedulers/iddpm/__init__.py:66-114): STDiT2 under null-caption classifier-free guidance, the IDDPM learned-variance
step and the per-frame VAE decode. Prompt embeddings (T5) come from the caller, as in the SD / SD3 pipelines.

Per step: one transformer call on the [2B] model input (conditional rows first, as the reference orders them) and one
b200mix_iddpm_step, which writes the new state into both halves of that input. The reference's 2B-row state only ever
feeds back its first half (forward_with_cfg uses x[: len(x) // 2]) and returns the first half, so B rows give the same
result.
"""
from typing import Optional

import torch

from ..sampling import seed_from
from .iddpm import IDDPM

bf16 = torch.bfloat16
IMG_FPS = 120  # inference.py:90-91 (utils/config_utils.py): the fps a single frame is conditioned on


class OpenSoraPipeline:
    def __init__(self, transformer, scheduler: IDDPM, vae=None):
        """transformer: STDiT2, or any callable with its forward signature; vae: a VideoAutoencoderKL for
        output_type="pt"."""
        self.transformer, self.scheduler, self.vae = transformer, scheduler, vae

    def __call__(self, prompt_embeds: torch.Tensor, prompt_attention_mask: Optional[torch.Tensor] = None,
                 negative_prompt_embeds: Optional[torch.Tensor] = None, num_frames: int = 16, height: int = 512,
                 width: int = 512, fps: int = 24, latents: Optional[torch.Tensor] = None,
                 generator: Optional[torch.Generator] = None, output_type: str = "latent", callback_on_step_end=None):
        """prompt_embeds [B, 1, L, caption]; prompt_attention_mask [B, L] (valid tokens first) or None;
        negative_prompt_embeds [B, 1, L, caption], by default the transformer's null caption. Returns the latents
        fp32 [B, 4, num_frames, height/8, width/8], or for output_type="pt" the decoded video fp32
        [B, 3, num_frames, height, width] in nominal range [-1, 1] (not clamped)."""
        if output_type not in ("latent", "pt"):
            raise ValueError(f"output_type must be 'latent' or 'pt', got {output_type!r}")
        if output_type == "pt" and self.vae is None:
            raise ValueError("output_type='pt' needs a vae (VideoAutoencoderKL)")
        if prompt_embeds.ndim != 4 or prompt_embeds.shape[1] != 1:
            raise ValueError(f"prompt_embeds must be [B, 1, L, caption], got {tuple(prompt_embeds.shape)}")
        B, _, L, _ = prompt_embeds.shape
        if negative_prompt_embeds is None:
            null = getattr(self.transformer, "null_caption", None)
            negative_prompt_embeds = null(B) if null is not None else None
            if negative_prompt_embeds is None:
                raise ValueError("negative_prompt_embeds is required: the transformer holds no null caption "
                                 "(y_embedder.y_embedding was not in its weights)")
        if tuple(negative_prompt_embeds.shape) != tuple(prompt_embeds.shape):
            raise ValueError(f"negative_prompt_embeds {tuple(negative_prompt_embeds.shape)} must match prompt_embeds "
                             f"{tuple(prompt_embeds.shape)}: the caption length L must equal the null caption's")
        if prompt_attention_mask is not None and tuple(prompt_attention_mask.shape) != (B, L):
            raise ValueError(f"prompt_attention_mask must be [{B}, {L}], got {tuple(prompt_attention_mask.shape)}")
        if num_frames < 1 or height <= 0 or width <= 0 or height % 16 or width % 16:
            raise ValueError(f"height and width must be positive multiples of 16 (8x VAE, 2x2 patches) and num_frames "
                             f">= 1, got {num_frames} x {height} x {width}")
        if num_frames == 1:
            fps = IMG_FPS
        cfg = getattr(self.transformer, "config", None)
        C = getattr(cfg, "in_channels", 4)
        shape = (B, C, num_frames, height // 8, width // 8)
        dev = getattr(self.transformer, "device", None) or torch.device("cuda")
        if latents is None:
            g = generator or torch.Generator().manual_seed(0)
            latents = torch.randn(shape, generator=g)
        elif tuple(latents.shape) != shape:
            raise ValueError(f"latents must be {shape}, got {tuple(latents.shape)}")
        seed = seed_from(generator)
        # the [2B] model input; the step writes the state into both halves
        buf = torch.empty((2 * B, *shape[1:]), device=dev, dtype=torch.float32)
        buf[:B] = latents
        buf[B:] = latents
        x, x_dup = buf[:B], buf[B:]
        y = torch.cat([prompt_embeds.to(dev, bf16), negative_prompt_embeds.to(dev, bf16)], 0)
        mask = None if prompt_attention_mask is None else prompt_attention_mask.to(dev)
        sizes = dict(num_frames=float(num_frames), height=float(height), width=float(width), ar=height / width, fps=float(fps))
        sizes = {k: torch.full((2 * B,), v, device=dev, dtype=torch.float32) for k, v in sizes.items()}
        ts = torch.tensor(self.scheduler.timestep_map, device=dev, dtype=torch.float32)
        for i in self.scheduler.indices():
            t = ts[i:i + 1].expand(2 * B)
            out = self.transformer(buf, t, y, mask, **sizes)
            self.scheduler.step(out, i, x, seed=seed, out=x, out_dup=x_dup)
            if callback_on_step_end is not None:
                callback_on_step_end(self, i, t, {"latents": x})
        return x if output_type == "latent" else self.vae.decode(x)
