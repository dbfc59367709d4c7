"""VideoAutoencoderKL.decode (ppdiffusers/examples/Open-Sora/models/vae/vae.py:54-69): the SD VAE applied to every
frame of a [B, 4, T, h, w] latent video, in micro-batches of frames. Encoding is not provided."""
from typing import Optional

import torch

SCALING_FACTOR = 0.18215  # vae.py:58,65 (the constant, not the wrapped VAE's config)


class VideoAutoencoderKL:
    def __init__(self, vae, micro_batch_size: Optional[int] = None):
        """vae: a loaded ppdiffusers.AutoencoderKL (e.g. stabilityai/sd-vae-ft-ema); micro_batch_size None decodes all
        B*T frames in one call."""
        if micro_batch_size is not None and micro_batch_size < 1:
            raise ValueError("micro_batch_size must be None or >= 1")
        self.module, self.micro_batch_size = vae, micro_batch_size
        self.out_channels = vae.config.latent_channels
        self.patch_size = (1, 8, 8)

    def decode(self, z: torch.Tensor) -> torch.Tensor:
        """z [B, C, T, h, w] -> fp32 [B, 3, T, 8h, 8w] in nominal range [-1, 1]: frames (b, t) in order b*T + t,
        each micro-batch divided by 0.18215 and decoded by AutoencoderKL.decode."""
        from .. import ops
        B, C, T, h, w = z.shape
        frames = z.to(self.module.device, torch.float32).permute(0, 2, 1, 3, 4).reshape(B * T, C, h, w).contiguous()
        frames = ops.scale_model_input(frames, SCALING_FACTOR)
        bs = B * T if self.micro_batch_size is None else self.micro_batch_size
        x = torch.cat([self.module.decode(frames[i:i + bs]).sample for i in range(0, B * T, bs)], 0)
        return x.reshape(B, T, *x.shape[1:]).permute(0, 2, 1, 3, 4).contiguous()
