"""The denoising loops of StableDiffusionPipeline / StableDiffusionXLPipeline / StableDiffusion3Pipeline
(ppdiffusers/pipelines/stable_diffusion/pipeline_stable_diffusion.py:858-908,
 ppdiffusers/pipelines/stable_diffusion_xl/pipeline_stable_diffusion_xl.py:1040-1082,
 ppdiffusers/pipelines/stable_diffusion_3/pipeline_stable_diffusion_3.py:794-866) on the H100-native denoisers.

Text encoders and the VAE run before / after the loop and are out of scope (SURVEY.md §8f): the pipelines here take
`prompt_embeds` (and `negative_prompt_embeds`) exactly as the reference pipelines accept them and return latents
(`output_type="latent"`). One timestep = denoiser forward on [uncond | cond] rows + one fused CFG + scheduler kernel.
For the UNet the forward is captured once into a CUDA graph (~1.5 k launches -> one graph launch; the timestep lives
in a device tensor) and replayed; the scheduler kernel, whose fp32 scalars change every step, is launched outside it.

Multi-GPU (data parallel over images, SURVEY.md §8e): each rank takes a contiguous slice of the batch, replicates the
weights, runs the loop with zero per-step communication, and `all_gather`s the finished latents once over NCCL.
"""
from typing import Any, Dict, Optional

import torch

from .schedulers import DDIMScheduler
from .unet_2d_condition import UNet2DConditionModel

bf16 = torch.bfloat16


class GraphedUNet:
    """Static-shape CUDA-graph wrapper around UNet2DConditionModel.forward_nhwc (+ NCHW<->NHWC conversion).
    Inputs are copied into static device buffers; the timestep lives in a device tensor so it can change per replay."""

    def __init__(self, unet: UNet2DConditionModel, sample_shape, ctx_shape, added_cond_shapes: Optional[Dict[str, Any]] = None,
                 warmup: int = 2):
        from .. import ops
        dev = unet.device
        self.unet = unet
        self.sample = torch.zeros(sample_shape, device=dev, dtype=torch.float32)  # NCHW fp32 latents (model input)
        self.ctx = torch.zeros(ctx_shape, device=dev, dtype=bf16)
        self.t = torch.zeros(sample_shape[0], device=dev, dtype=torch.float32)
        self.added = None
        if added_cond_shapes:
            self.added = {k: torch.zeros(s, device=dev, dtype=(bf16 if k == "text_embeds" else torch.float32))
                          for k, s in added_cond_shapes.items()}
        self.out = None
        self.launches_per_replay = 0

        def run():
            x = ops.nchw_to_nhwc(self.sample)
            y = unet.forward_nhwc(x, self.t, self.ctx, self.added)
            return ops.nhwc_to_nchw(y, out_dtype=bf16)

        s = torch.cuda.Stream(device=dev)
        s.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(s):
            for _ in range(warmup):
                run()
        torch.cuda.current_stream(dev).wait_stream(s)
        torch.cuda.synchronize(dev)
        self.graph = torch.cuda.CUDAGraph()
        n0 = ops.launches()
        with torch.cuda.graph(self.graph):
            self.out = run()
        self.launches_per_replay = ops.launches() - n0

    def __call__(self, sample, timestep, ctx=None, added_cond_kwargs=None):
        from .. import ops
        self.sample.copy_(sample, non_blocking=True)
        if ctx is not None:
            self.ctx.copy_(ctx, non_blocking=True)
        if torch.is_tensor(timestep):
            self.t.copy_(timestep.to(torch.float32).reshape(-1).expand(self.t.shape[0]), non_blocking=True)
        else:
            self.t.fill_(float(timestep))
        if added_cond_kwargs is not None and self.added is not None:
            for k, v in added_cond_kwargs.items():
                self.added[k].copy_(v, non_blocking=True)
        self.graph.replay()
        ops._count(self.launches_per_replay)
        return self.out


class StableDiffusionPipeline:
    """Loop-only mirror of ppdiffusers.StableDiffusionPipeline / StableDiffusionXLPipeline.__call__."""

    def __init__(self, unet: UNet2DConditionModel, scheduler: DDIMScheduler, use_cuda_graph: bool = True, vae=None):
        self.unet, self.scheduler, self.use_cuda_graph, self.vae = unet, scheduler, use_cuda_graph, vae
        self._graphed = {}

    def decode_latents(self, latents):
        """pipeline_stable_diffusion.py:910-917 + VaeImageProcessor.postprocess(output_type="pt"): image =
        vae.decode(latents / scaling_factor).sample, denormalised to [0, 1]. Returns fp32 [B, 3, H, W] on the device."""
        from .. import ops
        if self.vae is None:
            raise ValueError("output_type='pt' needs a VAE: StableDiffusionPipeline(unet, scheduler, vae=AutoencoderKL(...))")
        z = ops.scale_model_input(latents.contiguous(), float(self.vae.config.scaling_factor))  # IEEE fp32 division
        image = self.vae.decode(z, return_dict=False)[0]
        return (image / 2 + 0.5).clamp(0, 1)  # image_processor.py denormalize: host-side post-processing of the result

    def _denoiser(self, sample_shape, ctx_shape, added):
        if not self.use_cuda_graph:
            return None
        key = (tuple(sample_shape), tuple(ctx_shape), None if added is None else tuple((k, tuple(v.shape)) for k, v in added.items()))
        g = self._graphed.get(key)
        if g is None:
            g = GraphedUNet(self.unet, sample_shape, ctx_shape, None if added is None else {k: v.shape for k, v in added.items()})
            self._graphed[key] = g
        return g

    @torch.no_grad()
    def __call__(self, prompt=None, height: Optional[int] = None, width: Optional[int] = None,
                 num_inference_steps: int = 50, guidance_scale: float = 7.5, negative_prompt=None, eta: float = 0.0,
                 latents: Optional[torch.Tensor] = None, prompt_embeds: Optional[torch.Tensor] = None,
                 negative_prompt_embeds: Optional[torch.Tensor] = None, output_type: str = "latent",
                 added_cond_kwargs: Optional[Dict[str, torch.Tensor]] = None,
                 negative_added_cond_kwargs: Optional[Dict[str, torch.Tensor]] = None, callback_on_step_end=None,
                 generator: Optional[torch.Generator] = None, guidance_rescale: float = 0.0):
        if prompt is not None or negative_prompt is not None:
            raise NotImplementedError("text encoders are outside the hot path: pass prompt_embeds / negative_prompt_embeds")
        if prompt_embeds is None:
            raise ValueError("Provide either `prompt` or `prompt_embeds`. Cannot leave both `prompt` and `prompt_embeds` undefined.")
        if output_type not in ("latent", "pt"):
            raise NotImplementedError("output_type must be 'latent' or 'pt' (PIL / numpy conversion is the caller's)")
        if eta != 0.0:
            raise NotImplementedError("eta > 0 (stochastic DDIM) is outside the hot path")
        from .. import ops
        dev = self.unet.device
        B = prompt_embeds.shape[0]
        do_cfg = guidance_scale > 1.0  # pipeline_stable_diffusion.py:781
        if do_cfg and negative_prompt_embeds is None:
            negative_prompt_embeds = torch.zeros_like(prompt_embeds)
        if latents is None:
            if height is None or width is None:
                raise ValueError("height/width (or latents) are required")
            g = generator or torch.Generator().manual_seed(0)
            latents = torch.randn(B, self.unet.config.in_channels, height // 8, width // 8, generator=g)
        # timesteps first (pipeline_stable_diffusion.py:808-811), then prepare_latents scales the initial noise by the
        # scheduler's init_noise_sigma (:813-824, :583): for EulerDiscrete that value depends on the chosen timesteps
        self.scheduler.set_timesteps(num_inference_steps)
        latents = latents.to(device=dev, dtype=torch.float32).contiguous() * self.scheduler.init_noise_sigma
        ctx = prompt_embeds.to(device=dev, dtype=bf16)
        added = None
        if added_cond_kwargs is not None:
            added = {k: v.to(dev) for k, v in added_cond_kwargs.items()}
        if do_cfg:
            ctx = torch.cat([negative_prompt_embeds.to(device=dev, dtype=bf16), ctx], 0)
            if added is not None:
                neg = negative_added_cond_kwargs or added_cond_kwargs
                added = {k: torch.cat([neg[k].to(dev), added[k]], 0) for k in added}
        ctx = ctx.contiguous()
        if added is not None:
            added = {k: (v.to(bf16) if k == "text_embeds" else v.to(torch.float32)).contiguous() for k, v in added.items()}
        rows = 2 * B if do_cfg else B
        sample_shape = (rows,) + tuple(latents.shape[1:])
        den = self._denoiser(sample_shape, ctx.shape, added)
        model_in = torch.empty(sample_shape, device=dev, dtype=torch.float32)
        nxt = torch.empty_like(latents)
        first = True
        for i, t in enumerate(self.scheduler.timesteps):
            # latent_model_input = scheduler.scale_model_input(concat([latents] * 2) if CFG) (:860-861): the identity for
            # DDIM, x / sqrt(sigma^2 + 1) for EulerDiscrete
            scaled = self.scheduler.scale_model_input(latents, t)
            if do_cfg:
                model_in[:B].copy_(scaled)
                model_in[B:].copy_(scaled)
            else:
                model_in = scaled
            if den is not None:
                eps = den(model_in, float(t), ctx if first else None, added if first else None)
            else:
                eps = self.unet.forward(model_in, float(t), ctx, added_cond_kwargs=added, return_dict=False)[0]
            first = False
            if do_cfg and guidance_rescale > 0.0:
                # rescale_noise_cfg (pipeline_stable_diffusion.py:69-80, :886-888; SDXL :1061-1067): the guided
                # prediction is rescaled to the text branch's per-sample std before the scheduler step
                guided = ops.cfg_combine(eps[:B], eps[B:], guidance_scale, guidance_rescale)
                self.scheduler.step(guided, t, latents, out=nxt)
            elif do_cfg:  # noise_pred_uncond + g*(noise_pred_text - noise_pred_uncond) (:882-884), fused with the step
                self.scheduler.step(eps[:B], t, latents, model_output_cond=eps[B:], guidance_scale=guidance_scale, out=nxt)
            else:
                self.scheduler.step(eps, t, latents, out=nxt)
            latents, nxt = nxt, latents
            if callback_on_step_end is not None:
                callback_on_step_end(self, i, t, {"latents": latents})
        return latents if output_type == "latent" else self.decode_latents(latents)


class StableDiffusion3Pipeline:
    """Loop-only mirror of ppdiffusers.StableDiffusion3Pipeline.__call__ (pipeline_stable_diffusion_3.py:794-866):
    FlowMatchEuler timesteps, SD3Transformer2DModel on [uncond | cond] rows, CFG combine fused with the Euler step.
    The reference's INFERENCE_OPTIMIZE_BP mode (:803-839) splits the CFG pair over 2 GPUs with 4 scatters + 1
    all_gather PER STEP; here images (with their CFG pair) are sharded once and only the finished latents are gathered
    (`shard_batch` / `all_gather_latents`)."""

    def __init__(self, transformer, scheduler):
        self.transformer, self.scheduler = transformer, scheduler

    @torch.no_grad()
    def __call__(self, prompt=None, height: Optional[int] = None, width: Optional[int] = None,
                 num_inference_steps: int = 28, guidance_scale: float = 7.0, latents: Optional[torch.Tensor] = None,
                 prompt_embeds: Optional[torch.Tensor] = None, negative_prompt_embeds: Optional[torch.Tensor] = None,
                 pooled_prompt_embeds: Optional[torch.Tensor] = None,
                 negative_pooled_prompt_embeds: Optional[torch.Tensor] = None, output_type: str = "latent",
                 callback_on_step_end=None, generator: Optional[torch.Generator] = None):
        if prompt is not None:
            raise NotImplementedError("text encoders are outside the hot path: pass prompt_embeds / pooled_prompt_embeds")
        if prompt_embeds is None or pooled_prompt_embeds is None:
            raise ValueError("If `prompt_embeds` are provided, `pooled_prompt_embeds` also have to be passed.")
        if output_type != "latent":
            raise NotImplementedError("the VAE decoder is outside the hot path: use output_type='latent'")
        tr = self.transformer
        dev = tr.device
        B = prompt_embeds.shape[0]
        do_cfg = guidance_scale > 1  # pipeline_stable_diffusion_3.py:640-642
        if latents is None:
            if height is None or width is None:
                raise ValueError("height/width (or latents) are required")
            g = generator or torch.Generator().manual_seed(0)
            latents = torch.randn(B, tr.config.in_channels, height // 8, width // 8, generator=g)
        latents = latents.to(device=dev, dtype=torch.float32).contiguous()
        ctx, pooled = prompt_embeds.to(device=dev, dtype=bf16), pooled_prompt_embeds.to(device=dev, dtype=bf16)
        if do_cfg:
            if negative_prompt_embeds is None:
                negative_prompt_embeds = torch.zeros_like(prompt_embeds)
            if negative_pooled_prompt_embeds is None:
                negative_pooled_prompt_embeds = torch.zeros_like(pooled_prompt_embeds)
            ctx = torch.cat([negative_prompt_embeds.to(device=dev, dtype=bf16), ctx], 0)
            pooled = torch.cat([negative_pooled_prompt_embeds.to(device=dev, dtype=bf16), pooled], 0)
        self.scheduler.set_timesteps(num_inference_steps)
        rows = 2 * B if do_cfg else B
        model_in = torch.empty((rows,) + tuple(latents.shape[1:]), device=dev, dtype=torch.float32)
        nxt = torch.empty_like(latents)
        for i, t in enumerate(self.scheduler.timesteps):
            if do_cfg:  # latent_model_input = concat([latents] * 2) (:798)
                model_in[:B].copy_(latents)
                model_in[B:].copy_(latents)
            else:
                model_in = latents
            timestep = torch.full((rows,), float(t), device=dev, dtype=torch.float32)  # t.expand(batch) (:799)
            v = tr(hidden_states=model_in, timestep=timestep, encoder_hidden_states=ctx, pooled_projections=pooled,
                   return_dict=False)[0]
            if do_cfg:  # noise_pred_uncond + s * (noise_pred_text - noise_pred_uncond) (:843-846), fused with the step
                self.scheduler.step(v[:B], t, latents, model_output_cond=v[B:], guidance_scale=guidance_scale, out=nxt)
            else:
                self.scheduler.step(v, t, latents, out=nxt)
            latents, nxt = nxt, latents
            if callback_on_step_end is not None:
                callback_on_step_end(self, i, t, {"latents": latents})
        return latents


def all_gather_latents(latents: torch.Tensor) -> torch.Tensor:
    """The single collective of the data-parallel path: finished latents of every rank -> [world*B_local, ...].
    With a communicator created by paddlemix_b200.distributed.init_comm() the gather is the C-ABI call
    b200mix_allgather_latents (NCCL on libb200mix's own communicator); otherwise torch.distributed's NCCL all_gather."""
    import torch.distributed as dist

    from .. import distributed as bdist
    if not dist.is_available() or not dist.is_initialized() or dist.get_world_size() == 1:
        return latents
    if bdist.comm_ready():
        return bdist.all_gather_latents(latents)
    out = [torch.empty_like(latents) for _ in range(dist.get_world_size())]
    dist.all_gather(out, latents.contiguous())
    return torch.cat(out, 0)


def shard_batch(n: int, rank: int, world: int):
    """Contiguous slice [lo, hi) of an n-image batch owned by `rank`; CFG pairs stay on one rank because the
    uncond/cond rows are built per rank after sharding."""
    per = (n + world - 1) // world
    lo = min(n, rank * per)
    return lo, min(n, lo + per)
