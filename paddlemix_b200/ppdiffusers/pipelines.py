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
from types import SimpleNamespace
from typing import Any, Dict, List, Optional, Union

import torch

from .adapter import MultiAdapter
from .controlnet import MultiControlNetModel, controlnet_keep
from .schedulers import DDIMScheduler
from .unet_2d_condition import UNet2DConditionModel

bf16 = torch.bfloat16


class GraphedUNet:
    """Static-shape CUDA-graph wrapper around UNet2DConditionModel.forward_nhwc (+ NCHW<->NHWC conversion).
    Inputs are copied into static device buffers; the timestep lives in a device tensor so it can change per replay.
    With `controlnet` (a ControlNetModel or MultiControlNetModel) the graph runs the ControlNet(s) and hands their
    residuals to the UNet; the conditioning embeddings and the fp32 scale tables are static buffers too
    (`cond_embeddings` / `scale_tables` of __call__), so new scales need no new capture. `controlnet_rows` < rows:
    the ControlNet runs on the last `controlnet_rows` rows only (guess mode with CFG) and the residuals of the other
    rows stay zero. With `intrablock_residuals` (bf16 NHWC [rows, h, w, c] device buffers) the graph hands them to the
    UNet as down_intrablock_additional_residuals (T2I-Adapter); the caller writes new values into them between replays."""

    def __init__(self, unet: UNet2DConditionModel, sample_shape, ctx_shape, added_cond_shapes: Optional[Dict[str, Any]] = None,
                 warmup: int = 2, controlnet=None, controlnet_rows: Optional[int] = None, intrablock_residuals=None):
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
        self.cn = None
        if controlnet is not None:
            self.cn = controlnet_state(controlnet, sample_shape, controlnet_rows or sample_shape[0], dev)
        self.intra = None if intrablock_residuals is None else list(intrablock_residuals)
        self.out = None
        self.launches_per_replay = 0

        def run():
            x = ops.nchw_to_nhwc(self.sample)
            if self.intra is not None:
                y = unet.forward_nhwc(x, self.t, self.ctx, self.added, down_intrablock_additional_residuals=self.intra,
                                      residuals_nchw=False)
            elif controlnet is None:
                y = unet.forward_nhwc(x, self.t, self.ctx, self.added)
            else:
                y = denoise_with_controlnet(unet, controlnet, x, self.t, self.ctx, self.added, self.cn)
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

    def __call__(self, sample, timestep, ctx=None, added_cond_kwargs=None, cond_embeddings=None, scale_tables=None):
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
        for src, dst in ((cond_embeddings, "embs"), (scale_tables, "tables")):
            if src is not None:
                for a, b in zip(getattr(self.cn, dst), src):
                    a.copy_(b, non_blocking=True)
        self.graph.replay()
        ops._count(self.launches_per_replay)
        return self.out


def _nets(controlnet):
    return controlnet.nets if isinstance(controlnet, MultiControlNetModel) else [controlnet]


def controlnet_state(controlnet, sample_shape, controlnet_rows, dev):
    """Device buffers of the ControlNet part of one denoiser step for `sample_shape` latents: per net a conditioning
    embedding [controlnet_rows, H, W, C0] and a scale table; with controlnet_rows < rows, zeroed residual buffers
    [rows, ...] whose last controlnet_rows rows the zero convs overwrite (the first rows stay zero,
    pipeline_controlnet.py:1093-1100)."""
    rows, _, H, W = sample_shape
    nets = _nets(controlnet)
    cn = SimpleNamespace(lo=rows - controlnet_rows, out=None,
                         embs=[torch.zeros(controlnet_rows, H, W, n.config.block_out_channels[0], device=dev, dtype=bf16)
                               for n in nets],
                         tables=[torch.zeros(n.num_residuals, n._scale_width, device=dev, dtype=torch.float32)
                                 for n in nets])
    if cn.lo:
        bufs = [torch.zeros(rows, h, w, c, device=dev, dtype=bf16) for h, w, c in nets[0].residual_shapes(H, W)]
        cn.out = (bufs[:-1], bufs[-1])
    return cn


def denoise_with_controlnet(unet, controlnet, x, t, ctx, added, cn):
    """ControlNet(s) on rows [cn.lo:] of the NHWC model input, then the UNet on all rows with their residuals
    (pipeline_controlnet.py:1063-1113). t: device fp32 [rows]. Returns the UNet's NHWC output."""
    lo = cn.lo
    cadded = None if added is None else {k: v[lo:] for k, v in added.items()}
    out = None if cn.out is None else ([d[lo:] for d in cn.out[0]], cn.out[1][lo:])
    if isinstance(controlnet, MultiControlNetModel):
        down, mid = controlnet.forward_nhwc(x[lo:], t[lo:], ctx[lo:], cn.embs, cn.tables, cadded, out=out)
    else:
        down, mid = controlnet.forward_nhwc(x[lo:], t[lo:], ctx[lo:], cn.embs[0], cn.tables[0], cadded, out=out)
    if cn.out is not None:
        down, mid = cn.out
    return unet.forward_nhwc(x, t, ctx, added, down_block_additional_residuals=down, mid_block_additional_residual=mid,
                             residuals_nchw=False)


class StableDiffusionPipeline:
    """Loop-only mirror of ppdiffusers.StableDiffusionPipeline / StableDiffusionXLPipeline.__call__."""

    def __init__(self, unet: UNet2DConditionModel, scheduler: DDIMScheduler, use_cuda_graph: bool = True, vae=None):
        self.unet, self.scheduler, self.use_cuda_graph, self.vae = unet, scheduler, use_cuda_graph, vae
        self._graphed = {}
        self._lora_scale = 1.0  # the LoRA call scale of the call in progress

    # ---- LoRA (LoraLoaderMixin, loaders/lora.py:109-352; the weights live in self.unet) -------------------------------
    def load_lora_weights(self, pretrained_model_name_or_path_or_dict, adapter_name=None, **kwargs):
        """Loads a LoRA into the UNet (UNet2DConditionModel.load_attn_procs; text-encoder entries are skipped with a
        warning). Captured CUDA graphs stay valid: the weights change in place."""
        return self.unet.load_attn_procs(pretrained_model_name_or_path_or_dict, adapter_name=adapter_name, **kwargs)

    def lora_state_dict(self, pretrained_model_name_or_path_or_dict, **kwargs):
        """(state_dict, network_alphas, from_diffusers), text-encoder entries included (lora.lora_state_dict)."""
        from .lora import lora_state_dict
        return lora_state_dict(pretrained_model_name_or_path_or_dict, self.unet.config, **kwargs)

    def fuse_lora(self, lora_scale: float = 1.0):
        self.unet.fuse_lora(lora_scale)

    def unfuse_lora(self):
        self.unet.unfuse_lora()

    def set_adapters(self, adapter_names, adapter_weights=None):
        self.unet.set_adapters(adapter_names, adapter_weights)

    def unload_lora_weights(self):
        self.unet.unload_lora_weights()

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

    def _begin(self, sample_shape, ctx, added, B, do_cfg):
        """Per-call set-up of the denoiser once the loop's inputs are known: the CUDA graph (or None = eager)."""
        return self._denoiser(sample_shape, ctx.shape, added)

    def _predict(self, den, i, t, model_in, ctx, added, first):
        """The model output of step i for the NCHW fp32 model input (the static inputs are copied on the first step)."""
        if den is not None:
            return den(model_in, float(t), ctx if first else None, added if first else None)
        return self.unet.forward(model_in, float(t), ctx, added_cond_kwargs=added,
                                 cross_attention_kwargs={"scale": self._lora_scale}, return_dict=False)[0]

    @torch.no_grad()
    def __call__(self, prompt=None, height: Optional[int] = None, width: Optional[int] = None,
                 num_inference_steps: int = 50, guidance_scale: float = 7.5, negative_prompt=None, eta: float = 0.0,
                 latents: Optional[torch.Tensor] = None, prompt_embeds: Optional[torch.Tensor] = None,
                 negative_prompt_embeds: Optional[torch.Tensor] = None, output_type: str = "latent",
                 added_cond_kwargs: Optional[Dict[str, torch.Tensor]] = None,
                 negative_added_cond_kwargs: Optional[Dict[str, torch.Tensor]] = None, callback_on_step_end=None,
                 generator: Optional[torch.Generator] = None, guidance_rescale: float = 0.0,
                 cross_attention_kwargs: Optional[Dict[str, Any]] = None):
        """cross_attention_kwargs: {"scale": s} sets the LoRA call scale of the unfused adapters (default 1.0). It is
        applied once, before the loop (one kernel launch when it changes the weights); other keys would need custom
        attention processors, which the pipelines do not run."""
        if prompt is not None or negative_prompt is not None:
            raise NotImplementedError("text encoders are outside the hot path: pass prompt_embeds / negative_prompt_embeds")
        if prompt_embeds is None:
            raise ValueError("Provide either `prompt` or `prompt_embeds`. Cannot leave both `prompt` and `prompt_embeds` undefined.")
        if output_type not in ("latent", "pt"):
            raise NotImplementedError("output_type must be 'latent' or 'pt' (PIL / numpy conversion is the caller's)")
        kw = dict(cross_attention_kwargs or {})
        if set(kw) - {"scale"}:
            raise NotImplementedError(f"cross_attention_kwargs {sorted(set(kw) - {'scale'})}: only 'scale' (the LoRA "
                                      "scale) is supported by the pipelines")
        from .. import ops
        self._lora_scale = float(kw.get("scale", 1.0))
        self.unet._set_lora_scale(self._lora_scale)
        dev = self.unet.device
        B = prompt_embeds.shape[0]
        do_cfg = guidance_scale > 1.0  # pipeline_stable_diffusion.py:781
        if do_cfg and negative_prompt_embeds is None:
            negative_prompt_embeds = torch.zeros_like(prompt_embeds)
        g = generator or torch.Generator().manual_seed(0)
        if latents is None:
            if height is None or width is None:
                raise ValueError("height/width (or latents) are required")
            latents = torch.randn(B, self.unet.config.in_channels, height // 8, width // 8, generator=g)
        # prepare_extra_step_kwargs (pipeline_stable_diffusion.py:466-483): a scheduler whose step can draw noise (Euler
        # a, DDIM with eta > 0, DPM-Solver++ 2M SDE) takes the call's generator, which seeds its Philox stream; eta
        # goes to DDIM and, as in the reference, is ignored by every other scheduler
        extra = {"generator": g} if getattr(self.scheduler, "takes_generator", False) else {}
        if isinstance(self.scheduler, DDIMScheduler):
            extra["eta"] = eta
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
        den = self._begin(sample_shape, ctx, added, B, do_cfg)
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
            eps = self._predict(den, i, t, model_in, ctx, added, first)
            first = False
            if do_cfg and guidance_rescale > 0.0:
                # rescale_noise_cfg (pipeline_stable_diffusion.py:69-80, :886-888; SDXL :1061-1067): the guided
                # prediction is rescaled to the text branch's per-sample std before the scheduler step
                guided = ops.cfg_combine(eps[:B], eps[B:], guidance_scale, guidance_rescale)
                self.scheduler.step(guided, t, latents, out=nxt, **extra)
            elif do_cfg:  # noise_pred_uncond + g*(noise_pred_text - noise_pred_uncond) (:882-884), fused with the step
                self.scheduler.step(eps[:B], t, latents, model_output_cond=eps[B:], guidance_scale=guidance_scale, out=nxt,
                                    **extra)
            else:
                self.scheduler.step(eps, t, latents, out=nxt, **extra)
            latents, nxt = nxt, latents
            if callback_on_step_end is not None:
                callback_on_step_end(self, i, t, {"latents": latents})
        return latents if output_type == "latent" else self.decode_latents(latents)


class StableDiffusionControlNetPipeline(StableDiffusionPipeline):
    """Loop-only mirror of ppdiffusers.StableDiffusionControlNetPipeline / StableDiffusionXLControlNetPipeline.__call__
    (pipeline_controlnet.py:1047-1130, pipeline_controlnet_sd_xl.py's loop): each step runs the ControlNet(s) and the
    UNet with their residuals (one CUDA graph per shape), then the CFG combine + scheduler kernel. The control images'
    conditioning embedding does not depend on the timestep, so it runs once per call. Steps whose keep is 0 run the
    ControlNet with scale 0, as the reference does.
    `controlnet`: a ControlNetModel, a MultiControlNetModel or a list of ControlNetModels."""

    def __init__(self, unet: UNet2DConditionModel, controlnet, scheduler: DDIMScheduler, use_cuda_graph: bool = True,
                 vae=None):
        super().__init__(unet, scheduler, use_cuda_graph=use_cuda_graph, vae=vae)
        if isinstance(controlnet, (list, tuple)):
            controlnet = MultiControlNetModel(controlnet)
        self.controlnet = controlnet
        self._control = None  # the control arguments of the call in progress

    @torch.no_grad()
    def __call__(self, prompt=None, height: Optional[int] = None, width: Optional[int] = None,
                 image: Union[torch.Tensor, List[torch.Tensor]] = None, num_inference_steps: int = 50,
                 guidance_scale: float = 7.5, negative_prompt=None, eta: float = 0.0,
                 latents: Optional[torch.Tensor] = None, prompt_embeds: Optional[torch.Tensor] = None,
                 negative_prompt_embeds: Optional[torch.Tensor] = None, output_type: str = "latent",
                 controlnet_conditioning_scale: Union[float, List[float]] = 1.0, guess_mode: bool = False,
                 control_guidance_start: Union[float, List[float]] = 0.0,
                 control_guidance_end: Union[float, List[float]] = 1.0,
                 added_cond_kwargs: Optional[Dict[str, torch.Tensor]] = None,
                 negative_added_cond_kwargs: Optional[Dict[str, torch.Tensor]] = None, callback_on_step_end=None,
                 generator: Optional[torch.Generator] = None, guidance_rescale: float = 0.0,
                 cross_attention_kwargs: Optional[Dict[str, Any]] = None):
        """`image`: the control image, fp32 [B | 1, C, H, W] in [0, 1] (a list of them, one per net, for
        Multi-ControlNet); loading and resizing images is the caller's job. Other arguments as
        StableDiffusionPipeline.__call__ and the reference (pipeline_controlnet.py:905-1003)."""
        multi = isinstance(self.controlnet, MultiControlNetModel)
        nets = _nets(self.controlnet)
        if image is None:
            raise ValueError("`image` (the control image) is required")
        images = list(image) if multi else [image]
        if len(images) != len(nets):
            raise ValueError(f"{len(nets)} ControlNets need {len(nets)} control images, got {len(images)}")
        # pipeline_controlnet.py:951-965: align the guidance window (and the scale) with the number of nets
        if not isinstance(control_guidance_start, list) and isinstance(control_guidance_end, list):
            control_guidance_start = len(control_guidance_end) * [control_guidance_start]
        elif not isinstance(control_guidance_end, list) and isinstance(control_guidance_start, list):
            control_guidance_end = len(control_guidance_start) * [control_guidance_end]
        elif not isinstance(control_guidance_start, list) and not isinstance(control_guidance_end, list):
            control_guidance_start, control_guidance_end = [control_guidance_start] * len(nets), [control_guidance_end] * len(nets)
        if len(control_guidance_start) != len(nets) or len(control_guidance_end) != len(nets):
            raise ValueError(f"control_guidance_start / _end need one entry per ControlNet ({len(nets)})")
        for s, e in zip(control_guidance_start, control_guidance_end):
            # start == end is an empty window: the ControlNet runs at scale 0 on every step
            if s > e or s < 0.0 or e > 1.0:
                raise ValueError(f"control guidance window [{s}, {e}] must satisfy 0 <= start <= end <= 1")
        if multi and isinstance(controlnet_conditioning_scale, (float, int)):
            controlnet_conditioning_scale = [float(controlnet_conditioning_scale)] * len(nets)
        self._control = dict(images=images, scale=controlnet_conditioning_scale, guess_mode=guess_mode,
                             start=control_guidance_start, end=control_guidance_end,
                             steps=num_inference_steps, guidance_scale=guidance_scale)
        try:
            return super().__call__(prompt=prompt, height=height, width=width, num_inference_steps=num_inference_steps,
                                    guidance_scale=guidance_scale, negative_prompt=negative_prompt, eta=eta,
                                    latents=latents, prompt_embeds=prompt_embeds,
                                    negative_prompt_embeds=negative_prompt_embeds, output_type=output_type,
                                    added_cond_kwargs=added_cond_kwargs,
                                    negative_added_cond_kwargs=negative_added_cond_kwargs,
                                    callback_on_step_end=callback_on_step_end, generator=generator,
                                    guidance_rescale=guidance_rescale, cross_attention_kwargs=cross_attention_kwargs)
        finally:
            self._control = None

    def _begin(self, sample_shape, ctx, added, B, do_cfg):
        from .. import ops
        c = self._control
        dev = self.unet.device
        rows = sample_shape[0]
        # guess mode with CFG: the ControlNet sees the conditional rows only (pipeline_controlnet.py:1063-1068)
        cn_rows = B if (c["guess_mode"] and do_cfg) else rows
        nets = _nets(self.controlnet)
        c["keep"] = controlnet_keep(len(self.scheduler.timesteps), c["start"], c["end"], len(nets) > 1)
        embs = []
        for net, img in zip(nets, c["images"]):
            img = img.to(device=dev, dtype=torch.float32).contiguous()
            if img.shape[0] not in (1, B):
                raise ValueError(f"control image batch {img.shape[0]} must be 1 or the prompt batch {B}")
            if tuple(img.shape[2:]) != (sample_shape[2] * net.cond_downscale, sample_shape[3] * net.cond_downscale):
                raise ValueError(f"control image {tuple(img.shape[2:])} does not match the latents {tuple(sample_shape[2:])}")
            e = net.embed_condition(ops.nchw_to_nhwc(img))  # once per call (prepare_image repeats the image, :985-1003)
            embs.append(e if e.shape[0] == cn_rows else e.repeat(cn_rows // e.shape[0], 1, 1, 1))
        c["embs"] = embs
        if self.use_cuda_graph:
            key = ("controlnet", id(self.controlnet), cn_rows, tuple(sample_shape), tuple(ctx.shape),
                   None if added is None else tuple((k, tuple(v.shape)) for k, v in added.items()))
            g = self._graphed.get(key)
            if g is None:
                g = GraphedUNet(self.unet, sample_shape, ctx.shape,
                                None if added is None else {k: v.shape for k, v in added.items()},
                                controlnet=self.controlnet, controlnet_rows=cn_rows)
                self._graphed[key] = g
            return g
        c["state"] = controlnet_state(self.controlnet, sample_shape, cn_rows, dev)
        c["state"].embs = embs
        return None

    def _scale_tables(self, i):
        """Host scale tables of step i: controlnet_conditioning_scale x keep (pipeline_controlnet.py:1074-1080)."""
        c = self._control
        keep, scale = c["keep"][i], c["scale"]
        if isinstance(keep, list):
            cond_scale = [s * k for s, k in zip(scale, keep)]
        else:
            cond_scale = (scale[0] if isinstance(scale, list) else scale) * keep
        nets = _nets(self.controlnet)
        scales = cond_scale if len(nets) > 1 else [cond_scale]
        return [n.scale_table(n.residual_scales(s, c["guess_mode"])) for n, s in zip(nets, scales)]

    def _predict(self, den, i, t, model_in, ctx, added, first):
        from .. import ops
        c = self._control
        tables = self._scale_tables(i)
        if den is not None:
            return den(model_in, float(t), ctx if first else None, added if first else None,
                       cond_embeddings=c["embs"] if first else None, scale_tables=tables)
        st = c["state"]
        st.tables = [tab.to(self.unet.device) for tab in tables]
        tt = torch.full((model_in.shape[0],), float(t), device=self.unet.device, dtype=torch.float32)
        y = denoise_with_controlnet(self.unet, self.controlnet, ops.nchw_to_nhwc(model_in), tt, ctx, added, st)
        return ops.nhwc_to_nchw(y, out_dtype=bf16)


class StableDiffusionAdapterPipeline(StableDiffusionPipeline):
    """Loop-only mirror of ppdiffusers.StableDiffusionAdapterPipeline / StableDiffusionXLAdapterPipeline.__call__
    (pipeline_stable_diffusion_adapter.py:757-870, pipeline_stable_diffusion_xl_adapter.py:1019-1050). The adapter
    does not depend on the timestep: it runs once per call, and one b200mix_weighted_sum_rows pass per feature writes
    w * features into static bf16 NHWC residual buffers [rows, h, w, c]. That pass applies adapter_conditioning_scale
    (the MultiAdapter weights), the tile to the prompt batch and the CFG doubling at once. Each step is then the UNet
    with those residuals (one CUDA graph per shape and adapter) and the CFG combine + scheduler kernel. Steps
    i >= int(num_inference_steps * adapter_conditioning_factor) run with the buffers zeroed: bf16 h + 0 is h, so the
    same graph serves them.
    `adapter`: a T2IAdapter, a MultiAdapter or a list of T2IAdapters."""

    def __init__(self, unet: UNet2DConditionModel, adapter, scheduler: DDIMScheduler, use_cuda_graph: bool = True,
                 vae=None):
        super().__init__(unet, scheduler, use_cuda_graph=use_cuda_graph, vae=vae)
        if isinstance(adapter, (list, tuple)):
            adapter = MultiAdapter(adapter)
        self.adapter = adapter
        self._adapter = None  # the adapter arguments of the call in progress

    @torch.no_grad()
    def __call__(self, prompt=None, height: Optional[int] = None, width: Optional[int] = None,
                 image: Union[torch.Tensor, List[torch.Tensor]] = None, num_inference_steps: int = 50,
                 guidance_scale: float = 7.5, negative_prompt=None, eta: float = 0.0,
                 latents: Optional[torch.Tensor] = None, prompt_embeds: Optional[torch.Tensor] = None,
                 negative_prompt_embeds: Optional[torch.Tensor] = None, output_type: str = "latent",
                 adapter_conditioning_scale: Union[float, List[float]] = 1.0, adapter_conditioning_factor: float = 1.0,
                 added_cond_kwargs: Optional[Dict[str, torch.Tensor]] = None,
                 negative_added_cond_kwargs: Optional[Dict[str, torch.Tensor]] = None, callback_on_step_end=None,
                 generator: Optional[torch.Generator] = None, guidance_rescale: float = 0.0,
                 cross_attention_kwargs: Optional[Dict[str, Any]] = None):
        """`image`: the adapter input, fp32 [B | 1, C, H, W] in [0, 1] (a list of them, one per adapter, for a
        MultiAdapter), with H and W 8x the latent size; loading and resizing images is the caller's job.
        `adapter_conditioning_scale`: a float, or for a MultiAdapter a list of one weight per adapter.
        Other arguments as StableDiffusionPipeline.__call__."""
        multi = isinstance(self.adapter, MultiAdapter)
        if image is None:
            raise ValueError("`image` (the adapter input) is required")
        if multi:  # pipeline_stable_diffusion_adapter.py:543-552
            if not isinstance(image, list):
                raise ValueError("MultiAdapter is enabled, but `image` is not a list. Please pass a list of images to "
                                 "`image`.")
            if len(image) != self.adapter.num_adapter:
                raise ValueError(f"MultiAdapter requires passing the same number of images as adapters. Given "
                                 f"{len(image)} images and {self.adapter.num_adapter} adapters.")
            images, weights = image, self.adapter.weights(adapter_conditioning_scale)  # passed as weights (:823-826)
        else:
            if not torch.is_tensor(image):
                raise ValueError(f"a single T2IAdapter takes one image tensor, got {type(image).__name__}")
            images, weights = [image], [float(adapter_conditioning_scale)]  # v * scale (:827-830)
        self._adapter = dict(images=images, weights=weights,
                             cut=int(num_inference_steps * adapter_conditioning_factor))  # xl :1029-1032
        try:
            return super().__call__(prompt=prompt, height=height, width=width, num_inference_steps=num_inference_steps,
                                    guidance_scale=guidance_scale, negative_prompt=negative_prompt, eta=eta,
                                    latents=latents, prompt_embeds=prompt_embeds,
                                    negative_prompt_embeds=negative_prompt_embeds, output_type=output_type,
                                    added_cond_kwargs=added_cond_kwargs,
                                    negative_added_cond_kwargs=negative_added_cond_kwargs,
                                    callback_on_step_end=callback_on_step_end, generator=generator,
                                    guidance_rescale=guidance_rescale, cross_attention_kwargs=cross_attention_kwargs)
        finally:
            self._adapter = None

    def _begin(self, sample_shape, ctx, added, B, do_cfg):
        from .. import ops
        c = self._adapter
        dev = self.unet.device
        rows, _, H, W = sample_shape
        adapters = self.adapter.adapters if isinstance(self.adapter, MultiAdapter) else [self.adapter]
        feats = []
        for adapter, img in zip(adapters, c["images"]):
            if img.dim() != 4 or img.shape[0] not in (1, B):
                raise ValueError(f"adapter image of shape {tuple(img.shape)} must be [1 or {B}, C, H, W]")
            if tuple(img.shape[2:]) != (8 * H, 8 * W):
                raise ValueError(f"adapter image {tuple(img.shape[2:])} does not match the latents {(H, W)} (8x)")
            feats.append(adapter.forward(img.to(device=dev, dtype=torch.float32)))
        shapes = [tuple(f.shape[1:]) for f in feats[0]]
        den = None
        if self.use_cuda_graph:
            key = ("adapter", id(self.adapter), tuple(sample_shape), tuple(ctx.shape), tuple(shapes),
                   None if added is None else tuple((k, tuple(v.shape)) for k, v in added.items()))
            den = self._graphed.get(key)
            if den is None:
                bufs = [torch.zeros((rows,) + s, device=dev, dtype=bf16) for s in shapes]
                den = GraphedUNet(self.unet, sample_shape, ctx.shape,
                                  None if added is None else {k: v.shape for k, v in added.items()},
                                  intrablock_residuals=bufs)
                self._graphed[key] = den
            c["bufs"] = den.intra
        else:
            c["bufs"] = [torch.empty((rows,) + s, device=dev, dtype=bf16) for s in shapes]
        for k, buf in enumerate(c["bufs"]):
            ops.weighted_sum_rows([f[k] for f in feats], c["weights"], out=buf)
        return den

    def _predict(self, den, i, t, model_in, ctx, added, first):
        from .. import ops
        c = self._adapter
        if i == c["cut"]:  # from here on without residuals
            for buf in c["bufs"]:
                ops.zero_(buf)
        if den is not None:
            return den(model_in, float(t), ctx if first else None, added if first else None)
        tt = torch.full((model_in.shape[0],), float(t), device=self.unet.device, dtype=torch.float32)
        y = self.unet.forward_nhwc(ops.nchw_to_nhwc(model_in), tt, ctx, added,
                                   down_intrablock_additional_residuals=c["bufs"], residuals_nchw=False)
        return ops.nhwc_to_nchw(y, out_dtype=bf16)


StableDiffusionXLAdapterPipeline = StableDiffusionAdapterPipeline  # the SDXL loop is the same class (added_cond_kwargs)


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
        # always a copy: the loop alternates between two buffers and would otherwise write its steps into the
        # caller's tensor when that is already an fp32 tensor on the device
        latents = latents.to(device=dev, dtype=torch.float32, copy=True).contiguous()
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
