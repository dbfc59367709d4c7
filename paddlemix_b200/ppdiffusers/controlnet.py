"""ControlNetModel / MultiControlNetModel — host-side mirrors of ppdiffusers.models.controlnet.ControlNetModel
(ppdiffusers/models/controlnet.py:116-882) and pipelines/controlnet/multicontrolnet.py for the SD / SDXL configuration
family of UNet2DConditionModel, on the same sm_90a kernels.

The ControlNet is the UNet's encoder half (conv_in, time / added-condition embeddings, down blocks, mid block) plus
  * the conditioning embedding (ControlNetConditioningEmbedding, :71-113): 3x3 convs at image resolution with 3 / 16 /
    32 / 96 input channels on b200mix_conv3x3_narrow (SiLU fused), the 256 -> C0 conv_out on the wgmma conv3x3;
  * one zero conv (1x1) per down residual and one for the mid block: each is one ops.linear whose epilogue applies the
    conditioning scale through `row_gate` (v = s * (W c + b), plus the previous net's residual for Multi-ControlNet).
    The scales live in a device fp32 table, so a captured CUDA graph picks up new scales without a new capture.
It reuses the UNet's layer classes, time embedding, batched time_emb_proj / cross-attention K/V projections and
weight loading (it subclasses UNet2DConditionModel for them); its forward is its own.
"""
from dataclasses import dataclass
from typing import Any, Dict, List, Optional, Sequence, Tuple, Union

import torch

from ..modeling import FrozenDict, synthetic_state_dict
from .unet_2d_condition import UNet2DConditionModel, _check_reference_defaults, _Conv3x3, _Linear

bf16 = torch.bfloat16

# reference defaults of the ControlNetModel arguments this mirror does not implement (controlnet.py:188-227)
_CONTROLNET_DEFAULTS = dict(
    encoder_hid_dim=None, encoder_hid_dim_type=None, class_embed_type=None, num_class_embeds=None,
    upcast_attention=False, resnet_time_scale_shift="default", addition_embed_type_num_heads=64)
# UNet config keys from_unet() may meet that a ControlNet does not have (its up path, output conv, ...)
_UNET_ONLY = ("sample_size", "out_channels", "up_block_types", "resnet_out_scale_factor", "time_cond_proj_dim")


@dataclass
class ControlNetOutput:
    """ppdiffusers.models.controlnet.ControlNetOutput (:50-68)."""
    down_block_res_samples: Tuple[torch.Tensor, ...] = None
    mid_block_res_sample: torch.Tensor = None

    def __iter__(self):
        return iter((self.down_block_res_samples, self.mid_block_res_sample))


def guess_mode_scales(n_residuals: int, conditioning_scale) -> torch.Tensor:
    """controlnet.py:855-857: fp32 logspace(-1, 0, n + 1) (0.1 ... 1.0) times the conditioning scale."""
    return torch.logspace(-1, 0, n_residuals + 1, dtype=torch.float32) * conditioning_scale


def controlnet_keep(n_steps: int, control_guidance_start: Sequence[float], control_guidance_end: Sequence[float],
                    multi: bool):
    """pipeline_controlnet.py:1047-1053: per step, 1.0 while the step lies inside [start, end] of the schedule, else
    0.0; one float per step for a single ControlNetModel, one list per step for a MultiControlNetModel."""
    keep = []
    for i in range(n_steps):
        ks = [1.0 - float(i / n_steps < s or (i + 1) / n_steps > e)
              for s, e in zip(control_guidance_start, control_guidance_end)]
        keep.append(ks if multi else ks[0])
    return keep


def map_unet_state_dict(controlnet_shapes: Dict[str, tuple], unet_state_dict: Dict[str, Any]) -> Dict[str, Any]:
    """The parameters ControlNetModel.from_unet(load_weights_from_unet=True) copies from the UNet (controlnet.py:509-518):
    conv_in, time_embedding, down_blocks and mid_block, under the same names."""
    prefixes = ("conv_in.", "time_embedding.", "down_blocks.", "mid_block.")
    return {k: unet_state_dict[k] for k in controlnet_shapes if k.startswith(prefixes)}


class ControlNetModel(UNet2DConditionModel):
    """Drop-in for ppdiffusers.ControlNetModel on the denoising hot path (inference)."""

    def __init__(self, in_channels: int = 4, conditioning_channels: int = 3, flip_sin_to_cos: bool = True,
                 freq_shift: int = 0,
                 down_block_types: Tuple[str] = ("CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D",
                                                 "DownBlock2D"),
                 mid_block_type: Optional[str] = "UNetMidBlock2DCrossAttn",
                 only_cross_attention: Union[bool, Tuple[bool]] = False,
                 block_out_channels: Tuple[int] = (320, 640, 1280, 1280), layers_per_block: int = 2,
                 downsample_padding: int = 1, mid_block_scale_factor: float = 1, act_fn: str = "silu",
                 norm_num_groups: Optional[int] = 32, norm_eps: float = 1e-5, cross_attention_dim: int = 1280,
                 transformer_layers_per_block: Union[int, Tuple[int]] = 1,
                 attention_head_dim: Union[int, Tuple[int]] = 8, num_attention_heads=None,
                 use_linear_projection: bool = False, addition_embed_type: Optional[str] = None,
                 addition_time_embed_dim: Optional[int] = None,
                 projection_class_embeddings_input_dim: Optional[int] = None,
                 controlnet_conditioning_channel_order: str = "rgb",
                 conditioning_embedding_out_channels: Optional[Tuple[int]] = (16, 32, 96, 256),
                 global_pool_conditions: bool = False, data_format: str = "NCHW", **unsupported):
        if global_pool_conditions:
            raise NotImplementedError("ControlNetModel(b200): global_pool_conditions=True is not supported")
        if num_attention_heads is not None and num_attention_heads != attention_head_dim:
            raise NotImplementedError("ControlNetModel(b200): num_attention_heads must be None (it defaults to "
                                      "attention_head_dim, controlnet.py:236)")
        _check_reference_defaults("ControlNetModel", unsupported, _CONTROLNET_DEFAULTS)
        if len(block_out_channels) != len(down_block_types):
            raise ValueError(f"Must provide the same number of `block_out_channels` as `down_block_types`. "
                             f"`block_out_channels`: {block_out_channels}. `down_block_types`: {down_block_types}.")
        if act_fn != "silu" or mid_block_type != "UNetMidBlock2DCrossAttn" or only_cross_attention \
                or downsample_padding != 1 or mid_block_scale_factor != 1:
            raise NotImplementedError("ControlNetModel(b200) covers the SD / SDXL configuration family only")
        if addition_embed_type not in (None, "text_time"):
            raise NotImplementedError(f"addition_embed_type={addition_embed_type}")
        if controlnet_conditioning_channel_order not in ("rgb", "bgr"):
            raise ValueError(f"unknown `controlnet_conditioning_channel_order`: {controlnet_conditioning_channel_order}")
        ch = tuple(conditioning_embedding_out_channels)
        cfg = dict(in_channels=in_channels, conditioning_channels=conditioning_channels,
                   flip_sin_to_cos=flip_sin_to_cos, freq_shift=freq_shift, down_block_types=tuple(down_block_types),
                   mid_block_type=mid_block_type, only_cross_attention=only_cross_attention,
                   block_out_channels=tuple(block_out_channels), layers_per_block=layers_per_block,
                   downsample_padding=downsample_padding, mid_block_scale_factor=mid_block_scale_factor, act_fn=act_fn,
                   norm_num_groups=norm_num_groups, norm_eps=norm_eps, cross_attention_dim=cross_attention_dim,
                   transformer_layers_per_block=transformer_layers_per_block, attention_head_dim=attention_head_dim,
                   num_attention_heads=num_attention_heads, use_linear_projection=use_linear_projection,
                   addition_embed_type=addition_embed_type, addition_time_embed_dim=addition_time_embed_dim,
                   projection_class_embeddings_input_dim=projection_class_embeddings_input_dim,
                   controlnet_conditioning_channel_order=controlnet_conditioning_channel_order,
                   conditioning_embedding_out_channels=ch, global_pool_conditions=False, data_format=data_format,
                   resnet_out_scale_factor=1.0)  # the ControlNet's resnets keep get_down_block's output scale 1
        self.config = FrozenDict(cfg)
        self.in_channels, self.data_format = in_channels, data_format
        self.dtype = bf16
        self.device = None
        self._build()
        for conv, _ in self.cond_convs:  # b200mix_conv3x3 (Cin % 64 == 0) or b200mix_conv3x3_narrow
            if conv.cin % 64 and not (conv.cin <= 128 and conv.cout % 8 == 0 and conv.cout <= 256):
                raise NotImplementedError(f"conditioning embedding conv {conv.name}: {conv.cin} -> {conv.cout} channels "
                                          "(needs Cin % 64 == 0, or Cin <= 128 and Cout a multiple of 8 up to 256)")
        self._graphs: Dict[Any, Any] = {}

    def _build(self):
        self._build_encoder()
        c = self.config
        boc, ch = c.block_out_channels, c.conditioning_embedding_out_channels
        # (conv, stride) of ControlNetConditioningEmbedding: conv_in, then per step a same-width and a stride-2 conv
        self.cond_convs = [(_Conv3x3("controlnet_cond_embedding.conv_in", c.conditioning_channels, ch[0]), 1)]
        for i in range(len(ch) - 1):
            self.cond_convs.append((_Conv3x3(f"controlnet_cond_embedding.blocks.{2 * i}", ch[i], ch[i]), 1))
            self.cond_convs.append((_Conv3x3(f"controlnet_cond_embedding.blocks.{2 * i + 1}", ch[i], ch[i + 1]), 2))
        self.cond_convs.append((_Conv3x3("controlnet_cond_embedding.conv_out", ch[-1], boc[0]), 1))
        widths = [boc[0]]
        for blk in self.down:
            widths += [r.cout for r in blk.resnets] + ([blk.down.cout] if blk.down is not None else [])
        self.zero_convs = [_Linear(f"controlnet_down_blocks.{k}", w, w, conv1x1=True) for k, w in enumerate(widths)]
        self.zero_mid = _Linear("controlnet_mid_block", boc[-1], boc[-1], conv1x1=True)
        self.cond_downscale = 2 ** (len(ch) - 1)  # control image pixels per latent pixel (8 for the default)

    def _leaves(self):
        leaves = [self.conv_in, self.time_lin1, self.time_lin2, self.add_lin1, self.add_lin2, *self.resnets,
                  *self.transformers, *(b.down for b in self.down), *(cv for cv, _ in self.cond_convs),
                  *self.zero_convs, self.zero_mid]
        return [m for m in leaves if m is not None]

    @property
    def num_residuals(self) -> int:
        """Down residuals + the mid residual."""
        return len(self.zero_convs) + 1

    def residual_shapes(self, H: int, W: int) -> List[Tuple[int, int, int]]:
        """(h, w, channels) of every residual (down residuals, then the mid residual) for an H x W latent."""
        out = [(H, W, self.config.block_out_channels[0])]
        for blk in self.down:
            out += [(H, W, r.cout) for r in blk.resnets]
            if blk.down is not None:
                H, W = H // 2, W // 2
                out.append((H, W, blk.down.cout))
        return out + [(H, W, self.config.block_out_channels[-1])]

    def load_state_dict(self, state_dict: Dict[str, Any], device: Union[int, str] = 0):
        super().load_state_dict(state_dict, device)
        if self.config.controlnet_conditioning_channel_order == "bgr":
            # paddle.flip(controlnet_cond, axis=[1]) (controlnet.py:733-734) == conv_in reading its input channels in
            # reverse order: flip the filter's input-channel axis once, exactly
            conv = self.cond_convs[0][0]
            conv.w = conv.w.flip(-1).contiguous()
        self._scale_width = -(-max(z.cout for z in (*self.zero_convs, self.zero_mid)) // 4) * 4
        return self

    # ------------------------------------------------------------------------------------------------------------
    @classmethod
    def from_unet(cls, unet: UNet2DConditionModel, controlnet_conditioning_channel_order: str = "rgb",
                  conditioning_embedding_out_channels: Optional[Tuple[int]] = (16, 32, 96, 256),
                  load_weights_from_unet: bool = True, conditioning_channels: int = 3,
                  unet_state_dict: Optional[Dict[str, Any]] = None, seed: int = 1,
                  device: Optional[Union[int, str]] = None):
        """controlnet.py:449-520. The device UNet keeps only fused / transposed copies of its weights, so the
        reference-named `unet_state_dict` it was loaded from is passed alongside it. The ControlNet's own layers
        (conditioning embedding, add_embedding) get synthetic weights from `seed`; the zero convs and the
        conditioning embedding's conv_out are zero (zero_module, :885-889). Loaded onto `device` (default: the UNet's)."""
        c = unet.config
        kw = {k: v for k, v in c.items() if k not in _UNET_ONLY}
        cn = cls(**kw, controlnet_conditioning_channel_order=controlnet_conditioning_channel_order,
                 conditioning_embedding_out_channels=conditioning_embedding_out_channels,
                 conditioning_channels=conditioning_channels)
        shapes = cn.state_dict_shapes()
        P = synthetic_state_dict(shapes, seed, "cpu")
        for k in shapes:
            if k.startswith(("controlnet_down_blocks.", "controlnet_mid_block.", "controlnet_cond_embedding.conv_out.")):
                P[k] = torch.zeros(shapes[k], dtype=bf16)
        if load_weights_from_unet:
            if unet_state_dict is None:
                raise ValueError("from_unet(load_weights_from_unet=True) needs the UNet's reference-named "
                                 "`unet_state_dict`: the device UNet does not keep its weights in that form")
            P.update(map_unet_state_dict(shapes, unet_state_dict))
        dev = device if device is not None else unet.device
        return cn if dev is None else cn.load_state_dict(P, device=dev)

    # ------------------------------------------------------------------------------------------------------------
    def residual_scales(self, conditioning_scale: Union[float, Sequence[float]] = 1.0, guess_mode: bool = False):
        """fp32 [num_residuals] scale of each residual (controlnet.py:854-869): guess mode = logspace(-1, 0) times the
        scale; a list gives one scale per residual (the mid residual last)."""
        n = self.num_residuals
        if guess_mode:
            return guess_mode_scales(n - 1, conditioning_scale)
        if isinstance(conditioning_scale, (float, int)):
            return torch.full((n,), float(conditioning_scale), dtype=torch.float32)
        s = torch.as_tensor(list(conditioning_scale), dtype=torch.float32)
        if s.numel() != n:
            raise ValueError(f"conditioning_scale has {s.numel()} entries, this ControlNet has {n} residuals")
        return s

    def scale_table(self, scales: torch.Tensor) -> torch.Tensor:
        """Host fp32 [num_residuals, width] table (one row per residual, the scale repeated across the channels) that
        the zero convs read as their epilogue row_gate."""
        return scales.to(torch.float32)[:, None].expand(-1, self._scale_width).contiguous()

    def embed_condition(self, cond_nhwc: torch.Tensor) -> torch.Tensor:
        """ControlNetConditioningEmbedding (controlnet.py:103-113) on a bf16 NHWC control image [B, h, w, C]:
        conv + SiLU layers on b200mix_conv3x3_narrow (the wgmma conv3x3 where Cin % 64 == 0), then conv_out.
        Returns bf16 NHWC [B, h / 8, w / 8, block_out_channels[0]]. It does not depend on the timestep: pipelines
        run it once per call."""
        from .. import ops
        from .._lib import ACT_NONE, ACT_SILU
        e = cond_nhwc
        last = len(self.cond_convs) - 1
        for i, (conv, stride) in enumerate(self.cond_convs):
            act = ACT_NONE if i == last else ACT_SILU
            if conv.cin % 64 == 0:
                e = ops.conv3x3(e, conv.w, conv.b, stride=stride, act=act)
            else:
                e = ops.conv3x3_narrow(e, conv.w, conv.b, stride=stride, act=act)
        return e

    def forward_nhwc(self, x_nhwc, timestep, ctx, cond_embedding, scale_table, added_cond_kwargs=None,
                     cross_attention_kwargs=None, attention_mask=None, out=None, accumulate=False):
        """x_nhwc: bf16 / fp32 [B,H,W,Cin]; ctx: bf16 [B,L,D]; cond_embedding: embed_condition()'s output for these B
        rows; scale_table: device fp32 [num_residuals, width] (scale_table()). Returns (down list, mid), bf16 NHWC.
        out: optional (down list, mid) of bf16 NHWC buffers to write into (e.g. the conditional half of [2B, ...]
        buffers); accumulate: add to what `out` holds (Multi-ControlNet: the previous nets' sum) in the epilogue."""
        from .. import ops
        if accumulate and out is None:
            raise ValueError("accumulate=True needs the `out` buffers to add to")
        B = x_nhwc.shape[0]
        temb_all = self._embeddings(timestep, B, added_cond_kwargs)
        self._project_context(ctx)
        kw, am = cross_attention_kwargs, attention_mask
        h = ops.conv3x3_small_cin(x_nhwc, self.conv_in.w, self.conv_in.b)
        h = ops.add_residual_nhwc(h, cond_embedding, r_nchw=False, out=h)
        skips = [h]
        for blk in self.down:
            for j, r in enumerate(blk.resnets):
                h = r(h, temb_all)
                if blk.attns:
                    h = blk.attns[j](h, ctx, kw, am, None)
                skips.append(h)
            if blk.down is not None:
                h = ops.conv3x3(h, blk.down.w, blk.down.b, stride=2)
                skips.append(h)
        h = self.mid.res0(h, temb_all)
        h = self.mid.attn(h, ctx, kw, am, None)
        h = self.mid.res1(h, temb_all)
        # zero convs: v = scale * (W s + b) [+ previous residual], rounded to bf16 once (the reference rounds the
        # conv output and its product with the scale separately, controlnet.py:846-869)
        outs_d, out_m = (None, None) if out is None else out
        down = []
        for k, (zc, s) in enumerate(zip(self.zero_convs, skips)):
            o = None if out is None else outs_d[k]
            down.append(ops.linear(s, zc.w, zc.b, row_gate=scale_table[k:k + 1], residual=o if accumulate else None, out=o))
        mid = ops.linear(h, self.zero_mid.w, self.zero_mid.b, row_gate=scale_table[len(skips):len(skips) + 1],
                         residual=out_m if accumulate else None, out=out_m)
        return down, mid

    def forward(self, sample, timestep, encoder_hidden_states, controlnet_cond, conditioning_scale=1.0,
                class_labels=None, timestep_cond=None, attention_mask=None, added_cond_kwargs=None,
                cross_attention_kwargs=None, guess_mode: bool = False, return_dict: bool = True):
        """controlnet.py:670-882. sample [B,C,H,W] and controlnet_cond [B,3,8H,8W] (NCHW, or NHWC under
        data_format="NHWC"), host or device. Returns ControlNetOutput(down_block_res_samples, mid_block_res_sample)
        or the tuple (down, mid), bf16 in the input's layout."""
        from .. import ops
        for name, v in (("class_labels", class_labels), ("timestep_cond", timestep_cond)):
            if v is not None:
                raise NotImplementedError(f"ControlNetModel(b200).forward: `{name}` needs a class / condition embedding "
                                          "this configuration family does not have")
        if self.device is None:
            raise RuntimeError("load_state_dict() must be called before forward()")
        dev = self.device
        nhwc = self.config.data_format == "NHWC"
        x = _to_nhwc(sample.to(dev), nhwc, keep_fp32=True)
        cond = _to_nhwc(controlnet_cond.to(dev), nhwc, keep_fp32=False)
        if cond.shape[0] != x.shape[0]:
            raise ValueError(f"controlnet_cond has batch {cond.shape[0]}, sample has {x.shape[0]}")
        ctx = encoder_hidden_states.to(device=dev, dtype=bf16).contiguous()
        table = self.scale_table(self.residual_scales(conditioning_scale, guess_mode)).to(dev)
        down, mid = self.forward_nhwc(x, timestep, ctx, self.embed_condition(cond), table, added_cond_kwargs,
                                      cross_attention_kwargs, attention_mask=self._mask_to_bias(attention_mask, dev))
        if not nhwc:
            down = [ops.nhwc_to_nchw(d, out_dtype=bf16) for d in down]
            mid = ops.nhwc_to_nchw(mid, out_dtype=bf16)
        down = tuple(down)
        if not return_dict:
            return (down, mid)
        return ControlNetOutput(down_block_res_samples=down, mid_block_res_sample=mid)

    __call__ = forward


class MultiControlNetModel:
    """pipelines/controlnet/multicontrolnet.py: several ControlNets whose residuals are summed. Net k's zero convs add
    net k-1's residuals in their epilogue, so the sum costs no extra pass."""

    def __init__(self, controlnets: Sequence[ControlNetModel]):
        self.nets = list(controlnets)
        if not self.nets:
            raise ValueError("MultiControlNetModel needs at least one ControlNetModel")
        if len({n.num_residuals for n in self.nets}) != 1:
            raise ValueError("all ControlNets of a MultiControlNetModel must have the same block structure")

    @property
    def device(self):
        return self.nets[0].device

    @property
    def num_residuals(self) -> int:
        return self.nets[0].num_residuals

    def forward_nhwc(self, x_nhwc, timestep, ctx, cond_embeddings, scale_tables, added_cond_kwargs=None,
                     cross_attention_kwargs=None, attention_mask=None, out=None):
        """Lists of per-net cond_embeddings / scale_tables; see ControlNetModel.forward_nhwc."""
        for k, (net, e, tab) in enumerate(zip(self.nets, cond_embeddings, scale_tables)):
            out = net.forward_nhwc(x_nhwc, timestep, ctx, e, tab, added_cond_kwargs, cross_attention_kwargs,
                                   attention_mask, out=out, accumulate=k > 0)
        return out

    def forward(self, sample, timestep, encoder_hidden_states, controlnet_cond: List[torch.Tensor],
                conditioning_scale: List[float], class_labels=None, timestep_cond=None, attention_mask=None,
                added_cond_kwargs=None, cross_attention_kwargs=None, guess_mode: bool = False,
                return_dict: bool = True):
        """multicontrolnet.py:45-90: one control image and one conditioning scale per net."""
        from .. import ops
        if len(controlnet_cond) != len(self.nets) or len(conditioning_scale) != len(self.nets):
            raise ValueError(f"{len(self.nets)} ControlNets need as many control images and conditioning scales")
        for name, v in (("class_labels", class_labels), ("timestep_cond", timestep_cond)):
            if v is not None:
                raise NotImplementedError(f"MultiControlNetModel(b200).forward: `{name}` is not supported")
        net0 = self.nets[0]
        dev = net0.device
        nhwc = net0.config.data_format == "NHWC"
        x = _to_nhwc(sample.to(dev), nhwc, keep_fp32=True)
        ctx = encoder_hidden_states.to(device=dev, dtype=bf16).contiguous()
        embs = [n.embed_condition(_to_nhwc(c.to(dev), nhwc, keep_fp32=False)) for n, c in zip(self.nets, controlnet_cond)]
        tabs = [n.scale_table(n.residual_scales(s, guess_mode)).to(dev) for n, s in zip(self.nets, conditioning_scale)]
        down, mid = self.forward_nhwc(x, timestep, ctx, embs, tabs, added_cond_kwargs, cross_attention_kwargs,
                                      attention_mask=net0._mask_to_bias(attention_mask, dev))
        if not nhwc:
            down = [ops.nhwc_to_nchw(d, out_dtype=bf16) for d in down]
            mid = ops.nhwc_to_nchw(mid, out_dtype=bf16)
        down = tuple(down)
        if not return_dict:
            return (down, mid)
        return ControlNetOutput(down_block_res_samples=down, mid_block_res_sample=mid)

    __call__ = forward


def _to_nhwc(t, nhwc_in, keep_fp32):
    """Caller's tensor -> contiguous NHWC on the device: bf16, or the fp32 / bf16 input as is for the UNet-style
    sample (conv3x3_small_cin reads fp32)."""
    from .. import ops
    if t.dtype not in (torch.float32, bf16):
        t = t.float()
    t = t.contiguous()
    if not nhwc_in:
        return ops.nchw_to_nhwc(t)
    if keep_fp32 or t.dtype == bf16:
        return t
    return ops.cast(t, bf16)

