"""AutoencoderKL.decode on the sm_90a kernels — host-side mirror of ppdiffusers/models/autoencoder_kl.py:288-325 and
vae.py:182-282 (Decoder), the step that turns the denoising loop's latents into pixels
(pipeline_stable_diffusion.py:910-917; SURVEY.md §8 f2).

Device graph (NHWC bf16): post_quant_conv (1x1 on 4 channels: the tiny-Cin conv kernel with a centre-tap filter) ->
conv_in (tiny-Cin kernel) -> mid block: ResnetBlock2D (GroupNorm+SiLU -> conv3x3 -> GroupNorm+SiLU -> conv3x3 +residual),
one-head attention over H*W tokens, ResnetBlock2D -> 4 x UpDecoderBlock2D (3 resnets each, 1x1 shortcut GEMM where the
width changes, nearest x2 + conv3x3) -> GroupNorm+SiLU -> conv_out -> NCHW fp32.
The mid attention has ONE 512-wide head: it runs as score GEMM (fp32 out) -> row softmax kernel -> PV GEMM per image
(a 512-wide head does not fit the flash kernel's register / shared-memory budget; at 128x128 latents the score matrix is
16384^2 fp32 = 1 GB of scratch that is reused across the batch).
"""
from dataclasses import dataclass
from typing import Any, Dict, Tuple, Union

import torch

from ..modeling import FrozenDict, bind, linear_bias, linear_weight, synthetic_state_dict, to_f32
from .unet_2d_condition import _Conv3x3, _Linear, _Norm

bf16 = torch.bfloat16


@dataclass
class DecoderOutput:
    """ppdiffusers.models.vae.DecoderOutput."""
    sample: torch.Tensor = None


class _VaeResnet:
    """ResnetBlock2D with temb_channels = None (resnet.py:587-808), eps 1e-6, output_scale_factor 1."""

    def __init__(self, name, cin, cout, groups):
        self.name, self.cin, self.cout, self.groups = name, cin, cout, groups
        self.norm1, self.conv1 = _Norm(name + ".norm1", cin), _Conv3x3(name + ".conv1", cin, cout)
        self.norm2, self.conv2 = _Norm(name + ".norm2", cout), _Conv3x3(name + ".conv2", cout, cout)
        self.shortcut = _Linear(name + ".conv_shortcut", cin, cout, conv1x1=True) if cin != cout else None

    def parts(self):
        return [m for m in (self.norm1, self.conv1, self.norm2, self.conv2, self.shortcut) if m is not None]

    def __call__(self, x):
        from .. import ops
        n1 = ops.groupnorm_nhwc(x, self.norm1.w, self.norm1.b, groups=self.groups, eps=1e-6, silu=True)
        h = ops.conv3x3(n1, self.conv1.w, self.conv1.b)
        n2 = ops.groupnorm_nhwc(h, self.norm2.w, self.norm2.b, groups=self.groups, eps=1e-6, silu=True)
        res = x if self.shortcut is None else ops.linear(x, self.shortcut.w, self.shortcut.b)
        return ops.conv3x3(n2, self.conv2.w, self.conv2.b, residual=res)


class AutoencoderKL:
    """Decoder half of ppdiffusers.AutoencoderKL: decode(z, return_dict=True) -> DecoderOutput(sample [B,3,8h,8w])."""

    def __init__(self, in_channels: int = 3, out_channels: int = 3, block_out_channels: Tuple[int] = (128, 256, 512, 512),
                 layers_per_block: int = 2, act_fn: str = "silu", latent_channels: int = 4, norm_num_groups: int = 32,
                 sample_size: int = 512, scaling_factor: float = 0.18215, force_upcast: bool = True, **unsupported):
        if act_fn != "silu":
            raise NotImplementedError("AutoencoderKL(b200): act_fn must be silu")
        for k, v in unsupported.items():
            if k.startswith("_") or k in ("down_block_types", "up_block_types"):
                continue
            raise NotImplementedError(f"AutoencoderKL(b200): config option {k}={v!r} is outside the decode path")
        if any(c % 64 for c in block_out_channels) or latent_channels > 8:
            raise NotImplementedError("AutoencoderKL(b200): block_out_channels must be multiples of 64, latent_channels <= 8")
        self.config = FrozenDict(dict(in_channels=in_channels, out_channels=out_channels, block_out_channels=tuple(block_out_channels),
                                      layers_per_block=layers_per_block, act_fn=act_fn, latent_channels=latent_channels,
                                      norm_num_groups=norm_num_groups, sample_size=sample_size, scaling_factor=scaling_factor,
                                      force_upcast=force_upcast))
        self.device, self.dtype = None, bf16
        boc, g = self.config.block_out_channels, norm_num_groups
        C = boc[-1]
        self.mid_res0 = _VaeResnet("decoder.mid_block.resnets.0", C, C, g)
        self.mid_res1 = _VaeResnet("decoder.mid_block.resnets.1", C, C, g)
        self.attn_norm = _Norm("decoder.mid_block.attentions.0.group_norm", C)
        self.attn_out = _Linear("decoder.mid_block.attentions.0.to_out.0", C, C)
        self.up = []
        rev = list(reversed(boc))
        out = rev[0]
        for i in range(len(boc)):
            prev, out = out, rev[i]
            res = [_VaeResnet(f"decoder.up_blocks.{i}.resnets.{j}", prev if j == 0 else out, out, g) for j in range(layers_per_block + 1)]
            ups = _Conv3x3(f"decoder.up_blocks.{i}.upsamplers.0.conv", out, out, upsample=True) if i != len(boc) - 1 else None
            self.up.append((res, ups))
        self.norm_out = _Norm("decoder.conv_norm_out", boc[0])
        self.conv_out = _Conv3x3("decoder.conv_out", boc[0], out_channels)

    def state_dict_shapes(self) -> Dict[str, tuple]:
        c = self.config
        lc, C = c.latent_channels, c.block_out_channels[-1]
        S = {"post_quant_conv.weight": (lc, lc, 1, 1), "post_quant_conv.bias": (lc,),
             "decoder.conv_in.weight": (C, lc, 3, 3), "decoder.conv_in.bias": (C,)}
        leaves = [*self.mid_res0.parts(), *self.mid_res1.parts(), self.attn_norm, self.attn_out, self.norm_out, self.conv_out]
        for res, ups in self.up:
            for r in res:
                leaves += r.parts()
            if ups is not None:
                leaves.append(ups)
        for m in leaves:
            S.update(m.shapes())
        a = "decoder.mid_block.attentions.0"
        for n in ("to_q", "to_k", "to_v"):
            S[f"{a}.{n}.weight"], S[f"{a}.{n}.bias"] = (C, C), (C,)
        return S

    def init_synthetic_weights(self, seed: int = 1, device: Union[int, str] = 0):
        return self.load_state_dict(synthetic_state_dict(self.state_dict_shapes(), seed, device), device)

    def load_state_dict(self, P: Dict[str, Any], device: Union[int, str] = 0):
        dev = bind(self, P, device)
        c = self.config
        lc, C = c.latent_channels, c.block_out_channels[-1]
        # post_quant_conv (1x1, lc -> lc) as a 3x3 filter with only the centre tap set, output padded to 8 channels
        # (zeros), so that conv_in reads an 8-channel NHWC tensor: both run on the tiny-Cin conv kernel
        wpq = torch.zeros(8, 3, 3, lc)
        wpq[:lc, 1, 1, :] = to_f32(P["post_quant_conv.weight"])[:, :, 0, 0].cpu()
        bpq = torch.zeros(8)
        bpq[:lc] = to_f32(P["post_quant_conv.bias"]).cpu()
        self.pq_w, self.pq_b = wpq.to(dev, bf16).contiguous(), bpq.to(dev)
        win = torch.zeros(C, 3, 3, 8)
        win[:, :, :, :lc] = to_f32(P["decoder.conv_in.weight"]).permute(0, 2, 3, 1).cpu()
        self.in_w, self.in_b = win.to(dev, bf16).contiguous(), to_f32(P["decoder.conv_in.bias"]).to(dev)
        leaves = [*self.mid_res0.parts(), *self.mid_res1.parts(), self.attn_norm, self.attn_out, self.norm_out, self.conv_out]
        for res, ups in self.up:
            for r in res:
                leaves += r.parts()
            if ups is not None:
                leaves.append(ups)
        for m in leaves:
            m.load(P, dev)
        a = "decoder.mid_block.attentions.0"
        self.qkv_w = torch.cat([linear_weight(P, f"{a}.{n}") for n in ("to_q", "to_k", "to_v")], 0).to(dev, bf16)
        self.qkv_b = torch.cat([linear_bias(P, f"{a}.{n}") for n in ("to_q", "to_k", "to_v")], 0).to(dev)
        self._scratch = {}
        return self

    def _mid_attention(self, x):
        """Attention(heads = 1, dim_head = C, residual_connection = True) via AttnProcessor (attention_processor.py:673-735)."""
        from .. import ops
        B, H, W, C = x.shape
        HW = H * W
        n = ops.groupnorm_nhwc(x, self.attn_norm.w, self.attn_norm.b, groups=self.config.norm_num_groups, eps=1e-6, silu=False)
        qkv = ops.linear(n.reshape(B, HW, C), self.qkv_w, self.qkv_b)  # [B, HW, 3C]
        o = torch.empty(B, HW, C, device=x.device, dtype=bf16)
        key = (HW, x.device)
        if key not in self._scratch:
            self._scratch[key] = (torch.empty(HW, HW, device=x.device, dtype=torch.float32),
                                  torch.empty(HW, HW, device=x.device, dtype=bf16))
        s_buf, p_buf = self._scratch[key]
        for b in range(B):
            q, k, v = qkv[b, :, :C], qkv[b, :, C:2 * C], qkv[b, :, 2 * C:]
            ops.linear(q, k, out_fp32=True, out=s_buf)                  # scores = q k^T, fp32 (upcast_softmax)
            ops.softmax_rows(s_buf, scale=C ** -0.5, out=p_buf)         # softmax(scores / sqrt(C)) -> bf16
            ops.linear(p_buf, v.t().contiguous(), out=o[b])             # P V (V transposed once: K-major operand)
        out = ops.linear(o, self.attn_out.w, self.attn_out.b, residual=x.reshape(B, HW, C))
        return out.reshape(B, H, W, C)

    def _decode(self, z_nchw):
        from .. import ops
        z = z_nchw.to(self.device)
        if z.dtype not in (torch.float32, bf16):
            z = z.float()
        x = ops.nchw_to_nhwc(z.contiguous())                     # [B, h, w, lc] bf16
        x = ops.conv3x3_small_cin(x, self.pq_w, self.pq_b)       # post_quant_conv (autoencoder_kl.py:293-294)
        h = ops.conv3x3_small_cin(x, self.in_w, self.in_b)       # decoder.conv_in (vae.py:229)
        h = self.mid_res0(h)
        h = self._mid_attention(h)
        h = self.mid_res1(h)
        for res, ups in self.up:
            for r in res:
                h = r(h)
            if ups is not None:
                h = ups.up2x(h)
        n = ops.groupnorm_nhwc(h, self.norm_out.w, self.norm_out.b, groups=self.config.norm_num_groups, eps=1e-6, silu=True)
        y = ops.conv3x3(n, self.conv_out.w, self.conv_out.b)
        return ops.nhwc_to_nchw(y, out_dtype=torch.float32)

    def decode(self, z, return_dict: bool = True, generator=None):
        """autoencoder_kl.py:302-325. z: latents ALREADY divided by config.scaling_factor (the pipeline does that, :911)."""
        if self.device is None:
            raise RuntimeError("load_state_dict() must be called before decode()")
        dec = self._decode(z)
        return DecoderOutput(sample=dec) if return_dict else (dec,)
