"""ORACLE (test infrastructure, not product code): CPU fp32 restatement of AutoencoderKL.decode — the exit of the denoising
loop (pipelines/stable_diffusion/pipeline_stable_diffusion.py:910-917) — ppdiffusers/ppdiffusers/models/
autoencoder_kl.py:288-325 (_decode / decode: post_quant_conv then Decoder), vae.py:182-282 (Decoder: conv_in ->
UNetMidBlock2D [resnet, one-head attention over H*W tokens with GroupNorm / residual, resnet] -> UpDecoderBlock2D x N
[layers_per_block + 1 resnets, nearest x2 + conv3x3] -> GroupNorm -> SiLU -> conv_out), unet_2d_blocks.py:529-660
(UNetMidBlock2D), :2482-2580 (UpDecoderBlock2D), resnet.py:587-808 (ResnetBlock2D with temb = None),
attention_processor.py:673-735 (AttnProcessor: group_norm, q/k/v, softmax, to_out, residual_connection).

parity unpinned: the reference's VAE tests need Paddle's RNG / downloaded weights; no external implementation (diffusers)
is installed here to cross-check against. Guarded by shape / parameter-count checks in tests.
"""
import math
from typing import Dict

import torch
import torch.nn.functional as F

Params = Dict[str, torch.Tensor]

VAE_CONFIGS = {
    # stabilityai sd-vae / sdxl-vae decoder
    "sd_vae": dict(latent_channels=4, out_channels=3, block_out_channels=(128, 256, 512, 512), layers_per_block=2,
                   norm_num_groups=32, scaling_factor=0.18215),
    "sdxl_vae": dict(latent_channels=4, out_channels=3, block_out_channels=(128, 256, 512, 512), layers_per_block=2,
                     norm_num_groups=32, scaling_factor=0.13025),
    "tiny": dict(latent_channels=4, out_channels=3, block_out_channels=(64, 128), layers_per_block=1, norm_num_groups=16,
                 scaling_factor=0.18215),
}


def vae_decoder_param_shapes(cfg) -> Dict[str, tuple]:
    boc, L, lc = cfg["block_out_channels"], cfg["layers_per_block"], cfg["latent_channels"]
    S = {"post_quant_conv.weight": (lc, lc, 1, 1), "post_quant_conv.bias": (lc,),
         "decoder.conv_in.weight": (boc[-1], lc, 3, 3), "decoder.conv_in.bias": (boc[-1],)}

    def resnet(p, i, o):
        S[p + ".norm1.weight"], S[p + ".norm1.bias"] = (i,), (i,)
        S[p + ".conv1.weight"], S[p + ".conv1.bias"] = (o, i, 3, 3), (o,)
        S[p + ".norm2.weight"], S[p + ".norm2.bias"] = (o,), (o,)
        S[p + ".conv2.weight"], S[p + ".conv2.bias"] = (o, o, 3, 3), (o,)
        if i != o:
            S[p + ".conv_shortcut.weight"], S[p + ".conv_shortcut.bias"] = (o, i, 1, 1), (o,)

    C = boc[-1]
    resnet("decoder.mid_block.resnets.0", C, C)
    resnet("decoder.mid_block.resnets.1", C, C)
    a = "decoder.mid_block.attentions.0"
    S[a + ".group_norm.weight"], S[a + ".group_norm.bias"] = (C,), (C,)
    for n in ("to_q", "to_k", "to_v", "to_out.0"):
        S[f"{a}.{n}.weight"], S[f"{a}.{n}.bias"] = (C, C), (C,)
    rev = list(reversed(boc))
    out = rev[0]
    for i in range(len(boc)):
        prev, out = out, rev[i]
        for j in range(L + 1):
            resnet(f"decoder.up_blocks.{i}.resnets.{j}", prev if j == 0 else out, out)
        if i != len(boc) - 1:
            S[f"decoder.up_blocks.{i}.upsamplers.0.conv.weight"] = (out, out, 3, 3)
            S[f"decoder.up_blocks.{i}.upsamplers.0.conv.bias"] = (out,)
    S["decoder.conv_norm_out.weight"], S["decoder.conv_norm_out.bias"] = (boc[0],), (boc[0],)
    S["decoder.conv_out.weight"], S["decoder.conv_out.bias"] = (cfg["out_channels"], boc[0], 3, 3), (cfg["out_channels"],)
    return S


def vae_decoder_layout(cfg, B, h, w):
    """Every kernel call of AutoencoderKL.decode on a [B, latent_channels, h, w] latent, in execution order, as dicts
    with keys name (the parameter prefix), op, B, H, W (the spatial size the op reads), cin, cout, groups and, for
    conv3x3, residual (the resnet's conv2 adds the block input or its shortcut). op is one of small_cin (post_quant_conv,
    conv_in), groupnorm (silu: whether SiLU follows), conv3x3, shortcut (the 1x1 GEMM), attention (the one-head mid
    attention: cin = cout = head width) and up2x (nearest 2x + conv3x3)."""
    boc, L, lc, G = cfg["block_out_channels"], cfg["layers_per_block"], cfg["latent_channels"], cfg["norm_num_groups"]
    sites = []

    def site(name, op, H, W, cin, cout, **kw):
        sites.append(dict(name=name, op=op, B=B, H=H, W=W, cin=cin, cout=cout, groups=G, **kw))

    def resnet(p, H, W, i, o):
        site(p + ".norm1", "groupnorm", H, W, i, i, silu=True)
        site(p + ".conv1", "conv3x3", H, W, i, o, residual=False)
        site(p + ".norm2", "groupnorm", H, W, o, o, silu=True)
        if i != o:
            site(p + ".conv_shortcut", "shortcut", H, W, i, o)
        site(p + ".conv2", "conv3x3", H, W, o, o, residual=True)

    C = boc[-1]
    site("post_quant_conv", "small_cin", h, w, lc, lc)
    site("decoder.conv_in", "small_cin", h, w, lc, C)
    resnet("decoder.mid_block.resnets.0", h, w, C, C)
    site("decoder.mid_block.attentions.0.group_norm", "groupnorm", h, w, C, C, silu=False)
    site("decoder.mid_block.attentions.0", "attention", h, w, C, C)
    resnet("decoder.mid_block.resnets.1", h, w, C, C)
    rev = list(reversed(boc))
    out, H, W = rev[0], h, w
    for i in range(len(boc)):
        prev, out = out, rev[i]
        for j in range(L + 1):
            resnet(f"decoder.up_blocks.{i}.resnets.{j}", H, W, prev if j == 0 else out, out)
        if i != len(boc) - 1:
            site(f"decoder.up_blocks.{i}.upsamplers.0.conv", "up2x", H, W, out, out)
            H, W = 2 * H, 2 * W
    site("decoder.conv_norm_out", "groupnorm", H, W, boc[0], boc[0], silu=True)
    site("decoder.conv_out", "conv3x3", H, W, boc[0], cfg["out_channels"], residual=False)
    return sites


def init_vae_params(cfg, seed=1) -> Params:
    g = torch.Generator().manual_seed(seed)
    P = {}
    shapes = vae_decoder_param_shapes(cfg)
    for name in sorted(shapes):
        shp = shapes[name]
        if name.endswith(".weight") and len(shp) >= 2:
            fan_in = shp[0] if len(shp) == 2 else math.prod(shp[1:])
            t = (torch.rand(shp, generator=g) * 2 - 1) / math.sqrt(fan_in)
        elif name.endswith(".weight"):
            t = 1.0 + 0.1 * torch.randn(shp, generator=g)
        else:
            t = 0.05 * torch.randn(shp, generator=g)
        P[name] = t.to(torch.bfloat16).float()
    return P


def _resnet(x, P, p, groups, eps=1e-6):
    """ResnetBlock2D.forward with temb None (resnet.py:728-808), output_scale_factor 1."""
    h = F.conv2d(F.silu(F.group_norm(x, groups, P[p + ".norm1.weight"], P[p + ".norm1.bias"], eps)),
                 P[p + ".conv1.weight"], P[p + ".conv1.bias"], padding=1)
    h = F.conv2d(F.silu(F.group_norm(h, groups, P[p + ".norm2.weight"], P[p + ".norm2.bias"], eps)),
                 P[p + ".conv2.weight"], P[p + ".conv2.bias"], padding=1)
    if (p + ".conv_shortcut.weight") in P:
        x = F.conv2d(x, P[p + ".conv_shortcut.weight"], P[p + ".conv_shortcut.bias"])
    return x + h


def _mid_attention(x, P, p, groups, eps=1e-6):
    """Attention(heads = 1, dim_head = C, residual_connection, norm_num_groups) through AttnProcessor
    (attention_processor.py:673-735): [B,C,H,W] -> tokens, group_norm on the token tensor, softmax(q k^T / sqrt(C)) v."""
    B, C, H, W = x.shape
    res = x
    h = x.reshape(B, C, H * W)
    h = F.group_norm(h, groups, P[p + ".group_norm.weight"], P[p + ".group_norm.bias"], eps).transpose(1, 2)
    q = h @ P[p + ".to_q.weight"] + P[p + ".to_q.bias"]
    k = h @ P[p + ".to_k.weight"] + P[p + ".to_k.bias"]
    v = h @ P[p + ".to_v.weight"] + P[p + ".to_v.bias"]
    w = torch.softmax((q @ k.transpose(1, 2)) * C ** -0.5, -1)
    o = (w @ v) @ P[p + ".to_out.0.weight"] + P[p + ".to_out.0.bias"]
    return o.transpose(1, 2).reshape(B, C, H, W) + res  # residual_connection; rescale_output_factor = 1


def vae_decode(cfg, P: Params, z):
    """AutoencoderKL._decode (autoencoder_kl.py:288-300): z [B, 4, h, w] -> image [B, 3, 8h, 8w] (4 levels)."""
    g = cfg["norm_num_groups"]
    boc, L = cfg["block_out_channels"], cfg["layers_per_block"]
    z = F.conv2d(z, P["post_quant_conv.weight"], P["post_quant_conv.bias"])
    h = F.conv2d(z, P["decoder.conv_in.weight"], P["decoder.conv_in.bias"], padding=1)
    h = _resnet(h, P, "decoder.mid_block.resnets.0", g)
    h = _mid_attention(h, P, "decoder.mid_block.attentions.0", g)
    h = _resnet(h, P, "decoder.mid_block.resnets.1", g)
    for i in range(len(boc)):
        for j in range(L + 1):
            h = _resnet(h, P, f"decoder.up_blocks.{i}.resnets.{j}", g)
        if i != len(boc) - 1:  # Upsample2D: nearest x2 + conv3x3 (resnet.py:169-218)
            h = F.interpolate(h, scale_factor=2.0, mode="nearest")
            h = F.conv2d(h, P[f"decoder.up_blocks.{i}.upsamplers.0.conv.weight"], P[f"decoder.up_blocks.{i}.upsamplers.0.conv.bias"], padding=1)
    h = F.silu(F.group_norm(h, g, P["decoder.conv_norm_out.weight"], P["decoder.conv_norm_out.bias"], 1e-6))
    return F.conv2d(h, P["decoder.conv_out.weight"], P["decoder.conv_out.bias"], padding=1)


def vae_decode_flops(cfg, h, w):
    """2*MAC of one decode (convs + mid attention)."""
    boc, L, lc = cfg["block_out_channels"], cfg["layers_per_block"], cfg["latent_channels"]
    C = boc[-1]
    hw = h * w
    mac = hw * (lc * lc + 9 * lc * C) + 2 * hw * 18 * C * C + hw * 4 * C * C + 2 * hw * hw * C
    rev = list(reversed(boc))
    out = rev[0]
    for i in range(len(boc)):
        prev, out = out, rev[i]
        for j in range(L + 1):
            ci = prev if j == 0 else out
            mac += hw * (9 * ci * out + 9 * out * out + (ci * out if ci != out else 0))
        if i != len(boc) - 1:
            hw *= 4
            mac += hw * 9 * out * out
    mac += hw * 9 * boc[0] * cfg["out_channels"]
    return 2 * mac
