"""ORACLE (test infrastructure, not product code): CPU fp32 restatement of the reference's ControlNet
(ppdiffusers/models/controlnet.py: ControlNetConditioningEmbedding :71-113, ControlNetModel :116-882),
MultiControlNetModel (pipelines/controlnet/multicontrolnet.py) and the keep / guess-mode logic of the ControlNet
pipelines (pipelines/controlnet/pipeline_controlnet.py:1047-1100), built from oracle.unet's layer functions.

A ControlNet config is a UNet config (oracle.unet.UNET_CONFIGS) plus the optional keys `conditioning_channels`,
`conditioning_embedding_out_channels` and `controlnet_conditioning_channel_order`. Parameter names are the reference's
state-dict keys; conventions follow oracle.unet (Paddle Linear [in, out], NCHW).
"""
from typing import Dict, List, Sequence, Union

import torch
import torch.nn.functional as F

from . import unet as U

CONDITIONING_EMBEDDING_OUT_CHANNELS = (16, 32, 96, 256)  # ControlNetModel default (controlnet.py:224)
ENCODER_PREFIXES = ("conv_in.", "time_embedding.", "add_embedding.", "down_blocks.", "mid_block.")


def _cn(cfg, key, default):
    return cfg.get(key, default)


def _unet_cfg(cfg):
    """oracle.unet derives the encoder from down_block_types alone; give it an up path of the same length."""
    return {**cfg, "up_block_types": tuple("UpBlock2D" for _ in cfg["down_block_types"])}


def zero_conv_channels(cfg) -> List[int]:
    """Channels of controlnet_down_blocks.{k} (controlnet.py:369-410): conv_in output, then per down block one per
    resnet and one for the downsampler."""
    L = U.unet_layout(_unet_cfg(cfg))
    out = [cfg["block_out_channels"][0]]
    for d in L["down"]:
        out += [d["out_ch"]] * d["layers"]
        if d["downsample"]:
            out.append(d["out_ch"])
    return out


def controlnet_param_shapes(cfg) -> Dict[str, tuple]:
    S = {k: v for k, v in U.unet_param_shapes(_unet_cfg(cfg)).items() if k.startswith(ENCODER_PREFIXES)}
    ch = _cn(cfg, "conditioning_embedding_out_channels", CONDITIONING_EMBEDDING_OUT_CHANNELS)
    cc = _cn(cfg, "conditioning_channels", 3)

    def conv(name, i, o, k):
        S[name + ".weight"] = (o, i, k, k)
        S[name + ".bias"] = (o,)

    conv("controlnet_cond_embedding.conv_in", cc, ch[0], 3)
    for i in range(len(ch) - 1):
        conv(f"controlnet_cond_embedding.blocks.{2 * i}", ch[i], ch[i], 3)
        conv(f"controlnet_cond_embedding.blocks.{2 * i + 1}", ch[i], ch[i + 1], 3)
    conv("controlnet_cond_embedding.conv_out", ch[-1], cfg["block_out_channels"][0], 3)
    for k, c in enumerate(zero_conv_channels(cfg)):
        conv(f"controlnet_down_blocks.{k}", c, c, 1)
    conv("controlnet_mid_block", cfg["block_out_channels"][-1], cfg["block_out_channels"][-1], 1)
    return S


def zero_module_names(cfg) -> List[str]:
    """Parameters the reference initialises to zero (zero_module, controlnet.py:99-101, 371-417, 885-889)."""
    return [k for k in controlnet_param_shapes(cfg)
            if k.startswith(("controlnet_down_blocks.", "controlnet_mid_block.", "controlnet_cond_embedding.conv_out."))]


def from_unet_params(cfg, unet_P, P):
    """ControlNetModel.from_unet(load_weights_from_unet=True) (controlnet.py:509-518): conv_in, time_embedding,
    down_blocks and mid_block come from the UNet; everything else keeps the ControlNet's own values."""
    out = dict(P)
    for k in controlnet_param_shapes(cfg):
        if k.startswith(("conv_in.", "time_embedding.", "down_blocks.", "mid_block.")):
            out[k] = unet_P[k]
    return out


def conditioning_embedding(cfg, P, cond):
    """ControlNetConditioningEmbedding.forward (controlnet.py:103-113): conv_in, SiLU, (conv, SiLU) x 2(n-1), conv_out."""
    ch = _cn(cfg, "conditioning_embedding_out_channels", CONDITIONING_EMBEDDING_OUT_CHANNELS)
    e = F.silu(U.conv2d(cond, P, "controlnet_cond_embedding.conv_in"))
    for i in range(2 * (len(ch) - 1)):
        e = F.silu(U.conv2d(e, P, f"controlnet_cond_embedding.blocks.{i}", stride=1 + (i % 2)))
    return U.conv2d(e, P, "controlnet_cond_embedding.conv_out")


def guess_mode_scales(n_residuals: int, conditioning_scale: float) -> torch.Tensor:
    """controlnet.py:855-857: logspace(-1, 0, n + 1) (0.1 ... 1.0) times the conditioning scale, fp32."""
    return torch.logspace(-1, 0, n_residuals + 1, dtype=torch.float32) * conditioning_scale


def controlnet_forward(cfg, P, sample, timestep, encoder_hidden_states, controlnet_cond,
                       conditioning_scale: Union[float, Sequence[float]] = 1.0, added_cond_kwargs=None,
                       guess_mode=False, attention_mask=None):
    """ControlNetModel.forward (controlnet.py:670-882). Returns (down_block_res_samples list, mid_block_res_sample)."""
    L = U.unet_layout(_unet_cfg(cfg))
    order = _cn(cfg, "controlnet_conditioning_channel_order", "rgb")
    if order == "bgr":
        controlnet_cond = torch.flip(controlnet_cond, dims=[1])
    elif order != "rgb":
        raise ValueError(f"unknown `controlnet_conditioning_channel_order`: {order}")
    am = None
    if attention_mask is not None:  # :739-741
        am = ((1 - attention_mask.to(sample.dtype)) * -10000.0).unsqueeze(1)
    groups, eps = cfg["norm_num_groups"], cfg["norm_eps"]
    B = sample.shape[0]
    # 1. time (:743-805), as in oracle.unet.unet_forward
    t = torch.as_tensor(timestep)
    if t.ndim == 0:
        t = t[None]
    t = t.expand(B)
    t_emb = U.get_timestep_embedding(t, cfg["block_out_channels"][0], cfg["flip_sin_to_cos"], cfg["freq_shift"])
    emb = U.timestep_embedding_mlp(t_emb.to(sample.dtype), P, "time_embedding")
    if cfg["addition_embed_type"] == "text_time":
        text_embeds, time_ids = added_cond_kwargs["text_embeds"], added_cond_kwargs["time_ids"]
        time_embeds = U.get_timestep_embedding(time_ids.flatten(), cfg["addition_time_embed_dim"],
                                               cfg["flip_sin_to_cos"], cfg["freq_shift"])
        time_embeds = time_embeds.reshape(text_embeds.shape[0], -1)
        add_embeds = torch.cat([text_embeds, time_embeds], dim=-1).to(emb.dtype)
        emb = emb + U.timestep_embedding_mlp(add_embeds, P, "add_embedding")
    ctx = encoder_hidden_states
    # 2. pre-process (:807-811)
    h = U.conv2d(sample, P, "conv_in") + conditioning_embedding(cfg, P, controlnet_cond)
    # 3. down (:813-827); the ControlNet's resnets use output_scale_factor 1 (get_down_block's default)
    skips = [h]
    for i, d in enumerate(L["down"]):
        for j in range(d["layers"]):
            h = U.resnet_block(h, emb, P, f"down_blocks.{i}.resnets.{j}", groups, eps, 1.0)
            if d["type"] == "CrossAttnDownBlock2D":
                h = U.transformer_2d(h, ctx, P, f"down_blocks.{i}.attentions.{j}", d["heads"], d["tlayers"], groups,
                                     cfg["use_linear_projection"], None, am, None)
            skips.append(h)
        if d["downsample"]:
            h = U.conv2d(h, P, f"down_blocks.{i}.downsamplers.0.conv", stride=2, padding=1)
            skips.append(h)
    # 4. mid (:829-840)
    m = L["mid"]
    h = U.resnet_block(h, emb, P, "mid_block.resnets.0", groups, eps, 1.0)
    h = U.transformer_2d(h, ctx, P, "mid_block.attentions.0", m["heads"], m["tlayers"], groups,
                         cfg["use_linear_projection"], None, am, None)
    h = U.resnet_block(h, emb, P, "mid_block.resnets.1", groups, eps, 1.0)
    # 5. zero convs (:842-852)
    down = [U.conv2d(s, P, f"controlnet_down_blocks.{k}", padding=0) for k, s in enumerate(skips)]
    mid = U.conv2d(h, P, "controlnet_mid_block", padding=0)
    # 6. scaling (:854-869)
    if guess_mode:
        scales = guess_mode_scales(len(down), conditioning_scale)
        down = [s * sc for s, sc in zip(down, scales)]
        mid = mid * scales[-1]
    elif isinstance(conditioning_scale, (float, int)):
        down = [s * conditioning_scale for s in down]
        mid = mid * conditioning_scale
    else:
        down = [s * c for s, c in zip(down, conditioning_scale[:-1])]
        mid = mid * conditioning_scale[-1]
    return down, mid


def multi_controlnet_forward(cfgs, Ps, sample, timestep, encoder_hidden_states, controlnet_conds, conditioning_scales,
                             added_cond_kwargs=None, guess_mode=False):
    """MultiControlNetModel.forward (multicontrolnet.py:45-90): the residuals of all nets, summed."""
    down = mid = None
    for cfg, P, cond, scale in zip(cfgs, Ps, controlnet_conds, conditioning_scales):
        d, m = controlnet_forward(cfg, P, sample, timestep, encoder_hidden_states, cond, scale, added_cond_kwargs,
                                  guess_mode)
        if down is None:
            down, mid = d, m
        else:
            down = [a + b for a, b in zip(down, d)]
            mid = mid + m
    return down, mid


def controlnet_keep(n_steps: int, control_guidance_start: Sequence[float], control_guidance_end: Sequence[float],
                    multi: bool):
    """pipeline_controlnet.py:1047-1053: per step, 1.0 while i / n >= start and (i + 1) / n <= end, else 0.0; one
    float for a single ControlNetModel, one list for a MultiControlNetModel."""
    keep = []
    for i in range(n_steps):
        ks = [1.0 - float(i / n_steps < s or (i + 1) / n_steps > e)
              for s, e in zip(control_guidance_start, control_guidance_end)]
        keep.append(ks if multi else ks[0])
    return keep


def step_conditioning_scale(controlnet_conditioning_scale, keep):
    """pipeline_controlnet.py:1074-1080: the conditioning scale of one step."""
    if isinstance(keep, list):
        return [c * s for c, s in zip(controlnet_conditioning_scale, keep)]
    c = controlnet_conditioning_scale
    if isinstance(c, list):
        c = c[0]
    return c * keep


def controlnet_flops(cfg, B, H, W, L, image_hw):
    """2*MAC of one ControlNet forward, split like the reference's modules, for B samples at latent H x W, text length
    L and a control image of image_hw = (h, w) pixels. Keys: `encoder` (conv_in + down + mid, oracle.unet.unet_flops
    conventions), `zero_convs`, `cond_embedding` (once per image) and `cond_layers` (one dict per conditioning-embedding
    conv: cin, cout, stride, in_hw, flops, bytes = bf16 input + weights + output, read / written once)."""
    ucfg = _unet_cfg(cfg)
    Ly = U.unet_layout(ucfg)
    boc = cfg["block_out_channels"]
    ted = Ly["time_embed_dim"]
    # encoder: unet_flops with the up path, norm_out and conv_out removed = run the same accounting on the down half
    mac = 0

    def res(i, o, hw):
        return hw * (9 * i * o + 9 * o * o + (i * o if i != o else 0)) + ted * o

    def tr(c, ctx_dim, layers, hw):
        m = 2 * hw * c * c
        per = hw * (4 * c * c) + 2 * hw * hw * c
        per += hw * 2 * c * c + 2 * L * ctx_dim * c + 2 * hw * L * c
        per += hw * (c * 8 * c + 4 * c * c)
        return m + layers * per

    hw = H * W
    mac += hw * 9 * cfg["in_channels"] * boc[0]
    mac += boc[0] * ted + ted * ted
    if cfg["addition_embed_type"] == "text_time":
        mac += cfg["projection_class_embeddings_input_dim"] * ted + ted * ted
    zero = hw * boc[0] * boc[0]
    for d in Ly["down"]:
        for j in range(d["layers"]):
            mac += res(d["in_ch"] if j == 0 else d["out_ch"], d["out_ch"], hw)
            if d["type"] == "CrossAttnDownBlock2D":
                mac += tr(d["out_ch"], d["ctx_dim"], d["tlayers"], hw)
            zero += hw * d["out_ch"] ** 2
        if d["downsample"]:
            hw //= 4
            mac += hw * 9 * d["out_ch"] * d["out_ch"]
            zero += hw * d["out_ch"] ** 2
    m = Ly["mid"]
    mac += 2 * res(m["ch"], m["ch"], hw) + tr(m["ch"], m["ctx_dim"], m["tlayers"], hw)
    zero += hw * m["ch"] ** 2
    # conditioning embedding
    ch = _cn(cfg, "conditioning_embedding_out_channels", CONDITIONING_EMBEDDING_OUT_CHANNELS)
    convs = [(_cn(cfg, "conditioning_channels", 3), ch[0], 1)]
    for i in range(len(ch) - 1):
        convs += [(ch[i], ch[i], 1), (ch[i], ch[i + 1], 2)]
    convs.append((ch[-1], boc[0], 1))
    ih, iw = image_hw
    layers, emb = [], 0
    for cin, cout, s in convs:
        oh, ow = ih // s, iw // s
        f = 2 * B * oh * ow * 9 * cin * cout
        by = 2 * (B * ih * iw * cin + 9 * cin * cout + B * oh * ow * cout)
        layers.append(dict(cin=cin, cout=cout, stride=s, in_hw=(ih, iw), flops=f, bytes=by))
        emb += f
        ih, iw = oh, ow
    return dict(encoder=2 * mac * B, zero_convs=2 * zero * B, cond_embedding=emb, cond_layers=layers)
