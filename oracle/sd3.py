"""ORACLE (test infrastructure, not product code): CPU fp32 restatement of the reference's SD3 MMDiT denoiser,
SD3Transformer2DModel.forward (ppdiffusers/models/transformer_sd3.py:279-365) with JointTransformerBlock
(attention.py:96-214), AdaLayerNormZero / AdaLayerNormContinuous (normalization.py:50-86,165-202),
JointAttnProcessor2_5 (attention_processor.py:909-985), PatchEmbed (embeddings.py:122-247) and
CombinedTimestepTextProjEmbeddings (embeddings.py:530-546).

PARITY UNPINNED: the reference's SD3 test asserts shapes/determinism only
(ppdiffusers/tests/models/test_models_transformer_sd3.py:25-80); no reference golden value exists for this model.
Conventions as in oracle/unet.py (Paddle Linear weight [in, out]; NCHW).
"""
import math
from typing import Dict

import numpy as np
import torch
import torch.nn.functional as F

from .unet import get_timestep_embedding, init_params, linear  # noqa: F401

Params = Dict[str, torch.Tensor]

SD3_CONFIGS = {
    # stabilityai/stable-diffusion-3-medium transformer/config.json (the reference loads it by name,
    # ppdiffusers/deploy/sd3/text_to_image_generation-stable_diffusion_3.py:84-87)
    "sd3_medium": dict(sample_size=128, patch_size=2, in_channels=16, num_layers=24, attention_head_dim=64,
                       num_attention_heads=24, joint_attention_dim=4096, caption_projection_dim=1536,
                       pooled_projection_dim=2048, out_channels=16, pos_embed_max_size=192),
    # the reference's unit-test model (tests/models/test_models_transformer_sd3.py:49-62) has inner dim 32 with
    # 8-wide heads; `tiny` keeps the structure with kernel-friendly 64-wide heads
    "ref_tiny": dict(sample_size=32, patch_size=1, in_channels=4, num_layers=1, attention_head_dim=8,
                     num_attention_heads=4, joint_attention_dim=32, caption_projection_dim=32,
                     pooled_projection_dim=64, out_channels=4, pos_embed_max_size=96),
    "tiny": dict(sample_size=32, patch_size=2, in_channels=16, num_layers=3, attention_head_dim=64,
                 num_attention_heads=2, joint_attention_dim=96, caption_projection_dim=128,
                 pooled_projection_dim=64, out_channels=16, pos_embed_max_size=48),
}


def get_1d_sincos_pos_embed_from_grid(embed_dim, pos):  # embeddings.py:100-119
    omega = np.arange(embed_dim // 2, dtype=np.float64)
    omega /= embed_dim / 2.0
    omega = 1.0 / 10000 ** omega
    out = np.einsum("m,d->md", pos.reshape(-1), omega)
    return np.concatenate([np.sin(out), np.cos(out)], axis=1)


def get_2d_sincos_pos_embed(embed_dim, grid_size, interpolation_scale=1.0, base_size=16):  # embeddings.py:66-98
    if isinstance(grid_size, int):
        grid_size = (grid_size, grid_size)
    grid_h = np.arange(grid_size[0], dtype=np.float32) / (grid_size[0] / base_size) / interpolation_scale
    grid_w = np.arange(grid_size[1], dtype=np.float32) / (grid_size[1] / base_size) / interpolation_scale
    grid = np.stack(np.meshgrid(grid_w, grid_h), axis=0).reshape([2, 1, grid_size[1], grid_size[0]])
    emb_h = get_1d_sincos_pos_embed_from_grid(embed_dim // 2, grid[0])
    emb_w = get_1d_sincos_pos_embed_from_grid(embed_dim // 2, grid[1])
    return np.concatenate([emb_h, emb_w], axis=1)


def sd3_param_shapes(cfg) -> Dict[str, tuple]:
    D = cfg["num_attention_heads"] * cfg["attention_head_dim"]
    p = cfg["patch_size"]
    S: Dict[str, tuple] = {}

    def lin(name, i, o):
        S[name + ".weight"], S[name + ".bias"] = (i, o), (o,)

    S["pos_embed.proj.weight"], S["pos_embed.proj.bias"] = (D, cfg["in_channels"], p, p), (D,)
    S["pos_embed.pos_embed"] = (1, cfg["pos_embed_max_size"] ** 2, D)
    lin("time_text_embed.timestep_embedder.linear_1", 256, D), lin("time_text_embed.timestep_embedder.linear_2", D, D)
    lin("time_text_embed.text_embedder.linear_1", cfg["pooled_projection_dim"], D)
    lin("time_text_embed.text_embedder.linear_2", D, D)
    lin("context_embedder", cfg["joint_attention_dim"], cfg["caption_projection_dim"])
    for i in range(cfg["num_layers"]):
        b = f"transformer_blocks.{i}"
        last = i == cfg["num_layers"] - 1
        lin(b + ".norm1.linear", D, 6 * D)
        lin(b + ".norm1_context.linear", D, 2 * D if last else 6 * D)
        if last:  # AdaLayerNormContinuous(elementwise_affine=False, bias=True): nn.LayerNorm has a bias, no weight
            S[b + ".norm1_context.norm.bias"] = (D,)  # (normalization.py:184, SURVEY.md A5)
        for n in ("to_q", "to_k", "to_v", "add_q_proj", "add_k_proj", "add_v_proj", "to_out.0"):
            lin(f"{b}.attn.{n}", D, D)
        lin(b + ".ff.net.0.proj", D, 4 * D), lin(b + ".ff.net.2", 4 * D, D)
        if not last:
            lin(b + ".attn.to_add_out", D, D)
            lin(b + ".ff_context.net.0.proj", D, 4 * D), lin(b + ".ff_context.net.2", 4 * D, D)
    lin("norm_out.linear", D, 2 * D)
    S["norm_out.norm.bias"] = (D,)
    lin("proj_out", D, p * p * cfg["out_channels"])
    return S


def init_sd3_params(cfg, seed=1) -> Params:
    shapes = sd3_param_shapes(cfg)
    pe_shape = shapes.pop("pos_embed.pos_embed")
    P = init_params(shapes, seed)
    D = pe_shape[-1]
    pe = get_2d_sincos_pos_embed(D, cfg["pos_embed_max_size"], base_size=cfg["sample_size"] // cfg["patch_size"])
    P["pos_embed.pos_embed"] = torch.from_numpy(pe).float().unsqueeze(0).to(torch.bfloat16).float()
    return P


def _ln(x, eps=1e-6):
    return F.layer_norm(x, (x.shape[-1],), None, None, eps)


def _ff(x, P, p):  # FeedForward(activation_fn="gelu-approximate"): Linear -> GELU(tanh) -> Linear (attention.py:145)
    return linear(F.gelu(linear(x, P, p + ".net.0.proj"), approximate="tanh"), P, p + ".net.2")


def joint_attention(x, c, P, p, heads, context_pre_only):
    """JointAttnProcessor2_5.__call__, attention_processor.py:916-983 (sample tokens first, then context)."""
    q = torch.cat([linear(x, P, p + ".to_q"), linear(c, P, p + ".add_q_proj")], 1)
    k = torch.cat([linear(x, P, p + ".to_k"), linear(c, P, p + ".add_k_proj")], 1)
    v = torch.cat([linear(x, P, p + ".to_v"), linear(c, P, p + ".add_v_proj")], 1)
    B, S, D = q.shape
    d = D // heads
    sp = lambda t: t.reshape(B, S, heads, d).permute(0, 2, 1, 3)
    s = (sp(q) @ sp(k).transpose(-1, -2)) * (d ** -0.5)  # paddle_patch.py:445-461, scale = head_dim^-0.5
    o = (torch.softmax(s, -1) @ sp(v)).permute(0, 2, 1, 3).reshape(B, S, D)
    xo, co = o[:, : x.shape[1]], o[:, x.shape[1]:]
    xo = linear(xo, P, p + ".to_out.0")
    if not context_pre_only:
        co = linear(co, P, p + ".to_add_out")
    return xo, co


def joint_block(x, c, temb, P, p, heads, last):
    """JointTransformerBlock.forward, attention.py:164-214."""
    e = linear(F.silu(temb), P, p + ".norm1.linear")  # AdaLayerNormZero, normalization.py:72-86
    shift_msa, scale_msa, gate_msa, shift_mlp, scale_mlp, gate_mlp = e.chunk(6, dim=1)
    nx = _ln(x) * (1 + scale_msa[:, None]) + shift_msa[:, None]
    ec = linear(F.silu(temb), P, p + ".norm1_context.linear")
    if last:  # AdaLayerNormContinuous: chunk order is (scale, shift), normalization.py:193
        c_scale, c_shift = ec.chunk(2, dim=1)
        nc = (_ln(c) + P[p + ".norm1_context.norm.bias"]) * (1 + c_scale)[:, None, :] + c_shift[:, None, :]
    else:
        c_shift_msa, c_scale_msa, c_gate_msa, c_shift_mlp, c_scale_mlp, c_gate_mlp = ec.chunk(6, dim=1)
        nc = _ln(c) * (1 + c_scale_msa[:, None]) + c_shift_msa[:, None]
    ax, ac = joint_attention(nx, nc, P, p + ".attn", heads, last)
    x = x + gate_msa.unsqueeze(1) * ax
    nx = _ln(x) * (1 + scale_mlp[:, None]) + shift_mlp[:, None]
    x = x + gate_mlp.unsqueeze(1) * _ff(nx, P, p + ".ff")
    if last:
        return None, x
    c = c + c_gate_msa.unsqueeze(1) * ac
    nc = _ln(c) * (1 + c_scale_mlp[:, None]) + c_shift_mlp[:, None]
    c = c + c_gate_mlp.unsqueeze(1) * _ff(nc, P, p + ".ff_context")
    return c, x


def sd3_embed(cfg, P: Params, hidden_states, encoder_hidden_states, pooled_projections, timestep):
    """The part of SD3Transformer2DModel.forward before the blocks (transformer_sd3.py:318-324): returns the patch
    embedding x [B, h*w, D], the context stream c [B, L, D] and temb [B, D]."""
    ps = cfg["patch_size"]
    B, _, H, W = hidden_states.shape
    # PatchEmbed.forward, embeddings.py:212-247 (conv p x p stride p, flatten, + cropped sincos pos embed)
    x = F.conv2d(hidden_states, P["pos_embed.proj.weight"], P["pos_embed.proj.bias"], stride=ps)
    x = x.flatten(2).transpose(1, 2)
    x = x + sd3_pos_embed(cfg, P, H // ps, W // ps)
    # CombinedTimestepTextProjEmbeddings, embeddings.py:530-546
    t = torch.as_tensor(timestep, dtype=torch.float32).reshape(-1).expand(B)
    t_proj = get_timestep_embedding(t, 256, flip_sin_to_cos=True, downscale_freq_shift=0)
    t_emb = linear(F.silu(linear(t_proj, P, "time_text_embed.timestep_embedder.linear_1")), P,
                   "time_text_embed.timestep_embedder.linear_2")
    p_emb = linear(F.silu(linear(pooled_projections, P, "time_text_embed.text_embedder.linear_1")), P,
                   "time_text_embed.text_embedder.linear_2")
    temb = t_emb + p_emb
    c = linear(encoder_hidden_states, P, "context_embedder")
    return x, c, temb


def sd3_pos_embed(cfg, P: Params, h, w):
    """PatchEmbed.cropped_pos_embed, embeddings.py:186-210: the centred h x w crop of the max-size table, [1, h*w, D]."""
    mx = cfg["pos_embed_max_size"]
    top, left = (mx - h) // 2, (mx - w) // 2
    return P["pos_embed.pos_embed"].reshape(1, mx, mx, -1)[:, top:top + h, left:left + w, :].reshape(1, h * w, -1)


def sd3_final(cfg, P: Params, x, temb, h, w):
    """norm_out (AdaLayerNormContinuous, (scale, shift)), proj_out and the unpatchify of transformer_sd3.py:345-356."""
    ps, oc = cfg["patch_size"], cfg["out_channels"]
    B = x.shape[0]
    e = linear(F.silu(temb), P, "norm_out.linear")
    scale, shift = e.chunk(2, dim=1)
    x = (_ln(x) + P["norm_out.norm.bias"]) * (1 + scale)[:, None, :] + shift[:, None, :]
    x = linear(x, P, "proj_out")
    x = x.reshape(B, h, w, ps, ps, oc).permute(0, 5, 1, 3, 2, 4)
    return x.reshape(B, oc, h * ps, w * ps)


def sd3_forward(cfg, P: Params, hidden_states, encoder_hidden_states, pooled_projections, timestep):
    """SD3Transformer2DModel.forward, transformer_sd3.py:279-365. hidden_states [B,16,H,W]; timestep [B] float."""
    ps, heads = cfg["patch_size"], cfg["num_attention_heads"]
    x, c, temb = sd3_embed(cfg, P, hidden_states, encoder_hidden_states, pooled_projections, timestep)
    for i in range(cfg["num_layers"]):
        c, x = joint_block(x, c, temb, P, f"transformer_blocks.{i}", heads, i == cfg["num_layers"] - 1)
    return sd3_final(cfg, P, x, temb, hidden_states.shape[2] // ps, hidden_states.shape[3] // ps)


def sd3_flops(cfg, B, H, W, L):
    D = cfg["num_attention_heads"] * cfg["attention_head_dim"]
    ps = cfg["patch_size"]
    n = (H // ps) * (W // ps)
    mac = n * cfg["in_channels"] * ps * ps * D + 256 * D + D * D + cfg["pooled_projection_dim"] * D + D * D
    mac += L * cfg["joint_attention_dim"] * D
    for i in range(cfg["num_layers"]):
        last = i == cfg["num_layers"] - 1
        mac += D * 6 * D + D * (2 * D if last else 6 * D)
        mac += (n + L) * 3 * D * D + 2 * (n + L) ** 2 * D + n * D * D + n * 8 * D * D
        if not last:
            mac += L * D * D + L * 8 * D * D
    mac += D * 2 * D + n * D * ps * ps * cfg["out_channels"]
    return 2 * mac * B
