"""ORACLE (test infrastructure, not product code): CPU fp32 restatement of Open-Sora's STDiT2 video denoiser,
ppdiffusers/examples/Open-Sora/models/stdit/stdit2.py (STDiT2Block.forward :119-191, STDiT2.forward :334-448,
unpatchify :450-474) with layers/blocks.py (Attention :167-241, MultiHeadCrossAttention :257-331, t2i_modulate :85,
LlamaRMSNorm :46-68, PatchEmbed3D :94-164, T2IFinalLayer :334-392, SizeEmbedder :395-428, CaptionEmbedder :431-484,
PositionEmbedding2D :487-545, rotary embedding :566-720) and TimestepEmbedder (ppdiffusers/models/dit_llama.py:54-89).
Inference path only (x_mask = None, no dropout).

PARITY UNPINNED: the reference has no test for STDiT2 (SURVEY.md §8c). Paddle Linear weights are [in, out].
"""
import math
from typing import Dict

import torch
import torch.nn.functional as F

from .unet import init_params, linear

Params = Dict[str, torch.Tensor]

STDIT2_CONFIGS = {
    # hpcai-tech/OpenSora-STDiT-v2-stage3 (STDiT2Config defaults, stdit2.py:198-238, + qk_norm of the released model)
    "stdit2_xl": dict(input_sq_size=32, in_channels=4, patch_size=(1, 2, 2), hidden_size=1152, depth=28, num_heads=16,
                      mlp_ratio=4.0, pred_sigma=True, caption_channels=4096, model_max_length=120, qk_norm=True),
    "tiny": dict(input_sq_size=32, in_channels=4, patch_size=(1, 2, 2), hidden_size=144, depth=2, num_heads=2,
                 mlp_ratio=4.0, pred_sigma=True, caption_channels=64, model_max_length=12, qk_norm=True),
}


def stdit2_param_shapes(cfg) -> Dict[str, tuple]:
    D, L = cfg["hidden_size"], cfg["depth"]
    hd = D // cfg["num_heads"]
    pt, ph, pw = cfg["patch_size"]
    out_ch = cfg["in_channels"] * (2 if cfg["pred_sigma"] else 1)
    hidden = int(D * cfg["mlp_ratio"])
    S: Dict[str, tuple] = {}

    def lin(name, i, o):
        S[name + ".weight"], S[name + ".bias"] = (i, o), (o,)

    S["x_embedder.proj.weight"], S["x_embedder.proj.bias"] = (D, cfg["in_channels"], pt, ph, pw), (D,)
    lin("t_embedder.mlp.0", 256, D), lin("t_embedder.mlp.2", D, D)
    lin("t_block.1", D, 6 * D), lin("t_block_temp.1", D, 3 * D)
    lin("y_embedder.y_proj.fc1", cfg["caption_channels"], D), lin("y_embedder.y_proj.fc2", D, D)
    for name, d in (("csize_embedder", D // 3), ("ar_embedder", D // 3), ("fl_embedder", D), ("fps_embedder", D)):
        lin(name + ".mlp.0", 256, d), lin(name + ".mlp.2", d, d)
    for i in range(L):
        b = f"blocks.{i}"
        S[b + ".scale_shift_table"], S[b + ".scale_shift_table_temporal"] = (6, D), (3, D)
        for a in ("attn", "attn_temp"):
            lin(f"{b}.{a}.qkv", D, 3 * D), lin(f"{b}.{a}.proj", D, D)
            if cfg["qk_norm"]:
                S[f"{b}.{a}.q_norm.weight"], S[f"{b}.{a}.k_norm.weight"] = (hd,), (hd,)
        lin(b + ".cross_attn.q_linear", D, D), lin(b + ".cross_attn.kv_linear", D, 2 * D), lin(b + ".cross_attn.proj", D, D)
        lin(b + ".mlp.fc1", D, hidden), lin(b + ".mlp.fc2", hidden, D)
    S["final_layer.scale_shift_table"] = (2, D)
    lin("final_layer.linear", D, pt * ph * pw * out_ch)
    return S


def init_stdit2_params(cfg, seed=1) -> Params:
    shapes = stdit2_param_shapes(cfg)
    tables = {k: v for k, v in shapes.items() if "scale_shift_table" in k}
    conv = shapes["x_embedder.proj.weight"]
    P = init_params({k: v for k, v in shapes.items() if k not in tables and k != "x_embedder.proj.weight"}, seed)
    g = torch.Generator().manual_seed(seed + 7)
    D = cfg["hidden_size"]
    for k, shp in tables.items():  # randn / sqrt(hidden) like the reference initialiser (stdit2.py:66-74)
        P[k] = (torch.randn(shp, generator=g) / D ** 0.5).to(torch.bfloat16).float()
    fan = conv[1] * conv[2] * conv[3] * conv[4]
    P["x_embedder.proj.weight"] = ((torch.rand(conv, generator=g) * 2 - 1) / math.sqrt(fan)).to(torch.bfloat16).float()
    return P


def timestep_embedding(t, dim, max_period=10000):  # dit_llama.py:68-84: [cos | sin]
    half = dim // 2
    freqs = torch.exp(-math.log(max_period) * torch.arange(half, dtype=torch.float32) / half)
    args = t[:, None].float() * freqs[None]
    return torch.cat([torch.cos(args), torch.sin(args)], dim=-1)


def _embedder(P, name, s):  # TimestepEmbedder.forward / SizeEmbedder.mlp
    return linear(F.silu(linear(timestep_embedding(s, 256), P, name + ".mlp.0")), P, name + ".mlp.2")


def size_embedder(P, name, s, bs):  # SizeEmbedder.forward, blocks.py:409-423
    if s.ndim == 1:
        s = s[:, None]
    if s.shape[0] != bs:
        s = s.repeat(bs // s.shape[0], 1)
    b, dims = s.shape
    emb = _embedder(P, name, s.reshape(-1))
    return emb.reshape(b, dims * emb.shape[-1])


def position_embedding_2d(dim, h, w, scale, base_size):
    """PositionEmbedding2D._get_cached_emb, blocks.py:503-527, literally (including the swapped meshgrid naming)."""
    half = dim // 2
    inv_freq = 1.0 / 10000 ** (torch.arange(0, half, 2, dtype=torch.float32) / half)
    grid_h = torch.arange(h, dtype=torch.float32) / scale
    grid_w = torch.arange(w, dtype=torch.float32) / scale
    if base_size is not None:
        grid_h = grid_h * (base_size / h)
        grid_w = grid_w * (base_size / w)
    grid_h, grid_w = torch.meshgrid(grid_w, grid_h, indexing="ij")
    grid_h, grid_w = grid_h.t().reshape(-1), grid_w.t().reshape(-1)

    def sincos(t):
        out = torch.einsum("i,d->id", t, inv_freq)
        return torch.cat([torch.sin(out), torch.cos(out)], dim=-1)
    return torch.cat([sincos(grid_h), sincos(grid_w)], dim=-1).unsqueeze(0)


def rotate_half_interleaved(x):  # blocks.py:566-571 (pairs (2i, 2i+1))
    x = x.reshape(*x.shape[:-1], -1, 2)
    x1, x2 = x.unbind(-1)
    return torch.stack((-x2, x1), dim=-1).flatten(-2)


def rope_temporal(t, head_dim, theta=10000.0):
    """RotaryEmbedding(dim=head_dim).rotate_queries_or_keys on [..., T, head_dim] (blocks.py:606-700)."""
    T = t.shape[-2]
    freqs = 1.0 / theta ** (torch.arange(0, head_dim, 2)[: head_dim // 2].float() / head_dim)
    f = torch.einsum("n,f->nf", torch.arange(T, dtype=torch.float32), freqs).repeat_interleave(2, dim=-1)
    return t * f.cos() + rotate_half_interleaved(t) * f.sin()


def rms_norm(x, w, eps=1e-6):  # LlamaRMSNorm, blocks.py:62-68
    return w * (x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps))


def attention(x, P, p, heads, qk_norm, rope):
    """Attention.forward, blocks.py:200-241: x [B', N, C]."""
    Bq, N, C = x.shape
    hd = C // heads
    qkv = linear(x, P, p + ".qkv").reshape(Bq, N, 3, heads, hd).permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0], qkv[1], qkv[2]
    if rope:
        q, k = rope_temporal(q, hd), rope_temporal(k, hd)
    if qk_norm:
        q, k = rms_norm(q, P[p + ".q_norm.weight"]), rms_norm(k, P[p + ".k_norm.weight"])
    a = torch.softmax(q @ k.transpose(-1, -2) * hd ** -0.5, dim=-1) @ v
    return linear(a.transpose(1, 2).reshape(Bq, N, C), P, p + ".proj")


def cross_attention(x, cond, y_lens, P, p, heads):
    """MultiHeadCrossAttention.forward, blocks.py:275-331: cond packed [1, sum(y_lens), C], block-diagonal bias."""
    B, N, C = x.shape
    hd = C // heads
    q = linear(x, P, p + ".q_linear").reshape(1, -1, heads, hd)
    kv = linear(cond, P, p + ".kv_linear").reshape(1, -1, 2, heads, hd)
    k, v = kv.unbind(2)
    bias = torch.full((B * N, k.shape[1]), float("-inf"))
    ks = 0
    for i, L in enumerate(y_lens):
        bias[i * N:(i + 1) * N, ks:ks + L] = 0.0
        ks += L
    q, k, v = q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2)
    a = torch.softmax((q * hd ** -0.5) @ k.transpose(-1, -2) + bias, dim=-1) @ v
    return linear(a.transpose(1, 2).reshape(B, -1, C), P, p + ".proj")


def stdit2_block(x, y, t_mlp, t_tmp_mlp, y_lens, P, p, cfg, T, S):
    """STDiT2Block.forward, stdit2.py:119-191 (x_mask None)."""
    B, N, C = x.shape
    heads, qk = cfg["num_heads"], cfg["qk_norm"]
    shift_msa, scale_msa, gate_msa, shift_mlp, scale_mlp, gate_mlp = (P[p + ".scale_shift_table"][None] + t_mlp.reshape(B, 6, -1)).chunk(6, dim=1)
    shift_tmp, scale_tmp, gate_tmp = (P[p + ".scale_shift_table_temporal"][None] + t_tmp_mlp.reshape(B, 3, -1)).chunk(3, dim=1)
    ln = lambda z: F.layer_norm(z, (C,), None, None, 1e-6)
    x_m = ln(x) * (1 + scale_msa) + shift_msa
    x_s = attention(x_m.reshape(B * T, S, C), P, p + ".attn", heads, qk, rope=False).reshape(B, T * S, C)
    x = x + gate_msa * x_s
    x_m = ln(x) * (1 + scale_tmp) + shift_tmp
    x_t = x_m.reshape(B, T, S, C).transpose(1, 2).reshape(B * S, T, C)
    x_t = attention(x_t, P, p + ".attn_temp", heads, qk, rope=True)
    x = x + gate_tmp * x_t.reshape(B, S, T, C).transpose(1, 2).reshape(B, T * S, C)
    x = x + cross_attention(x, y, y_lens, P, p + ".cross_attn", heads)
    x_m = ln(x) * (1 + scale_mlp) + shift_mlp
    x_mlp = linear(F.gelu(linear(x_m, P, p + ".mlp.fc1"), approximate="tanh"), P, p + ".mlp.fc2")
    return x + gate_mlp * x_mlp


def stdit2_conditioning(cfg, P: Params, x, timestep, y, mask=None, num_frames=None, height=None, width=None, ar=None,
                        fps=None):
    """STDiT2.forward up to the first block, stdit2.py:338-394: returns dict(h = patch + position embedding [B, T*S, D],
    t, t_mlp [B, 6D], t_tmp_mlp [B, 3D], ye [B, 1, L, D] (before packing), y_packed [1, sum(y_lens), D], y_lens, T, H,
    W)."""
    B = x.shape[0]
    D = cfg["hidden_size"]
    pt, ph, pw = cfg["patch_size"]
    hw = torch.cat([height[:, None], width[:, None]], dim=1)
    rs = (height[0].item() * width[0].item()) ** 0.5
    csize = size_embedder(P, "csize_embedder", hw, B)
    data_info = torch.cat([csize, size_embedder(P, "ar_embedder", ar.unsqueeze(1), B)], dim=1)
    fl = size_embedder(P, "fl_embedder", num_frames.unsqueeze(1), B) + size_embedder(P, "fps_embedder", fps.unsqueeze(1), B)
    _, _, Tx, Hx, Wx = x.shape
    T, H, W = math.ceil(Tx / pt), math.ceil(Hx / ph), math.ceil(Wx / pw)
    S = H * W
    pos_emb = position_embedding_2d(D, H, W, scale=rs / cfg["input_sq_size"], base_size=round(S ** 0.5))
    xp = F.pad(x, (0, W * pw - Wx, 0, H * ph - Hx, 0, T * pt - Tx))
    h = F.conv3d(xp, P["x_embedder.proj.weight"], P["x_embedder.proj.bias"], stride=(pt, ph, pw)).flatten(2).transpose(1, 2)
    h = (h.reshape(B, T, S, D) + pos_emb).reshape(B, T * S, D)
    t = _embedder(P, "t_embedder", timestep)
    t_mlp = linear(F.silu(t + data_info), P, "t_block.1")
    t_tmp_mlp = linear(F.silu(t + fl), P, "t_block_temp.1")
    ye = linear(F.gelu(linear(y, P, "y_embedder.y_proj.fc1"), approximate="tanh"), P, "y_embedder.y_proj.fc2")
    if mask is not None:
        y_lens = mask.sum(dim=1).tolist()
        y_packed = ye.squeeze(1)[mask != 0].reshape(1, -1, D)
    else:
        y_lens = [ye.shape[2]] * B
        y_packed = ye.squeeze(1).reshape(1, -1, D)
    return dict(h=h, t=t, t_mlp=t_mlp, t_tmp_mlp=t_tmp_mlp, ye=ye, y_packed=y_packed, y_lens=y_lens, T=T, H=H, W=W)


def stdit2_forward(cfg, P: Params, x, timestep, y, mask=None, num_frames=None, height=None, width=None, ar=None, fps=None):
    """STDiT2.forward, stdit2.py:334-448. x [B,C,T,H,W]; y [B,1,L,caption]; mask [B,L] or None; returns fp32."""
    B = x.shape[0]
    D = cfg["hidden_size"]
    pt, ph, pw = cfg["patch_size"]
    _, _, Tx, Hx, Wx = x.shape
    c = stdit2_conditioning(cfg, P, x, timestep, y, mask, num_frames, height, width, ar, fps)
    T, H, W, t, h = c["T"], c["H"], c["W"], c["t"], c["h"]
    y, y_lens = c["y_packed"], c["y_lens"]
    for i in range(cfg["depth"]):
        h = stdit2_block(h, y, c["t_mlp"], c["t_tmp_mlp"], y_lens, P, f"blocks.{i}", cfg, T, H * W)
    shift, scale = (P["final_layer.scale_shift_table"][None] + t[:, None]).chunk(2, dim=1)  # T2IFinalLayer :376-385
    h = linear(F.layer_norm(h, (D,), None, None, 1e-6) * (1 + scale) + shift, P, "final_layer.linear")
    oc = cfg["in_channels"] * (2 if cfg["pred_sigma"] else 1)
    h = h.reshape(B, T, H, W, pt, ph, pw, oc).permute(0, 7, 1, 4, 2, 5, 3, 6).reshape(B, oc, T * pt, H * ph, W * pw)
    return h[:, :, :Tx, :Hx, :Wx].float()


def stdit2_flops(cfg, B, T, S, L):
    D, heads = cfg["hidden_size"], cfg["num_heads"]
    hidden = int(D * cfg["mlp_ratio"])
    N = T * S
    per = N * (3 * D * D + D * D) * 2 + 2 * T * S * S * D + 2 * S * T * T * D  # two self-attentions
    per += N * 2 * D * D + L * 2 * D * D + 2 * N * L * D + N * 2 * D * hidden  # cross attention + MLP
    return 2 * B * cfg["depth"] * per
