"""ORACLE (test infrastructure, not product code): CPU fp32 restatement of the reference's UNet2DConditionModel
denoiser forward (SD1.5 / SDXL) in plain functional PyTorch, following the reference files op for op.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / `--impl reference` legs may import this package.

Parity status: the timestep embedding is pinned against the reference's own golden slices
(ppdiffusers/tests/models/test_layers_utils.py:32-115, see tests/test_oracle_goldens.py); the block / model numerics
are PARITY UNPINNED — the reference's layer tests depend on Paddle's RNG stream and PaddlePaddle is not installable
here (SURVEY.md §8c) — and are guarded only by the self-consistency properties the reference's ModelTesterMixin uses.

Conventions follow Paddle, not torch: nn.Linear.weight is [in, out] (y = x W + b,
ppdiffusers/models/modeling_pytorch_paddle_utils.py:27-63); conv weights are [out, in, kh, kw]; tensors are NCHW.
Parameter names are the reference's state-dict keys.
"""
import math
from typing import Dict, Optional

import torch
import torch.nn.functional as F

Params = Dict[str, torch.Tensor]


# ----------------------------------------------------------------------------------------------------------------
# configs (public HF configs the reference loads by name; not vendored in the reference tree, SURVEY.md §8)
# ----------------------------------------------------------------------------------------------------------------
def _cfg(**kw):
    base = dict(  # defaults of UNet2DConditionModel.__init__, ppdiffusers/models/unet_2d_condition.py:172-228
        in_channels=4, out_channels=4, flip_sin_to_cos=True, freq_shift=0,
        down_block_types=("CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "DownBlock2D"),
        up_block_types=("UpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D"),
        block_out_channels=(320, 640, 1280, 1280), layers_per_block=2, norm_num_groups=32, norm_eps=1e-5,
        cross_attention_dim=1280, transformer_layers_per_block=1, attention_head_dim=8, use_linear_projection=False,
        addition_embed_type=None, addition_time_embed_dim=None, projection_class_embeddings_input_dim=None,
        resnet_out_scale_factor=1.0)
    base.update(kw)
    return base


UNET_CONFIGS = {
    # runwayml/stable-diffusion-v1-5 unet/config.json
    "sd15": _cfg(cross_attention_dim=768, attention_head_dim=8),
    # stabilityai/stable-diffusion-xl-base-1.0 unet/config.json
    "sdxl": _cfg(down_block_types=("DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D"),
                 up_block_types=("CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "UpBlock2D"),
                 block_out_channels=(320, 640, 1280), cross_attention_dim=2048,
                 transformer_layers_per_block=(1, 2, 10), attention_head_dim=(5, 10, 20), use_linear_projection=True,
                 addition_embed_type="text_time", addition_time_embed_dim=256,
                 projection_class_embeddings_input_dim=2816),
    # the reference's own unit-test model, ppdiffusers/tests/models/test_models_unet_2d_condition.py:181-194
    "ref_tiny": _cfg(block_out_channels=(32, 64), down_block_types=("CrossAttnDownBlock2D", "DownBlock2D"),
                     up_block_types=("UpBlock2D", "CrossAttnUpBlock2D"), cross_attention_dim=32, attention_head_dim=8),
    # small models with the same structure as sd15 / sdxl whose channel counts the tensor-core kernels accept
    "tiny_sd": _cfg(block_out_channels=(64, 128, 128), down_block_types=("CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "DownBlock2D"),
                    up_block_types=("UpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D"), cross_attention_dim=96,
                    attention_head_dim=(2, 4, 4)),
    "tiny_xl": _cfg(block_out_channels=(64, 128, 256), down_block_types=("DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D"),
                    up_block_types=("CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "UpBlock2D"), cross_attention_dim=128,
                    transformer_layers_per_block=(1, 1, 2), attention_head_dim=(1, 2, 4), use_linear_projection=True,
                    addition_embed_type="text_time", addition_time_embed_dim=32,
                    projection_class_embeddings_input_dim=32 * 6 + 64),
}


def _tup(v, n):
    return tuple(v) if isinstance(v, (tuple, list)) else (v,) * n


def unet_layout(cfg):
    """Static structure derived exactly as unet_2d_condition.py:416-600 derives it. Returns a list of block specs."""
    boc = cfg["block_out_channels"]
    n = len(boc)
    heads = _tup(cfg["attention_head_dim"], n)  # num_attention_heads = attention_head_dim (:245)
    tlpb = _tup(cfg["transformer_layers_per_block"], n)
    lpb = _tup(cfg["layers_per_block"], n)
    cad = _tup(cfg["cross_attention_dim"], n)
    down, up = [], []
    out_ch = boc[0]
    for i, t in enumerate(cfg["down_block_types"]):
        in_ch, out_ch = out_ch, boc[i]
        down.append(dict(type=t, in_ch=in_ch, out_ch=out_ch, layers=lpb[i], heads=heads[i], tlayers=tlpb[i],
                         ctx_dim=cad[i], downsample=(i != n - 1)))
    mid = dict(ch=boc[-1], heads=heads[-1], tlayers=tlpb[-1], ctx_dim=cad[-1])
    rboc, rheads, rtl, rlpb, rcad = [list(reversed(x)) for x in (boc, heads, tlpb, lpb, cad)]
    out_ch = rboc[0]
    for i, t in enumerate(cfg["up_block_types"]):
        prev, out_ch = out_ch, rboc[i]
        in_ch = rboc[min(i + 1, n - 1)]
        up.append(dict(type=t, in_ch=in_ch, out_ch=out_ch, prev_ch=prev, layers=rlpb[i] + 1, heads=rheads[i],
                       tlayers=rtl[i], ctx_dim=rcad[i], upsample=(i != n - 1)))
    return dict(down=down, mid=mid, up=up, time_embed_dim=boc[0] * 4)


# ----------------------------------------------------------------------------------------------------------------
# parameter shapes + synthetic initialisation (there are no checkpoints offline; SURVEY.md §8d)
# ----------------------------------------------------------------------------------------------------------------
def unet_param_shapes(cfg) -> Dict[str, tuple]:
    L = unet_layout(cfg)
    S: Dict[str, tuple] = {}
    ted = L["time_embed_dim"]
    boc = cfg["block_out_channels"]

    def lin(name, i, o, bias=True):
        S[name + ".weight"] = (i, o)  # Paddle layout [in, out]
        if bias:
            S[name + ".bias"] = (o,)

    def conv(name, i, o, k):
        S[name + ".weight"] = (o, i, k, k)
        S[name + ".bias"] = (o,)

    def norm(name, c):
        S[name + ".weight"] = (c,)
        S[name + ".bias"] = (c,)

    def resnet(p, i, o):
        norm(p + ".norm1", i), conv(p + ".conv1", i, o, 3), lin(p + ".time_emb_proj", ted, o)
        norm(p + ".norm2", o), conv(p + ".conv2", o, o, 3)
        if i != o:
            conv(p + ".conv_shortcut", i, o, 1)

    def attn(p, q_dim, ctx_dim):
        lin(p + ".to_q", q_dim, q_dim, False), lin(p + ".to_k", ctx_dim, q_dim, False)
        lin(p + ".to_v", ctx_dim, q_dim, False), lin(p + ".to_out.0", q_dim, q_dim)

    def transformer(p, c, ctx_dim, layers):
        norm(p + ".norm", c)
        if cfg["use_linear_projection"]:
            lin(p + ".proj_in", c, c), lin(p + ".proj_out", c, c)
        else:
            conv(p + ".proj_in", c, c, 1), conv(p + ".proj_out", c, c, 1)
        for j in range(layers):
            b = f"{p}.transformer_blocks.{j}"
            norm(b + ".norm1", c), attn(b + ".attn1", c, c)
            norm(b + ".norm2", c), attn(b + ".attn2", c, ctx_dim)
            norm(b + ".norm3", c), lin(b + ".ff.net.0.proj", c, 8 * c), lin(b + ".ff.net.2", 4 * c, c)

    conv("conv_in", cfg["in_channels"], boc[0], 3)
    lin("time_embedding.linear_1", boc[0], ted), lin("time_embedding.linear_2", ted, ted)
    if cfg["addition_embed_type"] == "text_time":
        lin("add_embedding.linear_1", cfg["projection_class_embeddings_input_dim"], ted)
        lin("add_embedding.linear_2", ted, ted)
    for i, d in enumerate(L["down"]):
        for j in range(d["layers"]):
            resnet(f"down_blocks.{i}.resnets.{j}", d["in_ch"] if j == 0 else d["out_ch"], d["out_ch"])
            if d["type"] == "CrossAttnDownBlock2D":
                transformer(f"down_blocks.{i}.attentions.{j}", d["out_ch"], d["ctx_dim"], d["tlayers"])
        if d["downsample"]:
            conv(f"down_blocks.{i}.downsamplers.0.conv", d["out_ch"], d["out_ch"], 3)
    m = L["mid"]
    resnet("mid_block.resnets.0", m["ch"], m["ch"])
    transformer("mid_block.attentions.0", m["ch"], m["ctx_dim"], m["tlayers"])
    resnet("mid_block.resnets.1", m["ch"], m["ch"])
    for i, u in enumerate(L["up"]):
        for j in range(u["layers"]):
            skip = u["in_ch"] if j == u["layers"] - 1 else u["out_ch"]  # unet_2d_blocks.py:2268-2269
            rin = u["prev_ch"] if j == 0 else u["out_ch"]
            resnet(f"up_blocks.{i}.resnets.{j}", rin + skip, u["out_ch"])
            if u["type"] == "CrossAttnUpBlock2D":
                transformer(f"up_blocks.{i}.attentions.{j}", u["out_ch"], u["ctx_dim"], u["tlayers"])
        if u["upsample"]:
            conv(f"up_blocks.{i}.upsamplers.0.conv", u["out_ch"], u["out_ch"], 3)
    norm("conv_norm_out", boc[0])
    conv("conv_out", boc[0], cfg["out_channels"], 3)
    return S


def init_params(shapes: Dict[str, tuple], seed: int = 1, dtype=torch.float32) -> Params:
    """Synthetic weights: U(-1/sqrt(fan_in), 1/sqrt(fan_in)) for matrices/filters, small random biases, norm scales
    around 1. Every tensor is rounded to bf16-representable values so the bf16 device copy is exact."""
    g = torch.Generator().manual_seed(seed)
    P = {}
    for name in sorted(shapes):
        shp = shapes[name]
        if name.endswith(".weight") and len(shp) >= 2:
            fan_in = shp[0] if len(shp) == 2 else shp[1] * shp[2] * shp[3]
            t = (torch.rand(shp, generator=g) * 2 - 1) / math.sqrt(fan_in)
        elif name.endswith(".weight"):  # norm scale
            t = 1.0 + 0.1 * torch.randn(shp, generator=g)
        else:
            t = 0.05 * torch.randn(shp, generator=g)
        P[name] = t.to(torch.bfloat16).to(dtype)
    return P


# ----------------------------------------------------------------------------------------------------------------
# layers
# ----------------------------------------------------------------------------------------------------------------
def get_timestep_embedding(timesteps, embedding_dim, flip_sin_to_cos=False, downscale_freq_shift=1.0, scale=1.0,
                           max_period=10000):
    """ppdiffusers/models/embeddings.py:26-64."""
    assert timesteps.ndim == 1
    half_dim = embedding_dim // 2
    exponent = -math.log(max_period) * torch.arange(0, half_dim, dtype=torch.float32, device=timesteps.device)
    exponent = exponent / (half_dim - downscale_freq_shift)
    emb = torch.exp(exponent)
    emb = timesteps[:, None].to(torch.float32) * emb[None, :]
    emb = scale * emb
    emb = torch.cat([torch.sin(emb), torch.cos(emb)], dim=-1)
    if flip_sin_to_cos:
        emb = torch.cat([emb[:, half_dim:], emb[:, :half_dim]], dim=-1)
    if embedding_dim % 2 == 1:
        emb = F.pad(emb, (0, 1, 0, 0))
    return emb


def linear(x, P, name):
    """F.linear with Paddle's [in, out] weight (lora.py:453-459 -> paddle.nn.functional.linear)."""
    y = x @ P[name + ".weight"]
    b = P.get(name + ".bias")
    return y if b is None else y + b


def conv2d(x, P, name, stride=1, padding=1):
    return F.conv2d(x, P[name + ".weight"], P.get(name + ".bias"), stride=stride, padding=padding)


def group_norm(x, P, name, groups, eps):
    return F.group_norm(x, groups, P[name + ".weight"], P[name + ".bias"], eps)


def layer_norm(x, P, name, eps=1e-5):
    return F.layer_norm(x, (x.shape[-1],), P[name + ".weight"], P[name + ".bias"], eps)


def timestep_embedding_mlp(x, P, name):
    """TimestepEmbedding.forward, embeddings.py:250-295: linear_1 -> SiLU -> linear_2."""
    return linear(F.silu(linear(x, P, name + ".linear_1")), P, name + ".linear_2")


def resnet_block(x, temb, P, p, groups, eps, out_scale):
    """ResnetBlock2D.forward, resnet.py:728-808 (time_embedding_norm='default', no up/down)."""
    h = F.silu(group_norm(x, P, p + ".norm1", groups, eps))
    h = conv2d(h, P, p + ".conv1")
    t = linear(F.silu(temb), P, p + ".time_emb_proj")[:, :, None, None]
    h = h + t
    h = F.silu(group_norm(h, P, p + ".norm2", groups, eps))
    h = conv2d(h, P, p + ".conv2")
    if (p + ".conv_shortcut.weight") in P:
        x = conv2d(x, P, p + ".conv_shortcut", padding=0)
    return (x + h) / out_scale


def attention(x, ctx, P, p, heads, attention_mask=None, processor=None):
    """Attention.forward + AttnProcessor.__call__ (attention_processor.py:478-510, 673-735): the eager processor a
    CPU-only Paddle selects (SURVEY.md A1). softmax(q k^T * scale + mask) v in the input dtype."""
    if processor is not None:
        return processor(x, ctx, P, p, heads, attention_mask)
    ctx = x if ctx is None else ctx
    q, k, v = linear(x, P, p + ".to_q"), linear(ctx, P, p + ".to_k"), linear(ctx, P, p + ".to_v")
    B, S, C = q.shape
    d = C // heads

    def split(t):  # head_to_batch_dim, :532-550
        return t.reshape(B, -1, heads, d).permute(0, 2, 1, 3)

    q, k, v = split(q), split(k), split(v)
    scores = (q @ k.transpose(-1, -2)) * (d ** -0.5)  # get_attention_scores, :552-586 (baddbmm alpha=scale)
    if attention_mask is not None:
        scores = scores + attention_mask
    probs = torch.softmax(scores, dim=-1)
    o = (probs @ v).permute(0, 2, 1, 3).reshape(B, S, C)
    return linear(o, P, p + ".to_out.0")


def feed_forward_geglu(x, P, p):
    """FeedForward with GEGLU (attention.py:623-677, activations.py:83-104): hidden, gate = proj(x).chunk(2);
    hidden * gelu_erf(gate); then Linear(4C -> C)."""
    h = linear(x, P, p + ".net.0.proj")
    hidden, gate = h.chunk(2, dim=-1)
    return linear(hidden * F.gelu(gate), P, p + ".net.2")


def basic_transformer_block(x, ctx, P, p, heads, processor=None, attention_mask=None, encoder_attention_mask=None):
    """BasicTransformerBlock.forward, attention.py:376-489 (layer_norm branch, eps 1e-5): attn1 takes attention_mask,
    attn2 takes encoder_attention_mask (:411-441); both are additive biases [B, 1, keys] here and are broadcast over
    heads like prepare_attention_mask (attention_processor.py:588-630) does by repeat_interleave."""
    am = None if attention_mask is None else attention_mask[:, None]
    eam = None if encoder_attention_mask is None else encoder_attention_mask[:, None]
    x = attention(layer_norm(x, P, p + ".norm1"), None, P, p + ".attn1", heads, am, processor=processor) + x
    x = attention(layer_norm(x, P, p + ".norm2"), ctx, P, p + ".attn2", heads, eam, processor=processor) + x
    x = feed_forward_geglu(layer_norm(x, P, p + ".norm3"), P, p + ".ff") + x
    return x


def transformer_2d(x, ctx, P, p, heads, layers, groups, use_linear, processor=None, attention_mask=None,
                   encoder_attention_mask=None):
    """Transformer2DModel.forward, transformer_2d.py:272-509 (continuous branch); its GroupNorm eps is hard-coded
    1e-6 (:161-163)."""
    B, C, H, W = x.shape
    res = x
    h = group_norm(x, P, p + ".norm", groups, 1e-6)
    if use_linear:
        h = h.permute(0, 2, 3, 1).reshape(B, H * W, C)
        h = linear(h, P, p + ".proj_in")
    else:
        h = conv2d(h, P, p + ".proj_in", padding=0)
        h = h.permute(0, 2, 3, 1).reshape(B, H * W, C)
    for j in range(layers):
        h = basic_transformer_block(h, ctx, P, f"{p}.transformer_blocks.{j}", heads, processor, attention_mask,
                                    encoder_attention_mask)
    if use_linear:
        h = linear(h, P, p + ".proj_out")
        h = h.reshape(B, H, W, C).permute(0, 3, 1, 2)
    else:
        h = h.reshape(B, H, W, C).permute(0, 3, 1, 2)
        h = conv2d(h, P, p + ".proj_out", padding=0)
    return h + res


# ----------------------------------------------------------------------------------------------------------------
# the model
# ----------------------------------------------------------------------------------------------------------------
def unet_forward(cfg, P: Params, sample, timestep, encoder_hidden_states, added_cond_kwargs: Optional[dict] = None,
                 processor=None, attention_mask=None, encoder_attention_mask=None, down_block_additional_residuals=None,
                 mid_block_additional_residual=None, down_intrablock_additional_residuals=None):
    """UNet2DConditionModel.forward, unet_2d_condition.py:809-1207. sample [B,C,H,W]; timestep number / 0-d / 1-d;
    encoder_hidden_states [B,L,Dctx]; SDXL: added_cond_kwargs = {text_embeds [B,1280], time_ids [B,6]}.
    attention_mask / encoder_attention_mask: [B, keys] keep-masks (1 = keep) -> biases (:916-927).
    ControlNet / T2I-Adapter residuals as in :1078-1155."""
    L = unet_layout(cfg)
    am = eam = None
    if attention_mask is not None:  # :916-922
        am = ((1 - attention_mask.to(sample.dtype)) * -10000.0).unsqueeze(1)
    if encoder_attention_mask is not None:  # :925-927
        eam = ((1 - encoder_attention_mask.to(sample.dtype)) * -10000.0).unsqueeze(1)
    is_controlnet = mid_block_additional_residual is not None and down_block_additional_residuals is not None
    is_adapter = down_intrablock_additional_residuals is not None
    if not is_adapter and mid_block_additional_residual is None and down_block_additional_residuals is not None:
        down_intrablock_additional_residuals, is_adapter = down_block_additional_residuals, True  # :1085-1095
    intra = list(down_intrablock_additional_residuals) if is_adapter else []
    groups, eps, osf = cfg["norm_num_groups"], cfg["norm_eps"], cfg["resnet_out_scale_factor"]
    B = sample.shape[0]
    # 1. time (:934-953): broadcast to batch, fp32 sinusoid, cast to sample dtype, MLP
    t = torch.as_tensor(timestep)
    if t.ndim == 0:
        t = t[None]
    t = t.expand(B)
    t_emb = get_timestep_embedding(t, cfg["block_out_channels"][0], cfg["flip_sin_to_cos"], cfg["freq_shift"])
    emb = timestep_embedding_mlp(t_emb.to(sample.dtype), P, "time_embedding")
    if cfg["addition_embed_type"] == "text_time":  # :991-1010
        text_embeds, time_ids = added_cond_kwargs["text_embeds"], added_cond_kwargs["time_ids"]
        time_embeds = get_timestep_embedding(time_ids.flatten(), cfg["addition_time_embed_dim"],
                                             cfg["flip_sin_to_cos"], cfg["freq_shift"])
        time_embeds = time_embeds.reshape(text_embeds.shape[0], -1)
        add_embeds = torch.cat([text_embeds, time_embeds], dim=-1).to(emb.dtype)
        emb = emb + timestep_embedding_mlp(add_embeds, P, "add_embedding")
    ctx = encoder_hidden_states
    # 2. pre-process (:1064)
    h = conv2d(sample, P, "conv_in")
    # 3. down (:1096-1119)
    skips = [h]
    for i, d in enumerate(L["down"]):
        cross = d["type"] == "CrossAttnDownBlock2D"
        extra = intra.pop(0) if (cross and intra) else None  # :1099-1102
        for j in range(d["layers"]):
            h = resnet_block(h, emb, P, f"down_blocks.{i}.resnets.{j}", groups, eps, osf)
            if cross:
                h = transformer_2d(h, ctx, P, f"down_blocks.{i}.attentions.{j}", d["heads"], d["tlayers"], groups,
                                   cfg["use_linear_projection"], processor, am, eam)
                if extra is not None and j == d["layers"] - 1:  # unet_2d_blocks.py:1211-1213
                    h = h + extra
            skips.append(h)
        if d["downsample"]:  # Downsample2D: conv3x3 stride 2 padding 1 (resnet.py:271-294)
            h = conv2d(h, P, f"down_blocks.{i}.downsamplers.0.conv", stride=2, padding=1)
            skips.append(h)
        if not cross and intra:  # :1115-1119: in-place add that also lands in the block's last res sample
            h = h + intra.pop(0)
            skips[-1] = h
    if is_controlnet:  # :1121-1131
        assert len(skips) == len(down_block_additional_residuals)
        skips = [s_ + r_ for s_, r_ in zip(skips, down_block_additional_residuals)]
    # 4. mid (:1133-1144, unet_2d_blocks.py:750-800)
    m = L["mid"]
    h = resnet_block(h, emb, P, "mid_block.resnets.0", groups, eps, osf)
    h = transformer_2d(h, ctx, P, "mid_block.attentions.0", m["heads"], m["tlayers"], groups,
                       cfg["use_linear_projection"], processor, am, eam)
    h = resnet_block(h, emb, P, "mid_block.resnets.1", groups, eps, osf)
    if intra and h.shape == intra[0].shape:  # T2I-Adapter-XL, :1145-1151
        h = h + intra.pop(0)
    if is_controlnet:  # :1153-1154
        h = h + mid_block_additional_residual
    # 5. up (:1158-1190): pop len(resnets) skips from the end, concat [hidden, skip] on channels
    for i, u in enumerate(L["up"]):
        for j in range(u["layers"]):
            h = torch.cat([h, skips.pop()], dim=1)
            h = resnet_block(h, emb, P, f"up_blocks.{i}.resnets.{j}", groups, eps, osf)
            if u["type"] == "CrossAttnUpBlock2D":
                h = transformer_2d(h, ctx, P, f"up_blocks.{i}.attentions.{j}", u["heads"], u["tlayers"], groups,
                                   cfg["use_linear_projection"], processor, am, eam)
        if u["upsample"]:  # Upsample2D: nearest x2 then conv3x3 (resnet.py:169-218)
            h = F.interpolate(h, scale_factor=2.0, mode="nearest")
            h = conv2d(h, P, f"up_blocks.{i}.upsamplers.0.conv")
    assert not skips
    # 6. post-process (:1193-1196)
    h = F.silu(group_norm(h, P, "conv_norm_out", groups, eps))
    return conv2d(h, P, "conv_out")


def unet_flops(cfg, B, H, W, L_ctx):
    """2*MAC over conv / linear / QK^T / PV of one forward (the 'algorithmic work' of SURVEY.md §8d)."""
    Ly = unet_layout(cfg)
    mac = 0
    boc = cfg["block_out_channels"]
    ted = Ly["time_embed_dim"]

    def res(i, o, hw):
        return hw * (9 * i * o + 9 * o * o + (i * o if i != o else 0)) + ted * o

    def tr(c, ctx_dim, layers, hw, heads):
        m = 2 * hw * c * c  # proj_in/out
        per = hw * (4 * c * c) + 2 * hw * hw * c  # self: q,k,v,out + QK^T + PV
        per += hw * 2 * c * c + 2 * L_ctx * ctx_dim * c + 2 * hw * L_ctx * c  # cross
        per += hw * (c * 8 * c + 4 * c * c)  # GEGLU FF
        return m + layers * per

    hw = H * W
    mac += hw * 9 * cfg["in_channels"] * boc[0]
    mac += boc[0] * ted + ted * ted
    if cfg["addition_embed_type"] == "text_time":
        mac += cfg["projection_class_embeddings_input_dim"] * ted + ted * ted
    for i, d in enumerate(Ly["down"]):
        for j in range(d["layers"]):
            mac += res(d["in_ch"] if j == 0 else d["out_ch"], d["out_ch"], hw)
            if d["type"] == "CrossAttnDownBlock2D":
                mac += tr(d["out_ch"], d["ctx_dim"], d["tlayers"], hw, d["heads"])
        if d["downsample"]:
            hw //= 4
            mac += hw * 9 * d["out_ch"] * d["out_ch"]
    m = Ly["mid"]
    mac += 2 * res(m["ch"], m["ch"], hw) + tr(m["ch"], m["ctx_dim"], m["tlayers"], hw, m["heads"])
    for i, u in enumerate(Ly["up"]):
        for j in range(u["layers"]):
            skip = u["in_ch"] if j == u["layers"] - 1 else u["out_ch"]
            rin = u["prev_ch"] if j == 0 else u["out_ch"]
            mac += res(rin + skip, u["out_ch"], hw)
            if u["type"] == "CrossAttnUpBlock2D":
                mac += tr(u["out_ch"], u["ctx_dim"], u["tlayers"], hw, u["heads"])
        if u["upsample"]:
            hw *= 4
            mac += hw * 9 * u["out_ch"] * u["out_ch"]
    mac += hw * 9 * boc[0] * cfg["out_channels"]
    return 2 * mac * B
