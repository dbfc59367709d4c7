"""UNet2DConditionModel — host-side mirror of ppdiffusers.models.unet_2d_condition.UNet2DConditionModel
(ppdiffusers/models/unet_2d_condition.py:172-228 constructor arguments, :809-824 forward signature) whose forward
runs entirely on hand-written sm_90a kernels through the C ABI (paddlemix_b200.ops).

Data layout on the device (H100-first, not the reference's NCHW nn.Layer graph):
  * activations are NHWC bf16 end to end (the reference's own data_format="NHWC" switch makes this API-legal);
    [B,H,W,C] doubles as the [B*H*W, C] token matrix, so Transformer2DModel's two transposes disappear;
  * every Linear / 1x1 conv / conv3x3 is one launch of the wgmma implicit-GEMM kernel with a fused epilogue
    (bias, temb broadcast, GEGLU, residual add);  q,k,v are one fused projection, cross-attention K/V of all blocks
    are one batched GEMM per forward; all resnet time_emb_proj layers are one batched GEMM per forward;
  * the skip-connection concat is never materialised: GroupNorm reads both sources, the 1x1 shortcut is two
    accumulating GEMMs;
  * heads whose size is not 64/128/192 (SD1.5: 40, 80, 160) are zero-padded once at weight-load time.
Weights are loaded from a reference-named state dict (Paddle layout: Linear weight [in, out]).
"""
from dataclasses import dataclass
from types import SimpleNamespace
from typing import Any, Dict, Optional, Tuple, Union

import os
import numpy as np
import torch

bf16 = torch.bfloat16


@dataclass
class UNet2DConditionOutput:
    """ppdiffusers.models.unet_2d_condition.UNet2DConditionOutput (:55-65)."""
    sample: torch.Tensor = None


class FrozenDict(dict):
    """Attribute-style read-only config, like ppdiffusers.configuration_utils.FrozenDict (:58)."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    def __setattr__(self, k, v):
        raise Exception(f"You cannot use ``__setattr__`` on a {self.__class__.__name__} instance.")


# reference defaults of the UNet2DConditionModel constructor arguments this mirror does not implement
# (ppdiffusers/models/unet_2d_condition.py:172-228)
_REFERENCE_DEFAULTS = dict(
    dual_cross_attention=False, encoder_hid_dim=None, encoder_hid_dim_type=None, class_embed_type=None,
    num_class_embeds=None, upcast_attention=False, resnet_time_scale_shift="default", resnet_skip_time_act=False,
    time_embedding_type="positional", time_embedding_dim=None, time_embedding_act_fn=None, timestep_post_act=None,
    time_cond_proj_dim=None, conv_in_kernel=3, conv_out_kernel=3, mid_block_only_cross_attention=None,
    cross_attention_norm=None, addition_embed_type_num_heads=64, class_embeddings_concat=False,
    reverse_transformer_layers_per_block=None, attention_type="default")


def _tup(v, n):
    return tuple(v) if isinstance(v, (tuple, list)) else (v,) * n


def _pad_head(d):
    for p in (64, 128, 192):
        if d <= p:
            return p
    raise ValueError(f"attention head size {d} > 192 is not supported by the sm_90a attention kernel")


def _to_t(x):
    """fp32 view of a parameter on whatever device it already lives on (host numpy / torch, or CUDA)."""
    if isinstance(x, np.ndarray):
        x = torch.from_numpy(x)
    return x.detach().to(torch.float32)


class AttnProcessorB200:
    """Default attention processor: fused qkv projection + flash SDPA + out-projection kernels.
    Follows the reference processor protocol (attention_processor.py:352-385, 673-735):
    proc(attn, hidden_states, encoder_hidden_states=None, attention_mask=None, temb=None, **cross_attention_kwargs)."""

    def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None, temb=None, **kwargs):
        return attn.fused_forward(hidden_states, encoder_hidden_states, attention_mask=attention_mask)


class Attention:
    """Device-side state of one ppdiffusers `Attention` layer (attention_processor.py:31-207)."""

    def __init__(self, name, heads, dim, ctx_dim, is_cross):
        self.name, self.heads, self.dim, self.ctx_dim, self.is_cross = name, heads, dim, ctx_dim, is_cross
        self.head_dim = dim // heads
        self.head_pad = _pad_head(self.head_dim)
        self.scale = self.head_dim ** -0.5
        self.inner = heads * self.head_pad
        self.processor = AttnProcessorB200()
        self._kv = None  # (k_view, v_view) for cross attention, set per forward by the model

    def set_processor(self, processor):
        self.processor = processor

    def shapes(self):
        n, c, x = self.name, self.dim, self.ctx_dim
        return {n + ".to_q.weight": (c, c), n + ".to_k.weight": (x, c), n + ".to_v.weight": (x, c),
                n + ".to_out.0.weight": (c, c), n + ".to_out.0.bias": (c,)}

    # -- weight preparation ------------------------------------------------------------------------------------
    def _pad_rows(self, w_out_in):  # [H*d, in] -> [H*dp, in]
        H, d, dp = self.heads, self.head_dim, self.head_pad
        if d == dp:
            return w_out_in
        w = w_out_in.reshape(H, d, -1)
        out = torch.zeros(H, dp, w.shape[-1], device=w.device)
        out[:, :d] = w
        return out.reshape(H * dp, -1)

    def load(self, P, dev, norm=None):
        """norm: the LayerNorm in front of this layer (BasicTransformerBlock.norm1 / norm2); its affine is folded into a
        second copy of the query-side projection so that the block can run without the LayerNorm kernel (see
        _BasicTransformerBlock.__call__); the plain weights stay for custom processors."""
        from .. import ops
        n = self.name
        wq = self._pad_rows(_to_t(P[n + ".to_q.weight"]).t().contiguous())
        wk = self._pad_rows(_to_t(P[n + ".to_k.weight"]).t().contiguous())
        wv = self._pad_rows(_to_t(P[n + ".to_v.weight"]).t().contiguous())
        wo = _to_t(P[n + ".to_out.0.weight"]).t().contiguous()  # [C, H*d]
        H, d, dp = self.heads, self.head_dim, self.head_pad
        if d != dp:
            wo3 = torch.zeros(wo.shape[0], H, dp, device=wo.device)
            wo3[:, :, :d] = wo.reshape(wo.shape[0], H, d)
            wo = wo3.reshape(wo.shape[0], H * dp)
        if self.is_cross:
            self.w_q = wq.to(dev, bf16).contiguous()
            self.w_kv_host = torch.cat([wk, wv], 0)  # batched across blocks by the model
            w_in = wq
        else:
            w_in = torch.cat([wq, wk, wv], 0)
            self.w_qkv = w_in.to(dev, bf16).contiguous()
        self.ln_fold = None
        if norm is not None:
            self.ln_fold = ops.fold_layernorm_into_linear(w_in.to(dev, torch.float32), norm.w, norm.b)
        self.w_o = wo.to(dev, bf16).contiguous()
        self.b_o = _to_t(P[n + ".to_out.0.bias"]).to(dev)

    # -- reference-style sub-layers for custom processors --------------------------------------------------------
    def to_q(self, x):
        from .. import ops
        w = self.w_q if self.is_cross else self.w_qkv[: self.inner]
        return ops.linear(x, w)

    def prepare_attention_mask(self, attention_mask, target_length, batch_size):
        """attention_processor.py:588-630 for the bias form the UNet hands down ([B, 1, key_tokens], :916-927): returns an
        additive [B, 1|heads, 1|query_tokens, key_tokens] bias for ops.sdpa (the head axis stays broadcast instead of
        being materialised by repeat_interleave). A mask whose length differs from the key length cannot be applied
        (the reference pads it by `target_length` zeros, :618-623, which only fits UnCLIP's prepended tokens)."""
        if attention_mask is None:
            return None
        m = attention_mask
        if m.dim() == 2:
            m = m[:, None, None, :]
        elif m.dim() == 3:
            m = m[:, None, :, :]
        if m.shape[-1] != target_length:
            raise ValueError(f"attention mask has {m.shape[-1]} key positions, the attention layer {self.name} has "
                             f"{target_length}")
        if m.shape[0] not in (1, batch_size):
            raise ValueError(f"attention mask batch {m.shape[0]} does not match the input batch {batch_size}")
        return m if m.dtype in (torch.float32, bf16) else m.float()

    def fused_forward(self, x, ctx=None, residual=None, attention_mask=None, x_stats=None, out_stats=None):
        """x: [B,S,C] bf16. Returns attention output after to_out, as the reference processors do; `residual` (optional)
        is added in the out-projection's epilogue. x_stats (ops.RowStats of x's rows): x is the UN-normalised hidden
        state and the query-side projection applies the folded LayerNorm; out_stats (a zeroed int64 [rows, 2] table):
        also return the RowStats of the result (for the next folded LayerNorm)."""
        from .. import ops
        B, S, C = x.shape
        H, dp = self.heads, self.head_pad
        if x_stats is not None:
            w_in, colsum, b_in = self.ln_fold
            ln = (x_stats, colsum, self.ln_eps)
        else:
            w_in, b_in, ln = (self.w_q if self.is_cross else self.w_qkv), None, None
        if not self.is_cross:
            qkv = ops.linear(x, w_in, b_in, ln=ln)  # [B,S,3*H*dp]
            q, k, v = (qkv[:, :, i * self.inner:(i + 1) * self.inner].unflatten(-1, (H, dp)) for i in range(3))
        else:
            q = ops.linear(x, w_in, b_in, ln=ln).unflatten(-1, (H, dp))
            k, v = self._kv
        mask = self.prepare_attention_mask(attention_mask, k.shape[1], B)
        o = ops.sdpa(q, k, v, scale=self.scale, attn_mask=mask)
        return ops.linear(o.reshape(B, S, H * dp), self.w_o, self.b_o, residual=residual, stats=out_stats)

    def fused_forward_residual(self, x, residual, attention_mask=None):
        """Same as fused_forward but with the residual add fused into the out-projection epilogue."""
        return self.fused_forward(x, None, residual=residual, attention_mask=attention_mask)


class _Norm:
    def __init__(self, name, c=None):
        self.name, self.c = name, c

    def shapes(self):
        return {self.name + ".weight": (self.c,), self.name + ".bias": (self.c,)}

    def load(self, P, dev):
        self.w = _to_t(P[self.name + ".weight"]).to(dev)
        self.b = _to_t(P[self.name + ".bias"]).to(dev)


class _Linear:
    def __init__(self, name, cin=None, cout=None, conv1x1=False):
        self.name, self.cin, self.cout, self.conv1x1 = name, cin, cout, conv1x1

    def shapes(self):
        w = (self.cout, self.cin, 1, 1) if self.conv1x1 else (self.cin, self.cout)  # Paddle Linear is [in, out]
        return {self.name + ".weight": w, self.name + ".bias": (self.cout,)}

    def load(self, P, dev):
        w = _to_t(P[self.name + ".weight"])
        if w.ndim == 4:  # 1x1 conv [out, in, 1, 1]
            w = w[:, :, 0, 0]
        else:  # Paddle Linear [in, out]
            w = w.t()
        self.w = w.contiguous().to(dev, bf16)
        b = P.get(self.name + ".bias")
        self.b = None if b is None else _to_t(b).to(dev)


class _Conv3x3:
    def __init__(self, name, cin=None, cout=None, upsample=False):
        # upsample: the conv of an Upsample2D (resnet.py:169-218); its filter is folded per output parity at load time so
        # that nearest-2x + conv3x3 run as one 4-tap pass over the low-resolution input (ops.conv3x3_up2x)
        self.name, self.cin, self.cout, self.upsample = name, cin, cout, upsample

    def shapes(self):
        return {self.name + ".weight": (self.cout, self.cin, 3, 3), self.name + ".bias": (self.cout,)}

    def load(self, P, dev):
        w = _to_t(P[self.name + ".weight"])  # [O, I, 3, 3] -> [O, 3, 3, I]
        self.w = w.permute(0, 2, 3, 1).contiguous().to(dev, bf16)
        self.b = _to_t(P[self.name + ".bias"]).to(dev)
        if self.upsample:
            from .. import ops
            self.w4 = ops.fold_upsample_conv_weight(w.permute(0, 2, 3, 1).to(dev, torch.float32))

    def up2x(self, h):
        """conv(nearest_upsample_2x(h))"""
        from .. import ops
        return ops.conv3x3_up2x(h, self.w4, self.b)


class _Resnet:
    """ResnetBlock2D (resnet.py:587-808), time_embedding_norm='default'."""

    def __init__(self, name, cin, cout, groups, eps, out_scale):
        self.name, self.cin, self.cout, self.groups, self.eps, self.out_scale = name, cin, cout, groups, eps, out_scale
        self.norm1, self.conv1 = _Norm(name + ".norm1", cin), _Conv3x3(name + ".conv1", cin, cout)
        self.norm2, self.conv2 = _Norm(name + ".norm2", cout), _Conv3x3(name + ".conv2", cout, cout)
        self.shortcut = _Linear(name + ".conv_shortcut", cin, cout, conv1x1=True) if cin != cout else None
        self.temb_slice = None  # (offset, size) into the batched time_emb_proj output
        self.ted = None

    def shapes(self):
        out = {}
        for m in (self.norm1, self.conv1, self.norm2, self.conv2, self.shortcut):
            if m is not None:
                out.update(m.shapes())
        out[self.name + ".time_emb_proj.weight"] = (self.ted, self.cout)
        out[self.name + ".time_emb_proj.bias"] = (self.cout,)
        return out

    def load(self, P, dev):
        for m in (self.norm1, self.conv1, self.norm2, self.conv2):
            m.load(P, dev)
        if self.shortcut is not None:
            self.shortcut.load(P, dev)
        self.temb_w = _to_t(P[self.name + ".time_emb_proj.weight"]).t().contiguous()  # [cout, ted], batched later
        self.temb_b = _to_t(P[self.name + ".time_emb_proj.bias"])

    def __call__(self, x, temb_all, skip=None):
        from .. import ops
        c1 = x.shape[-1]
        n1 = ops.groupnorm_nhwc(x, self.norm1.w, self.norm1.b, x2=skip, groups=self.groups, eps=self.eps, silu=True)
        off, size = self.temb_slice
        h = ops.conv3x3(n1, self.conv1.w, self.conv1.b, row_add=temb_all[:, off:off + size])
        n2 = ops.groupnorm_nhwc(h, self.norm2.w, self.norm2.b, groups=self.groups, eps=self.eps, silu=True)
        if self.shortcut is not None:
            w = self.shortcut.w
            if skip is None:
                res = ops.linear(x, w, self.shortcut.b)
            else:  # 1x1 conv over the virtual concat [x | skip] = two accumulating GEMMs
                res = ops.linear(x, w[:, :c1], self.shortcut.b)
                res = ops.linear(skip, w[:, c1:], None, residual=res, out=res)
        else:
            assert skip is None
            res = x
        return ops.conv3x3(n2, self.conv2.w, self.conv2.b, residual=res, out_scale=1.0 / self.out_scale)


class _BasicTransformerBlock:
    """BasicTransformerBlock (attention.py:217-489), layer_norm variant with GEGLU feed-forward."""

    def __init__(self, name, dim, heads, ctx_dim):
        self.name, self.dim = name, dim
        self.norm1, self.norm2, self.norm3 = (_Norm(name + f".norm{i}", dim) for i in (1, 2, 3))
        self.attn1 = Attention(name + ".attn1", heads, dim, dim, False)
        self.attn2 = Attention(name + ".attn2", heads, dim, ctx_dim, True)
        self.ff2 = _Linear(name + ".ff.net.2", 4 * dim, dim)

    def shapes(self):
        out = {}
        for m in (self.norm1, self.norm2, self.norm3, self.attn1, self.attn2, self.ff2):
            out.update(m.shapes())
        out[self.name + ".ff.net.0.proj.weight"] = (self.dim, 8 * self.dim)
        out[self.name + ".ff.net.0.proj.bias"] = (8 * self.dim,)
        return out

    LN_EPS = 1e-5

    def load(self, P, dev):
        from .. import ops
        for m in (self.norm1, self.norm2, self.norm3, self.ff2):
            m.load(P, dev)
        self.attn1.load(P, dev, norm=self.norm1)
        self.attn2.load(P, dev, norm=self.norm2)
        self.attn1.ln_eps = self.attn2.ln_eps = self.LN_EPS
        # GEGLU: proj(x).chunk(2) = (value, gate) -> interleave rows so both land in the same accumulator tile
        w = _to_t(P[self.name + ".ff.net.0.proj.weight"]).t().contiguous()  # [8C, C]
        b = _to_t(P[self.name + ".ff.net.0.proj.bias"])
        half = w.shape[0] // 2
        w_il = torch.stack([w[:half], w[half:]], 1).reshape(2 * half, -1).contiguous()
        b_il = torch.stack([b[:half], b[half:]], 1).reshape(2 * half).contiguous()
        self.ff1_w = w_il.to(dev, bf16)
        self.ff1_b = b_il.to(dev)
        # norm3 folded into the GEGLU projection (W' = W * gamma, bias' = bias + W beta, column sums of W')
        self.ff1_fold = ops.fold_layernorm_into_linear(w_il.to(dev, torch.float32), self.norm3.w, self.norm3.b, self.ff1_b)

    def __call__(self, h, ctx, cross_attention_kwargs, attention_mask=None, encoder_attention_mask=None, h_stats=None,
                 stats_tables=None):
        """attention.py:352-489: attn1 gets `attention_mask`, attn2 gets `encoder_attention_mask` (:411-441).
        h_stats = ops.RowStats of h (left by the GEMM that produced h): the three LayerNorms then never run as kernels.
        Each is folded into the projection that consumes it (norm1 -> to_q|k|v, norm2 -> attn2.to_q, norm3 -> GEGLU
        proj), whose epilogue rebuilds the row's mean / rstd from the statistics the producing GEMM's epilogue took of
        the residual stream (stats_tables: three zeroed int64 [rows, 2] tables for the three residual updates of this
        block). Returns (h, RowStats of h) in that mode. Custom processors get the reference order
        (norm -> processor -> residual add) on explicit LayerNorm kernels."""
        from .. import ops
        from .._lib import GLU_GEGLU
        kw = cross_attention_kwargs or {}
        default = type(self.attn1.processor) is AttnProcessorB200 and type(self.attn2.processor) is AttnProcessorB200
        if h_stats is not None and default and not kw:
            h, st = self.attn1.fused_forward(h, None, residual=h, attention_mask=attention_mask, x_stats=h_stats,
                                             out_stats=stats_tables[0])
            h, st = self.attn2.fused_forward(h, None, residual=h, attention_mask=encoder_attention_mask, x_stats=st,
                                             out_stats=stats_tables[1])
            w3, colsum3, b3 = self.ff1_fold
            ff = ops.linear(h, w3, b3, glu=GLU_GEGLU, ln=(st, colsum3, self.LN_EPS))
            return ops.linear(ff, self.ff2.w, self.ff2.b, residual=h, stats=stats_tables[2])
        n = ops.layernorm(h, self.norm1.w, self.norm1.b, eps=1e-5)
        if type(self.attn1.processor) is AttnProcessorB200 and not kw:
            h = self.attn1.fused_forward_residual(n, h, attention_mask)
        else:
            h = _add(self.attn1.processor(self.attn1, n, encoder_hidden_states=None, attention_mask=attention_mask,
                                          **kw), h)
        n = ops.layernorm(h, self.norm2.w, self.norm2.b, eps=1e-5)
        if type(self.attn2.processor) is AttnProcessorB200 and not kw:
            h = self.attn2.fused_forward_residual(n, h, encoder_attention_mask)
        else:
            h = _add(self.attn2.processor(self.attn2, n, encoder_hidden_states=ctx,
                                          attention_mask=encoder_attention_mask, **kw), h)
        n = ops.layernorm(h, self.norm3.w, self.norm3.b, eps=1e-5)
        ff = ops.linear(n, self.ff1_w, self.ff1_b, glu=GLU_GEGLU)
        return ops.linear(ff, self.ff2.w, self.ff2.b, residual=h, stats=None if h_stats is None else stats_tables[2])


def _add(a, b):
    """bf16 a + b through the GEMM-free path (only used with custom processors)."""
    return (a.float() + b.float()).to(bf16)


class _Transformer2D:
    """Transformer2DModel (transformer_2d.py:54-509), continuous-input branch."""
    FOLD_LAYERNORM = os.environ.get("B200MIX_FOLD_LN", "1") != "0"  # measurement switch: 0 = explicit LayerNorm kernels

    def __init__(self, name, dim, heads, ctx_dim, layers, groups, use_linear):
        self.name, self.dim, self.groups = name, dim, groups
        self.norm = _Norm(name + ".norm", dim)
        self.proj_in = _Linear(name + ".proj_in", dim, dim, conv1x1=not use_linear)
        self.proj_out = _Linear(name + ".proj_out", dim, dim, conv1x1=not use_linear)
        self.blocks = [_BasicTransformerBlock(f"{name}.transformer_blocks.{j}", dim, heads, ctx_dim) for j in range(layers)]

    def shapes(self):
        out = {}
        for m in (self.norm, self.proj_in, self.proj_out, *self.blocks):
            out.update(m.shapes())
        return out

    def load(self, P, dev):
        for m in (self.norm, self.proj_in, self.proj_out, *self.blocks):
            m.load(P, dev)

    def __call__(self, x, ctx, cross_attention_kwargs, attention_mask=None, encoder_attention_mask=None):
        from .. import ops
        B, H, W, C = x.shape
        n = ops.groupnorm_nhwc(x, self.norm.w, self.norm.b, groups=self.groups, eps=1e-6, silu=False)
        # the residual stream travels with its row statistics (taken by the epilogue of whichever GEMM wrote it), so
        # the blocks' LayerNorms are folded into their consumers; FOLD_LAYERNORM = False restores the explicit kernels
        if self.FOLD_LAYERNORM and C % 32 == 0:
            tables = ops.RowStats.arena(1 + 3 * len(self.blocks), B * H * W, x.device)  # one memset for the whole stack
            h, st = ops.linear(n.reshape(B, H * W, C), self.proj_in.w, self.proj_in.b, stats=tables[0])
            for j, blk in enumerate(self.blocks):
                h, st = blk(h, ctx, cross_attention_kwargs, attention_mask, encoder_attention_mask, h_stats=st,
                            stats_tables=tables[1 + 3 * j:4 + 3 * j])
        else:
            h = ops.linear(n.reshape(B, H * W, C), self.proj_in.w, self.proj_in.b)
            for blk in self.blocks:
                h = blk(h, ctx, cross_attention_kwargs, attention_mask, encoder_attention_mask)
        out = ops.linear(h, self.proj_out.w, self.proj_out.b, residual=x.reshape(B, H * W, C))
        return out.reshape(B, H, W, C)


class UNet2DConditionModel:
    """Drop-in for ppdiffusers.UNet2DConditionModel on the denoising hot path (inference, no adapters)."""

    def __init__(self, sample_size: Optional[int] = None, in_channels: int = 4, out_channels: int = 4,
                 center_input_sample: bool = False, flip_sin_to_cos: bool = True, freq_shift: int = 0,
                 down_block_types: Tuple[str] = ("CrossAttnDownBlock2D", "CrossAttnDownBlock2D",
                                                 "CrossAttnDownBlock2D", "DownBlock2D"),
                 mid_block_type: Optional[str] = "UNetMidBlock2DCrossAttn",
                 up_block_types: Tuple[str] = ("UpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D",
                                               "CrossAttnUpBlock2D"),
                 only_cross_attention: Union[bool, Tuple[bool]] = False,
                 block_out_channels: Tuple[int] = (320, 640, 1280, 1280), layers_per_block: Union[int, Tuple[int]] = 2,
                 downsample_padding: int = 1, mid_block_scale_factor: float = 1, dropout: float = 0.0,
                 act_fn: str = "silu", norm_num_groups: Optional[int] = 32, norm_eps: float = 1e-5,
                 cross_attention_dim: Union[int, Tuple[int]] = 1280,
                 transformer_layers_per_block: Union[int, Tuple[int]] = 1, attention_head_dim: Union[int, Tuple[int]] = 8,
                 num_attention_heads=None, use_linear_projection: bool = False, addition_embed_type: Optional[str] = None,
                 addition_time_embed_dim: Optional[int] = None, resnet_out_scale_factor: float = 1.0,
                 projection_class_embeddings_input_dim: Optional[int] = None, data_format: str = "NCHW", **unsupported):
        if num_attention_heads is not None:
            raise ValueError("At the moment it is not possible to define the number of attention heads via "
                             "`num_attention_heads` because of a naming issue as described in "
                             "https://github.com/huggingface/diffusers/issues/2011#issuecomment-1547958131. Passing "
                             "`num_attention_heads` will only be supported in diffusers v0.19.")
        # the remaining reference constructor arguments (unet_2d_condition.py:172-228) are accepted only at their
        # reference defaults: each is compared with ITS OWN default by type and value (True == 1.0 must not pass)
        for k, v in unsupported.items():
            if k.startswith("_"):  # _class_name / _ppdiffusers_version bookkeeping of config.json
                continue
            if k == "upcast_attention" and isinstance(v, bool):
                continue  # scores are always accumulated and soft-maxed in fp32 here (attention.cu), i.e. "upcast"
            if k not in _REFERENCE_DEFAULTS:
                raise NotImplementedError(f"UNet2DConditionModel(b200): unknown config option {k}={v!r}")
            d = _REFERENCE_DEFAULTS[k]
            if not (v is d or (type(v) is type(d) and v == d)):
                raise NotImplementedError(f"UNet2DConditionModel(b200): config option {k}={v!r} is outside the hot path "
                                          f"(only the reference default {d!r} is supported)")
        if len(down_block_types) != len(up_block_types):
            raise ValueError(f"Must provide the same number of `down_block_types` as `up_block_types`. "
                             f"`down_block_types`: {down_block_types}. `up_block_types`: {up_block_types}.")
        if len(block_out_channels) != len(down_block_types):
            raise ValueError(f"Must provide the same number of `block_out_channels` as `down_block_types`. "
                             f"`block_out_channels`: {block_out_channels}. `down_block_types`: {down_block_types}.")
        if act_fn != "silu" or mid_block_type != "UNetMidBlock2DCrossAttn" or only_cross_attention or dropout != 0.0 \
                or center_input_sample or downsample_padding != 1:
            raise NotImplementedError("UNet2DConditionModel(b200) covers the SD / SDXL configuration family only")
        if addition_embed_type not in (None, "text_time"):
            raise NotImplementedError(f"addition_embed_type={addition_embed_type}")
        cfg = dict(sample_size=sample_size, in_channels=in_channels, out_channels=out_channels,
                   flip_sin_to_cos=flip_sin_to_cos, freq_shift=freq_shift, down_block_types=tuple(down_block_types),
                   mid_block_type=mid_block_type, up_block_types=tuple(up_block_types),
                   block_out_channels=tuple(block_out_channels), layers_per_block=layers_per_block,
                   norm_num_groups=norm_num_groups, norm_eps=norm_eps, cross_attention_dim=cross_attention_dim,
                   transformer_layers_per_block=transformer_layers_per_block, attention_head_dim=attention_head_dim,
                   use_linear_projection=use_linear_projection, addition_embed_type=addition_embed_type,
                   addition_time_embed_dim=addition_time_embed_dim, resnet_out_scale_factor=resnet_out_scale_factor,
                   projection_class_embeddings_input_dim=projection_class_embeddings_input_dim, act_fn=act_fn,
                   data_format=data_format, time_cond_proj_dim=None)
        self.config = FrozenDict(cfg)
        self.sample_size, self.in_channels, self.data_format = sample_size, in_channels, data_format
        self.dtype = bf16
        self.device = None
        self._build()
        self._graphs: Dict[Any, Any] = {}

    # ------------------------------------------------------------------------------------------------------------
    def _build(self):
        c = self.config
        boc = c.block_out_channels
        n = len(boc)
        heads, tl = _tup(c.attention_head_dim, n), _tup(c.transformer_layers_per_block, n)
        lpb, cad = _tup(c.layers_per_block, n), _tup(c.cross_attention_dim, n)
        g, eps, osf = c.norm_num_groups, c.norm_eps, c.resnet_out_scale_factor
        self.time_embed_dim = boc[0] * 4
        ted = self.time_embed_dim
        self.conv_in = _Conv3x3("conv_in", c.in_channels, boc[0])
        self.time_lin1, self.time_lin2 = _Linear("time_embedding.linear_1", boc[0], ted), _Linear("time_embedding.linear_2", ted, ted)
        self.add_lin1 = self.add_lin2 = None
        if c.addition_embed_type == "text_time":
            self.add_lin1 = _Linear("add_embedding.linear_1", c.projection_class_embeddings_input_dim, ted)
            self.add_lin2 = _Linear("add_embedding.linear_2", ted, ted)
            # pipelines read unet.add_embedding.linear_1.in_features (pipeline_stable_diffusion_xl.py:609-611)
            self.add_embedding = SimpleNamespace(linear_1=SimpleNamespace(in_features=c.projection_class_embeddings_input_dim))
        self.down, self.up = [], []
        self.resnets, self.transformers = [], []

        def res(name, i, o):
            r = _Resnet(name, i, o, g, eps, osf)
            r.ted = ted
            self.resnets.append(r)
            return r

        def tr(name, ch, h, ctx, layers):
            t = _Transformer2D(name, ch, h, ctx, layers, g, c.use_linear_projection)
            self.transformers.append(t)
            return t

        out_ch = boc[0]
        for i, t in enumerate(c.down_block_types):
            in_ch, out_ch = out_ch, boc[i]
            blk = SimpleNamespace(resnets=[], attns=[], down=None)
            for j in range(lpb[i]):
                blk.resnets.append(res(f"down_blocks.{i}.resnets.{j}", in_ch if j == 0 else out_ch, out_ch))
                if t == "CrossAttnDownBlock2D":
                    blk.attns.append(tr(f"down_blocks.{i}.attentions.{j}", out_ch, heads[i], cad[i], tl[i]))
                elif t != "DownBlock2D":
                    raise NotImplementedError(f"down block type {t}")
            if i != n - 1:
                blk.down = _Conv3x3(f"down_blocks.{i}.downsamplers.0.conv", out_ch, out_ch)
            self.down.append(blk)
        self.mid = SimpleNamespace(
            res0=res("mid_block.resnets.0", boc[-1], boc[-1]),
            attn=tr("mid_block.attentions.0", boc[-1], heads[-1], cad[-1], tl[-1]),
            res1=res("mid_block.resnets.1", boc[-1], boc[-1]))
        rboc, rheads, rtl, rlpb, rcad = [list(reversed(x)) for x in (boc, heads, tl, lpb, cad)]
        out_ch = rboc[0]
        for i, t in enumerate(c.up_block_types):
            prev, out_ch = out_ch, rboc[i]
            in_ch = rboc[min(i + 1, n - 1)]
            blk = SimpleNamespace(resnets=[], attns=[], up=None)
            for j in range(rlpb[i] + 1):
                skip = in_ch if j == rlpb[i] else out_ch
                rin = prev if j == 0 else out_ch
                blk.resnets.append(res(f"up_blocks.{i}.resnets.{j}", rin + skip, out_ch))
                if t == "CrossAttnUpBlock2D":
                    blk.attns.append(tr(f"up_blocks.{i}.attentions.{j}", out_ch, rheads[i], rcad[i], rtl[i]))
                elif t != "UpBlock2D":
                    raise NotImplementedError(f"up block type {t}")
            if i != n - 1:
                blk.up = _Conv3x3(f"up_blocks.{i}.upsamplers.0.conv", out_ch, out_ch, upsample=True)
            self.up.append(blk)
        self.norm_out, self.conv_out = _Norm("conv_norm_out", boc[0]), _Conv3x3("conv_out", boc[0], c.out_channels)

    def state_dict_shapes(self) -> Dict[str, tuple]:
        """Names and shapes of the reference state dict this model consumes (Paddle layouts)."""
        out = {}
        leaves = [self.conv_in, self.time_lin1, self.time_lin2, self.add_lin1, self.add_lin2, self.norm_out, self.conv_out,
                  *self.resnets, *self.transformers, *(b.down for b in self.down), *(b.up for b in self.up)]
        for m in leaves:
            if m is not None:
                out.update(m.shapes())
        return out

    def init_synthetic_weights(self, seed: int = 1, device: Union[int, str] = 0):
        """Random-init weights of this architecture generated directly on the device (there are no checkpoints
        offline): U(-1/sqrt(fan_in), 1/sqrt(fan_in)) matrices, small biases, norm scales around 1."""
        dev = torch.device("cuda", device) if isinstance(device, int) else torch.device(device)
        g = torch.Generator(device=dev).manual_seed(seed)
        P = {}
        for name, shp in sorted(self.state_dict_shapes().items()):
            if name.endswith(".weight") and len(shp) >= 2:
                fan_in = shp[0] if len(shp) == 2 else shp[1] * shp[2] * shp[3]
                t = (torch.rand(shp, generator=g, device=dev) * 2 - 1) / fan_in ** 0.5
            elif name.endswith(".weight"):
                t = 1.0 + 0.1 * torch.randn(shp, generator=g, device=dev)
            else:
                t = 0.05 * torch.randn(shp, generator=g, device=dev)
            P[name] = t.to(bf16)
        return self.load_state_dict(P, device=device)

    # ------------------------------------------------------------------------------------------------------------
    @property
    def attn_processors(self) -> Dict[str, Any]:
        """unet_2d_condition.py:634-655."""
        out = {}
        for t in self.transformers:
            for b in t.blocks:
                out[b.attn1.name + ".processor"] = b.attn1.processor
                out[b.attn2.name + ".processor"] = b.attn2.processor
        return out

    def set_attn_processor(self, processor):
        """unet_2d_condition.py:657-691: one processor for all layers, or a dict keyed like attn_processors."""
        count = len(self.attn_processors)
        if isinstance(processor, dict) and len(processor) != count:
            raise ValueError(f"A dict of processors was passed, but the number of processors {len(processor)} does not"
                             f" match the number of attention layers: {count}. Please make sure to pass {count} "
                             f"processor classes.")
        for t in self.transformers:
            for b in t.blocks:
                for a in (b.attn1, b.attn2):
                    a.set_processor(processor if not isinstance(processor, dict) else processor[a.name + ".processor"])
        self._graphs.clear()

    def set_default_attn_processor(self):
        self.set_attn_processor(AttnProcessorB200())

    # ------------------------------------------------------------------------------------------------------------
    def load_state_dict(self, state_dict: Dict[str, Any], device: Union[int, str] = 0):
        """Reference-named parameters (ppdiffusers state-dict keys, Paddle layouts). Every Linear is transposed once,
        convs go to [O,kh,kw,I], q/k/v (and cross k/v, time_emb_proj) are concatenated for batched GEMMs."""
        from .. import ops
        dev = torch.device("cuda", device) if isinstance(device, int) else torch.device(device)
        ops.init(dev.index or 0)
        self.device = dev
        P = state_dict
        missing = [k for k in self.state_dict_shapes() if k not in P]
        if missing:
            raise KeyError(f"state dict is missing {len(missing)} parameters, e.g. {missing[:3]}")
        for m in (self.conv_in, self.time_lin1, self.time_lin2, self.norm_out, self.conv_out):
            m.load(P, dev)
        if self.add_lin1 is not None:
            self.add_lin1.load(P, dev), self.add_lin2.load(P, dev)
        for r in self.resnets:
            r.load(P, dev)
        for t in self.transformers:
            t.load(P, dev)
        for blk in self.down:
            if blk.down is not None:
                blk.down.load(P, dev)
        for blk in self.up:
            if blk.up is not None:
                blk.up.load(P, dev)
        # batched time_emb_proj: one GEMM [B, ted] x [sum(cout), ted]^T per forward
        off = 0
        ws, bs = [], []
        for r in self.resnets:
            r.temb_slice = (off, r.cout)
            off += r.cout
            ws.append(r.temb_w), bs.append(r.temb_b)
            del r.temb_w, r.temb_b
        self.temb_w_all = torch.cat(ws, 0).to(dev, bf16).contiguous()
        self.temb_b_all = torch.cat(bs, 0).to(dev)
        # batched cross-attention K/V projection of the text context, grouped by context width
        self._kv_groups = {}
        for t in self.transformers:
            for b in t.blocks:
                a = b.attn2
                grp = self._kv_groups.setdefault(a.ctx_dim, dict(w=[], attns=[], off=0))
                a._kv_off = grp["off"]
                grp["off"] += a.w_kv_host.shape[0]
                grp["w"].append(a.w_kv_host)
                grp["attns"].append(a)
                del a.w_kv_host
        for grp in self._kv_groups.values():
            grp["w"] = torch.cat(grp["w"], 0).to(dev, bf16).contiguous()
        self._graphs.clear()
        return self

    # ------------------------------------------------------------------------------------------------------------
    def _embeddings(self, timestep, B, added_cond_kwargs):
        """unet_2d_condition.py:934-1010 -> SiLU(emb) [B, ted] bf16, then all time_emb_proj at once (fp32)."""
        from .. import ops
        from .._lib import ACT_SILU
        c = self.config
        dev = self.device
        if not torch.is_tensor(timestep):
            timestep = torch.tensor([timestep], dtype=torch.float32, device=dev)
        t = timestep.to(device=dev, dtype=torch.float32).reshape(-1)
        if t.numel() == 1 and B > 1:
            t = t.expand(B)
        t = t.contiguous()
        t_emb = ops.timestep_embedding(t, c.block_out_channels[0], flip_sin_to_cos=c.flip_sin_to_cos,
                                       downscale_freq_shift=c.freq_shift)
        h = ops.linear(t_emb, self.time_lin1.w, self.time_lin1.b, act=ACT_SILU)
        emb = ops.linear(h, self.time_lin2.w, self.time_lin2.b)
        if c.addition_embed_type == "text_time":
            if added_cond_kwargs is None or "text_embeds" not in added_cond_kwargs:
                raise ValueError(f"{self.__class__} has the config param `addition_embed_type` set to 'text_time' which "
                                 "requires the keyword argument `text_embeds` to be passed in `added_cond_kwargs`")
            if "time_ids" not in added_cond_kwargs:
                raise ValueError(f"{self.__class__} has the config param `addition_embed_type` set to 'text_time' which "
                                 "requires the keyword argument `time_ids` to be passed in `added_cond_kwargs`")
            text_embeds = added_cond_kwargs["text_embeds"].to(dev)
            time_ids = added_cond_kwargs["time_ids"].to(device=dev, dtype=torch.float32).contiguous()
            nt, td = time_ids.shape[1], c.addition_time_embed_dim
            add = torch.empty(B, text_embeds.shape[1] + nt * td, device=dev, dtype=bf16)
            add[:, : text_embeds.shape[1]] = text_embeds
            # time_ids.flatten() -> sinusoid(td) -> reshape [B, nt*td], concatenated after text_embeds (:1003-1008)
            flat = time_ids.reshape(-1)
            emb_ids = ops.timestep_embedding(flat, td, flip_sin_to_cos=c.flip_sin_to_cos,
                                             downscale_freq_shift=c.freq_shift)
            add[:, text_embeds.shape[1]:] = emb_ids.reshape(B, nt * td)
            h2 = ops.linear(add, self.add_lin1.w, self.add_lin1.b, act=ACT_SILU)
            emb = ops.linear(h2, self.add_lin2.w, self.add_lin2.b, residual=emb)
        s_emb = ops.activation(emb, ACT_SILU)
        return ops.linear(s_emb, self.temb_w_all, self.temb_b_all, out_fp32=True)  # [B, sum(cout)] fp32

    def _project_context(self, ctx):
        from .. import ops
        B, L, Dc = ctx.shape
        grp = self._kv_groups.get(Dc)
        if grp is None:
            raise ValueError(f"encoder_hidden_states has width {Dc}, expected one of {list(self._kv_groups)}")
        kv_all = ops.linear(ctx, grp["w"])  # [B, L, sum(2*H*dp)]
        for a in grp["attns"]:
            k = kv_all[:, :, a._kv_off: a._kv_off + a.inner].unflatten(-1, (a.heads, a.head_pad))
            v = kv_all[:, :, a._kv_off + a.inner: a._kv_off + 2 * a.inner].unflatten(-1, (a.heads, a.head_pad))
            a._kv = (k, v)

    def forward_nhwc(self, x_nhwc, timestep, ctx, added_cond_kwargs=None, cross_attention_kwargs=None,
                     attention_mask=None, encoder_attention_mask=None, down_block_additional_residuals=None,
                     mid_block_additional_residual=None, down_intrablock_additional_residuals=None,
                     residuals_nchw=True):
        """x_nhwc: bf16/fp32 [B,H,W,Cin]; ctx: bf16 [B,L,Dctx]. Returns bf16 [B,H,W,Cout].
        attention_mask / encoder_attention_mask: additive biases [B,1,keys] (already converted, see forward()).
        ControlNet / T2I-Adapter residuals (unet_2d_condition.py:1078-1155) are in the caller's NCHW layout unless
        `residuals_nchw` is False."""
        from .. import ops
        B = x_nhwc.shape[0]
        temb_all = self._embeddings(timestep, B, added_cond_kwargs)
        self._project_context(ctx)
        kw = cross_attention_kwargs
        am, eam = attention_mask, encoder_attention_mask
        add = lambda t, r: ops.add_residual_nhwc(t, r, r_nchw=residuals_nchw)  # noqa: E731
        is_controlnet = mid_block_additional_residual is not None and down_block_additional_residuals is not None
        is_adapter = down_intrablock_additional_residuals is not None
        if not is_adapter and mid_block_additional_residual is None and down_block_additional_residuals is not None:
            # legacy T2I-Adapter usage through the ControlNet argument (:1085-1095)
            down_intrablock_additional_residuals, is_adapter = down_block_additional_residuals, True
        intra = list(down_intrablock_additional_residuals) if is_adapter else []
        h = ops.conv3x3_small_cin(x_nhwc, self.conv_in.w, self.conv_in.b)
        skips = [h]
        for blk in self.down:
            extra = intra.pop(0) if (blk.attns and intra) else None  # CrossAttnDownBlock2D: after the last pair
            for j, r in enumerate(blk.resnets):
                h = r(h, temb_all)
                if blk.attns:
                    h = blk.attns[j](h, ctx, kw, am, eam)
                    if extra is not None and j == len(blk.resnets) - 1:
                        h = add(h, extra)
                skips.append(h)
            if blk.down is not None:
                h = ops.conv3x3(h, blk.down.w, blk.down.b, stride=2)
                skips.append(h)
            if not blk.attns and intra:  # DownBlock2D: added to the block output, which is also its last skip (:1118-1122)
                h = add(h, intra.pop(0))
                skips[-1] = h
        if is_controlnet:
            if len(down_block_additional_residuals) != len(skips):
                raise ValueError(f"expected {len(skips)} down_block_additional_residuals, got "
                                 f"{len(down_block_additional_residuals)}")
            skips = [add(s_, r_) for s_, r_ in zip(skips, down_block_additional_residuals)]
        h = self.mid.res0(h, temb_all)
        h = self.mid.attn(h, ctx, kw, am, eam)
        h = self.mid.res1(h, temb_all)
        if intra and tuple(intra[0].shape) == ((h.shape[0], h.shape[3], h.shape[1], h.shape[2]) if residuals_nchw
                                               else tuple(h.shape)):  # T2I-Adapter-XL (:1145-1151)
            h = add(h, intra.pop(0))
        if is_controlnet:
            h = add(h, mid_block_additional_residual)
        for blk in self.up:
            for j, r in enumerate(blk.resnets):
                h = r(h, temb_all, skip=skips.pop())
                if blk.attns:
                    h = blk.attns[j](h, ctx, kw, am, eam)
            if blk.up is not None:
                h = blk.up.up2x(h)
        n = ops.groupnorm_nhwc(h, self.norm_out.w, self.norm_out.b, groups=self.config.norm_num_groups,
                               eps=self.config.norm_eps, silu=True)
        return ops.conv3x3(n, self.conv_out.w, self.conv_out.b)

    @staticmethod
    def _mask_to_bias(mask, dev):
        """unet_2d_condition.py:916-927: a [batch, key_tokens] keep-mask (1 = keep, 0 = discard; bool / int / float)
        becomes the additive bias (1 - mask) * -10000 with a singleton query axis; anything else is already a bias."""
        if mask is None:
            return None
        mask = mask.to(dev)
        if mask.dim() == 2:
            return ((1.0 - mask.to(torch.float32)) * -10000.0).unsqueeze(1)
        return mask if mask.dtype in (torch.float32, bf16) else mask.to(torch.float32)

    def forward(self, sample, timestep, encoder_hidden_states, class_labels=None, timestep_cond=None,
                attention_mask=None, cross_attention_kwargs: Optional[Dict[str, Any]] = None,
                added_cond_kwargs: Optional[Dict[str, Any]] = None, down_block_additional_residuals=None,
                mid_block_additional_residual=None, down_intrablock_additional_residuals=None,
                encoder_attention_mask=None, return_dict: bool = True):
        """Same signature as the reference (unet_2d_condition.py:809-824). sample: [B,C,H,W] (NCHW, or NHWC when
        config.data_format == "NHWC") host or device tensor; timestep: number, 0-d or 1-d tensor; returns
        UNet2DConditionOutput(sample) or (sample,) in bf16 with the input's layout."""
        from .. import ops
        for name, v in (("class_labels", class_labels), ("timestep_cond", timestep_cond)):
            if v is not None:
                raise NotImplementedError(f"UNet2DConditionModel(b200).forward: `{name}` needs a class / condition "
                                          "embedding this configuration family does not have")
        if self.device is None:
            raise RuntimeError("load_state_dict() must be called before forward()")
        dev = self.device
        sample = sample.to(dev)
        if sample.dtype not in (torch.float32, bf16):
            sample = sample.float()
        ctx = encoder_hidden_states.to(device=dev, dtype=bf16).contiguous()
        nhwc_in = self.config.data_format == "NHWC"
        x = sample.contiguous() if nhwc_in else ops.nchw_to_nhwc(sample.contiguous())
        y = self.forward_nhwc(x, timestep, ctx, added_cond_kwargs, cross_attention_kwargs,
                              attention_mask=self._mask_to_bias(attention_mask, dev),
                              encoder_attention_mask=self._mask_to_bias(encoder_attention_mask, dev),
                              down_block_additional_residuals=down_block_additional_residuals,
                              mid_block_additional_residual=mid_block_additional_residual,
                              down_intrablock_additional_residuals=down_intrablock_additional_residuals,
                              residuals_nchw=not nhwc_in)
        out = y if nhwc_in else ops.nhwc_to_nchw(y, out_dtype=bf16)
        if not return_dict:
            return (out,)
        return UNet2DConditionOutput(sample=out)

    __call__ = forward
