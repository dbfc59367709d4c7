"""SD3Transformer2DModel — host-side mirror of ppdiffusers.models.transformer_sd3.SD3Transformer2DModel
(ppdiffusers/models/transformer_sd3.py:44-122 constructor, :279-287 forward signature) on sm_90a kernels.

The reference offers two block stacks: 24 x JointTransformerBlock (attention.py:96-214) and its own fused
replacement SimplifiedSD3 (simplified_sd3.py:43-160, Triton ops). This graph goes further along the same lines:
  * all 49 AdaLN projections (norm1 / norm1_context of every block + norm_out) are ONE GEMM per forward whose fp32
    output is sliced into the shift / scale / gate vectors (the reference runs 49 tiny Linear layers per step);
  * LayerNorm + (1+scale), shift modulation is one kernel (= the Triton adaptive_layer_norm);
  * q|k|v of each stream are one GEMM writing straight into the token range of the joint [B, n_img+n_txt, 3D]
    buffer (batched-strided epilogue) — the reference's paddle.concat x3 / split_concat_kernel never happens;
  * gate * (.) + residual of both the attention out-projection and the FF second Linear are GEMM epilogues (the
    Triton fused_adaLN_scale_residual does the residual half in the next LayerNorm);
  * PatchEmbed = patchify kernel + GEMM with the cropped sin-cos table added in the epilogue.
"""
from dataclasses import dataclass
from typing import Any, Dict, Optional, Union

import torch

from ..modeling import (FrozenDict, bind, device_linear, device_vector, linear_bias, linear_weight, synthetic_state_dict,
                        to_f32)

bf16 = torch.bfloat16


@dataclass
class Transformer2DModelOutput:
    """ppdiffusers.models.transformer_2d.Transformer2DModelOutput."""
    sample: torch.Tensor = None


class SD3Transformer2DModel:
    def __init__(self, sample_size: int = 128, patch_size: int = 2, in_channels: int = 16, num_layers: int = 18,
                 attention_head_dim: int = 64, num_attention_heads: int = 18, joint_attention_dim: int = 4096,
                 caption_projection_dim: int = 1152, pooled_projection_dim: int = 2048, out_channels: int = 16,
                 pos_embed_max_size: int = 96):
        self.config = FrozenDict(sample_size=sample_size, patch_size=patch_size, in_channels=in_channels,
                                 num_layers=num_layers, attention_head_dim=attention_head_dim,
                                 num_attention_heads=num_attention_heads, joint_attention_dim=joint_attention_dim,
                                 caption_projection_dim=caption_projection_dim,
                                 pooled_projection_dim=pooled_projection_dim, out_channels=out_channels,
                                 pos_embed_max_size=pos_embed_max_size)
        self.out_channels = out_channels if out_channels is not None else in_channels
        self.inner_dim = num_attention_heads * attention_head_dim
        if attention_head_dim not in (64, 128):
            raise NotImplementedError("SD3Transformer2DModel(b200): attention_head_dim must be 64 or 128")
        if caption_projection_dim != self.inner_dim:
            raise ValueError("caption_projection_dim must equal num_attention_heads * attention_head_dim")
        self.dtype = bf16
        self.device = None

    # ------------------------------------------------------------------------------------------------------------
    def state_dict_shapes(self) -> Dict[str, tuple]:
        c, D = self.config, self.inner_dim
        p = c.patch_size
        S: Dict[str, tuple] = {}

        def lin(name, i, o):
            S[name + ".weight"], S[name + ".bias"] = (i, o), (o,)

        S["pos_embed.proj.weight"], S["pos_embed.proj.bias"] = (D, c.in_channels, p, p), (D,)
        S["pos_embed.pos_embed"] = (1, c.pos_embed_max_size ** 2, D)
        lin("time_text_embed.timestep_embedder.linear_1", 256, D), lin("time_text_embed.timestep_embedder.linear_2", D, D)
        lin("time_text_embed.text_embedder.linear_1", c.pooled_projection_dim, D)
        lin("time_text_embed.text_embedder.linear_2", D, D)
        lin("context_embedder", c.joint_attention_dim, c.caption_projection_dim)
        for i in range(c.num_layers):
            b = f"transformer_blocks.{i}"
            last = i == c.num_layers - 1
            lin(b + ".norm1.linear", D, 6 * D)
            lin(b + ".norm1_context.linear", D, 2 * D if last else 6 * D)
            if last:
                S[b + ".norm1_context.norm.bias"] = (D,)
            for n in ("to_q", "to_k", "to_v", "add_q_proj", "add_k_proj", "add_v_proj", "to_out.0"):
                lin(f"{b}.attn.{n}", D, D)
            lin(b + ".ff.net.0.proj", D, 4 * D), lin(b + ".ff.net.2", 4 * D, D)
            if not last:
                lin(b + ".attn.to_add_out", D, D)
                lin(b + ".ff_context.net.0.proj", D, 4 * D), lin(b + ".ff_context.net.2", 4 * D, D)
        lin("norm_out.linear", D, 2 * D)
        S["norm_out.norm.bias"] = (D,)
        lin("proj_out", D, p * p * self.out_channels)
        return S

    def default_missing_parameters(self, sd) -> Dict[str, Any]:
        """AdaLayerNormContinuous builds its LayerNorm with weight_attr=False, bias_attr=True on Paddle, so Paddle
        archives carry a `norm.bias` that torch-format (format='pt') SD3 archives do not have; the reference leaves it
        at its zero initialisation in that case (from_pretrained ignores missing keys with a default)."""
        D = self.inner_dim
        last = self.config.num_layers - 1
        return {k: torch.zeros(D) for k in ("norm_out.norm.bias", f"transformer_blocks.{last}.norm1_context.norm.bias")
                if k not in sd}

    def init_synthetic_weights(self, seed: int = 1, device: Union[int, str] = 0):
        def special(name, shp, randn):
            return 0.5 * randn(shp) if name == "pos_embed.pos_embed" else None
        return self.load_state_dict(synthetic_state_dict(self.state_dict_shapes(), seed, device, special), device)

    def load_state_dict(self, P: Dict[str, Any], device: Union[int, str] = 0):
        dev = bind(self, P, device)
        c, D = self.config, self.inner_dim

        self.w_patch = to_f32(P["pos_embed.proj.weight"]).reshape(D, -1).contiguous().to(dev, bf16)  # [D, C*p*p]
        self.b_patch = device_vector(P, "pos_embed.proj.bias", dev)
        self.pos_table = to_f32(P["pos_embed.pos_embed"]).reshape(c.pos_embed_max_size, c.pos_embed_max_size, D).to(dev)
        self._pos_cache = {}
        self.t1 = device_linear(P, "time_text_embed.timestep_embedder.linear_1", dev)
        self.t2 = device_linear(P, "time_text_embed.timestep_embedder.linear_2", dev)
        self.p1 = device_linear(P, "time_text_embed.text_embedder.linear_1", dev)
        self.p2 = device_linear(P, "time_text_embed.text_embedder.linear_2", dev)
        self.ctx_emb = device_linear(P, "context_embedder", dev)
        # one GEMM for every AdaLN projection: rows = [blk0.norm1 (6D) | blk0.norm1_context (6D|2D) | ... | norm_out (2D)]
        ws, bs, self.mod_off = [], [], []
        off = 0
        self.blocks = []
        for i in range(c.num_layers):
            b = f"transformer_blocks.{i}"
            last = i == c.num_layers - 1
            blk = dict(last=last)
            for key in ("norm1", "norm1_context"):
                w, bias = linear_weight(P, f"{b}.{key}.linear"), linear_bias(P, f"{b}.{key}.linear")
                blk[key + "_off"] = off
                off += w.shape[0]
                ws.append(w), bs.append(bias)
            for key, names in (("qkv", ("to_q", "to_k", "to_v")), ("cqkv", ("add_q_proj", "add_k_proj", "add_v_proj"))):
                blk["w_" + key] = torch.cat([linear_weight(P, f"{b}.attn.{n}") for n in names], 0).to(dev, bf16)
                blk["b_" + key] = torch.cat([linear_bias(P, f"{b}.attn.{n}") for n in names], 0).to(dev)
            blk["w_o"], blk["b_o"] = device_linear(P, f"{b}.attn.to_out.0", dev)
            blk["ff1"], blk["ff2"] = device_linear(P, f"{b}.ff.net.0.proj", dev), device_linear(P, f"{b}.ff.net.2", dev)
            if last:
                blk["ctx_ln_bias"] = device_vector(P, f"{b}.norm1_context.norm.bias", dev)
            else:
                blk["w_co"], blk["b_co"] = device_linear(P, f"{b}.attn.to_add_out", dev)
                blk["cff1"] = device_linear(P, f"{b}.ff_context.net.0.proj", dev)
                blk["cff2"] = device_linear(P, f"{b}.ff_context.net.2", dev)
            self.blocks.append(blk)
        w, bias = linear_weight(P, "norm_out.linear"), linear_bias(P, "norm_out.linear")
        self.norm_out_off = off
        off += w.shape[0]
        ws.append(w), bs.append(bias)
        self.mod_w = torch.cat(ws, 0).to(dev, bf16).contiguous()
        self.mod_b = torch.cat(bs, 0).to(dev).contiguous()
        self.norm_out_bias = device_vector(P, "norm_out.norm.bias", dev)
        self.proj_out = device_linear(P, "proj_out", dev)
        return self

    # ------------------------------------------------------------------------------------------------------------
    def _pos(self, h, w):
        """PatchEmbed.cropped_pos_embed (embeddings.py:186-210), cached per latent size as a bf16 [h*w, D] table."""
        key = (h, w)
        t = self._pos_cache.get(key)
        if t is None:
            mx = self.config.pos_embed_max_size
            if h > mx:
                raise ValueError(f"Height ({h}) cannot be greater than `pos_embed_max_size`: {mx}.")
            if w > mx:
                raise ValueError(f"Width ({w}) cannot be greater than `pos_embed_max_size`: {mx}.")
            top, left = (mx - h) // 2, (mx - w) // 2
            t = self.pos_table[top:top + h, left:left + w].reshape(h * w, -1).to(bf16).contiguous()
            self._pos_cache[key] = t
        return t

    def _embed(self, hidden_states, encoder_hidden_states, pooled_projections, timestep):
        """PatchEmbed, CombinedTimestepTextProjEmbeddings, the context embedder and the one GEMM for every AdaLN
        projection. Returns (x [B, n, D] bf16, context stream [B, L, D] bf16, temb [B, D] bf16, mod [B, sum] fp32,
        (h, w))."""
        from .. import ops
        from .._lib import ACT_SILU
        dev, c = self.device, self.config
        x_in = hidden_states.to(dev)
        if x_in.dtype not in (torch.float32, bf16):
            x_in = x_in.float()
        B, _, H, Wd = x_in.shape
        ps = c.patch_size
        h, w = H // ps, Wd // ps
        n = h * w
        ctx = encoder_hidden_states.to(device=dev, dtype=bf16).contiguous()
        pooled = pooled_projections.to(device=dev, dtype=bf16).contiguous()
        t = timestep if torch.is_tensor(timestep) else torch.tensor([float(timestep)])
        t = t.to(device=dev, dtype=torch.float32).reshape(-1)
        if t.numel() == 1 and B > 1:
            t = t.expand(B)
        t = t.contiguous()

        # PatchEmbed (embeddings.py:212-247): conv p x p stride p == GEMM on patch rows, + cropped pos embed
        x = ops.linear(ops.patchify(x_in.contiguous(), ps), self.w_patch, self.b_patch, residual=self._pos(h, w),
                       residual_row_mod=n)  # [B, n, D]
        # CombinedTimestepTextProjEmbeddings (embeddings.py:530-546)
        t_proj = ops.timestep_embedding(t, 256, flip_sin_to_cos=True, downscale_freq_shift=0.0)
        t_emb = ops.linear(ops.linear(t_proj, *self.t1, act=ACT_SILU), *self.t2)
        temb = ops.linear(ops.linear(pooled, *self.p1, act=ACT_SILU), *self.p2, residual=t_emb)
        mod = ops.linear(ops.activation(temb, ACT_SILU), self.mod_w, self.mod_b, out_fp32=True)  # [B, sum] fp32
        cst = ops.linear(ctx, *self.ctx_emb)  # [B, L, D]
        return x, cst, temb, mod, (h, w)

    def _block(self, i, x, cst, mod, n, L):
        """JointTransformerBlock i on the image stream x [B, n, D] and the context stream cst [B, L, D], with its AdaLN
        vectors read from mod. Returns (x, cst); the last block (context_pre_only) returns cst unchanged."""
        from .. import ops
        from .._lib import ACT_GELU_TANH
        c, D = self.config, self.inner_dim
        Hh, hd = c.num_attention_heads, c.attention_head_dim
        B, S = x.shape[0], n + L
        blk = self.blocks[i]
        last = blk["last"]
        m1 = mod[:, blk["norm1_off"]:]
        # AdaLayerNormZero chunk order: shift_msa, scale_msa, gate_msa, shift_mlp, scale_mlp, gate_mlp
        nx = ops.layernorm(x, eps=1e-6, scale=m1[:, D:], shift=m1[:, 0:], rows_per_group=n)
        mc = mod[:, blk["norm1_context_off"]:]
        if last:  # AdaLayerNormContinuous: (scale, shift); its LayerNorm carries a bias and no weight
            nc = ops.layernorm(cst, None, blk["ctx_ln_bias"], eps=1e-6, scale=mc[:, 0:], shift=mc[:, D:], rows_per_group=L)
        else:
            nc = ops.layernorm(cst, eps=1e-6, scale=mc[:, D:], shift=mc[:, 0:], rows_per_group=L)
        qkv = torch.empty(B, S, 3 * D, device=x.device, dtype=bf16)
        ops.linear_batched(nx, blk["w_qkv"], blk["b_qkv"], out=qkv[:, :n])
        ops.linear_batched(nc, blk["w_cqkv"], blk["b_cqkv"], out=qkv[:, n:])
        q, k, v = (qkv[:, :, j * D:(j + 1) * D].unflatten(-1, (Hh, hd)) for j in range(3))
        o = ops.sdpa(q, k, v, scale=hd ** -0.5).reshape(B, S, D)
        x_new = torch.empty_like(x)
        ops.linear_batched(o[:, :n], blk["w_o"], blk["b_o"], out=x_new, row_gate=m1[:, 2 * D:], residual=x)
        nx2 = ops.layernorm(x_new, eps=1e-6, scale=m1[:, 4 * D:], shift=m1[:, 3 * D:], rows_per_group=n)
        ff = ops.linear(nx2, *blk["ff1"], act=ACT_GELU_TANH)
        x = ops.linear(ff, *blk["ff2"], row_gate=m1[:, 5 * D:], rows_per_group=n, residual=x_new)
        if not last:
            c_new = torch.empty_like(cst)
            ops.linear_batched(o[:, n:], blk["w_co"], blk["b_co"], out=c_new, row_gate=mc[:, 2 * D:], residual=cst)
            nc2 = ops.layernorm(c_new, eps=1e-6, scale=mc[:, 4 * D:], shift=mc[:, 3 * D:], rows_per_group=L)
            cff = ops.linear(nc2, *blk["cff1"], act=ACT_GELU_TANH)
            cst = ops.linear(cff, *blk["cff2"], row_gate=mc[:, 5 * D:], rows_per_group=L, residual=c_new)
        return x, cst

    def _final(self, x, mod, h, w):
        """norm_out (AdaLayerNormContinuous), proj_out and unpatchify: bf16 [B, out_channels, h*p, w*p]."""
        from .. import ops
        D, n = self.inner_dim, h * w
        mo = mod[:, self.norm_out_off:]
        xn = ops.layernorm(x, None, self.norm_out_bias, eps=1e-6, scale=mo[:, 0:], shift=mo[:, D:], rows_per_group=n)
        y = ops.linear(xn, *self.proj_out)  # [B, n, p*p*oc]
        return ops.unpatchify(y, self.out_channels, h, w, self.config.patch_size, out_dtype=bf16)

    def forward(self, hidden_states, encoder_hidden_states=None, pooled_projections=None, timestep=None,
                joint_attention_kwargs: Optional[Dict[str, Any]] = None, return_dict: bool = True):
        """Same signature as the reference (transformer_sd3.py:279-287). hidden_states [B,C,H,W] (fp32 / bf16),
        encoder_hidden_states [B,L,joint_attention_dim], pooled_projections [B,pooled_dim], timestep [B] or scalar."""
        if self.device is None:
            raise RuntimeError("load_state_dict() must be called before forward()")
        if joint_attention_kwargs:
            extra = {k: v for k, v in joint_attention_kwargs.items() if k != "scale"}
            if extra:
                raise NotImplementedError(f"joint_attention_kwargs {list(extra)} are outside the hot path")
        x, cst, _, mod, (h, w) = self._embed(hidden_states, encoder_hidden_states, pooled_projections, timestep)
        n, L = h * w, cst.shape[1]
        for i in range(len(self.blocks)):
            x, cst = self._block(i, x, cst, mod, n, L)
        out = self._final(x, mod, h, w)
        if not return_dict:
            return (out,)
        return Transformer2DModelOutput(sample=out)

    __call__ = forward
