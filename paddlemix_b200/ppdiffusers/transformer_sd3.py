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

from .unet_2d_condition import FrozenDict, _to_t

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
        dev = torch.device("cuda", device) if isinstance(device, int) else torch.device(device)
        g = torch.Generator(device=dev).manual_seed(seed)
        P = {}
        for name, shp in sorted(self.state_dict_shapes().items()):
            if name == "pos_embed.pos_embed":
                t = 0.5 * torch.randn(shp, generator=g, device=dev)
            elif name.endswith(".weight"):
                fan_in = shp[0] if len(shp) == 2 else shp[1] * shp[2] * shp[3]
                t = (torch.rand(shp, generator=g, device=dev) * 2 - 1) / fan_in ** 0.5
            else:
                t = 0.05 * torch.randn(shp, generator=g, device=dev)
            P[name] = t.to(bf16)
        return self.load_state_dict(P, device=device)

    def load_state_dict(self, P: Dict[str, Any], device: Union[int, str] = 0):
        from .. import ops
        dev = torch.device("cuda", device) if isinstance(device, int) else torch.device(device)
        ops.init(dev.index or 0)
        self.device = dev
        missing = [k for k in self.state_dict_shapes() if k not in P]
        if missing:
            raise KeyError(f"state dict is missing {len(missing)} parameters, e.g. {missing[:3]}")
        c, D = self.config, self.inner_dim

        def W(name):  # Paddle Linear [in, out] -> [out, in] bf16
            return _to_t(P[name + ".weight"]).t().contiguous().to(dev, bf16)

        def Bv(name):
            return _to_t(P[name + ".bias"]).to(dev)

        self.w_patch = _to_t(P["pos_embed.proj.weight"]).reshape(D, -1).contiguous().to(dev, bf16)  # [D, C*p*p]
        self.b_patch = Bv("pos_embed.proj")
        self.pos_table = _to_t(P["pos_embed.pos_embed"]).reshape(c.pos_embed_max_size, c.pos_embed_max_size, D).to(dev)
        self._pos_cache = {}
        self.t1, self.t2 = (W("time_text_embed.timestep_embedder.linear_1"), Bv("time_text_embed.timestep_embedder.linear_1")), \
                           (W("time_text_embed.timestep_embedder.linear_2"), Bv("time_text_embed.timestep_embedder.linear_2"))
        self.p1, self.p2 = (W("time_text_embed.text_embedder.linear_1"), Bv("time_text_embed.text_embedder.linear_1")), \
                           (W("time_text_embed.text_embedder.linear_2"), Bv("time_text_embed.text_embedder.linear_2"))
        self.ctx_emb = (W("context_embedder"), Bv("context_embedder"))
        # one GEMM for every AdaLN projection: rows = [blk0.norm1 (6D) | blk0.norm1_context (6D|2D) | ... | norm_out (2D)]
        ws, bs, self.mod_off = [], [], []
        off = 0
        self.blocks = []
        for i in range(c.num_layers):
            b = f"transformer_blocks.{i}"
            last = i == c.num_layers - 1
            blk = dict(last=last)
            for key in ("norm1", "norm1_context"):
                w, bias = _to_t(P[f"{b}.{key}.linear.weight"]).t().contiguous(), _to_t(P[f"{b}.{key}.linear.bias"])
                blk[key + "_off"] = off
                off += w.shape[0]
                ws.append(w), bs.append(bias)
            blk["w_qkv"] = torch.cat([W(f"{b}.attn.to_q"), W(f"{b}.attn.to_k"), W(f"{b}.attn.to_v")], 0).contiguous()
            blk["b_qkv"] = torch.cat([Bv(f"{b}.attn.to_q"), Bv(f"{b}.attn.to_k"), Bv(f"{b}.attn.to_v")], 0).contiguous()
            blk["w_cqkv"] = torch.cat([W(f"{b}.attn.add_q_proj"), W(f"{b}.attn.add_k_proj"), W(f"{b}.attn.add_v_proj")], 0).contiguous()
            blk["b_cqkv"] = torch.cat([Bv(f"{b}.attn.add_q_proj"), Bv(f"{b}.attn.add_k_proj"), Bv(f"{b}.attn.add_v_proj")], 0).contiguous()
            blk["w_o"], blk["b_o"] = W(f"{b}.attn.to_out.0"), Bv(f"{b}.attn.to_out.0")
            blk["ff1"], blk["ff2"] = (W(f"{b}.ff.net.0.proj"), Bv(f"{b}.ff.net.0.proj")), (W(f"{b}.ff.net.2"), Bv(f"{b}.ff.net.2"))
            if last:
                blk["ctx_ln_bias"] = _to_t(P[f"{b}.norm1_context.norm.bias"]).to(dev)
            else:
                blk["w_co"], blk["b_co"] = W(f"{b}.attn.to_add_out"), Bv(f"{b}.attn.to_add_out")
                blk["cff1"] = (W(f"{b}.ff_context.net.0.proj"), Bv(f"{b}.ff_context.net.0.proj"))
                blk["cff2"] = (W(f"{b}.ff_context.net.2"), Bv(f"{b}.ff_context.net.2"))
            self.blocks.append(blk)
        w, bias = _to_t(P["norm_out.linear.weight"]).t().contiguous(), _to_t(P["norm_out.linear.bias"])
        self.norm_out_off = off
        off += w.shape[0]
        ws.append(w), bs.append(bias)
        self.mod_w = torch.cat(ws, 0).to(dev, bf16).contiguous()
        self.mod_b = torch.cat(bs, 0).to(dev).contiguous()
        self.norm_out_bias = _to_t(P["norm_out.norm.bias"]).to(dev)
        self.proj_out = (W("proj_out"), Bv("proj_out"))
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

    def forward(self, hidden_states, encoder_hidden_states=None, pooled_projections=None, timestep=None,
                joint_attention_kwargs: Optional[Dict[str, Any]] = None, return_dict: bool = True):
        """Same signature as the reference (transformer_sd3.py:279-287). hidden_states [B,C,H,W] (fp32 / bf16),
        encoder_hidden_states [B,L,joint_attention_dim], pooled_projections [B,pooled_dim], timestep [B] or scalar."""
        from .. import ops
        from .._lib import ACT_GELU_TANH, ACT_SILU
        if self.device is None:
            raise RuntimeError("load_state_dict() must be called before forward()")
        if joint_attention_kwargs:
            extra = {k: v for k, v in joint_attention_kwargs.items() if k != "scale"}
            if extra:
                raise NotImplementedError(f"joint_attention_kwargs {list(extra)} are outside the hot path")
        dev, c, D = self.device, self.config, self.inner_dim
        Hh, hd = c.num_attention_heads, c.attention_head_dim
        x_in = hidden_states.to(dev)
        if x_in.dtype not in (torch.float32, bf16):
            x_in = x_in.float()
        B, _, H, Wd = x_in.shape
        ps = c.patch_size
        h, w = H // ps, Wd // ps
        n = h * w
        ctx = encoder_hidden_states.to(device=dev, dtype=bf16).contiguous()
        L = ctx.shape[1]
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

        S = n + L
        for blk in self.blocks:
            last = blk["last"]
            m1 = mod[:, blk["norm1_off"]:]
            # AdaLayerNormZero chunk order: shift_msa, scale_msa, gate_msa, shift_mlp, scale_mlp, gate_mlp
            nx = ops.layernorm(x, eps=1e-6, scale=m1[:, D:], shift=m1[:, 0:], rows_per_group=n)
            mc = mod[:, blk["norm1_context_off"]:]
            if last:  # AdaLayerNormContinuous: (scale, shift); its LayerNorm carries a bias and no weight
                nc = ops.layernorm(cst, None, blk["ctx_ln_bias"], eps=1e-6, scale=mc[:, 0:], shift=mc[:, D:], rows_per_group=L)
            else:
                nc = ops.layernorm(cst, eps=1e-6, scale=mc[:, D:], shift=mc[:, 0:], rows_per_group=L)
            qkv = torch.empty(B, S, 3 * D, device=dev, dtype=bf16)
            ops.linear_batched(nx, blk["w_qkv"], blk["b_qkv"], out=qkv[:, :n])
            ops.linear_batched(nc, blk["w_cqkv"], blk["b_cqkv"], out=qkv[:, n:])
            q, k, v = (qkv[:, :, i * D:(i + 1) * D].unflatten(-1, (Hh, hd)) for i in range(3))
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
        mo = mod[:, self.norm_out_off:]
        xn = ops.layernorm(x, None, self.norm_out_bias, eps=1e-6, scale=mo[:, 0:], shift=mo[:, D:], rows_per_group=n)
        y = ops.linear(xn, *self.proj_out)  # [B, n, p*p*oc]
        out = ops.unpatchify(y, self.out_channels, h, w, ps, out_dtype=bf16)
        if not return_dict:
            return (out,)
        return Transformer2DModelOutput(sample=out)

    __call__ = forward
