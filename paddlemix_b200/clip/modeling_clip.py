"""CLIP text / vision transformers on the sm_90a kernels — host-side mirrors of
ppdiffusers/ppdiffusers/transformers/clip/modeling.py (CLIPTextModel :845-897, CLIPTextModelWithProjection :1231-1304,
CLIPVisionModel :956-1006) — the text encoders in front of the denoising loop (SURVEY.md §8 f2) and LLaVA's vision
tower (paddlemix/models/llava/clip_model.py:945-1078, §8 a19).

Device graph per encoder layer (modeling.py:353-400): LayerNorm -> fused q|k|v GEMM (+bias) -> flash SDPA (causal for the
text tower; q * head_dim**-0.5 is the SDPA scale) -> out_proj GEMM (+bias, +residual) -> LayerNorm -> fc1 GEMM +
quick_gelu / gelu epilogue -> fc2 GEMM (+bias, +residual). Embedding lookups are row gathers; every arithmetic op is a
libb200mix kernel (torch only allocates / copies).
"""
from types import SimpleNamespace
from typing import Any, Dict, Optional, Union

import torch

from ..ppdiffusers.unet_2d_condition import FrozenDict, _to_t

bf16 = torch.bfloat16
_ACTS = {"quick_gelu": 4, "gelu": 2}  # B200MIX_ACT_QUICK_GELU, B200MIX_ACT_GELU_ERF


class _CLIPBase:
    prefix = ""

    def _layer_shapes(self, S):
        c = self.config
        D, I = c.hidden_size, c.intermediate_size
        for i in range(c.num_hidden_layers):
            b = f"{self.prefix}.encoder.layers.{i}"
            for n in ("q_proj", "k_proj", "v_proj", "out_proj"):
                S[f"{b}.self_attn.{n}.weight"], S[f"{b}.self_attn.{n}.bias"] = (D, D), (D,)
            for n in ("layer_norm1", "layer_norm2"):
                S[f"{b}.{n}.weight"], S[f"{b}.{n}.bias"] = (D,), (D,)
            S[f"{b}.mlp.fc1.weight"], S[f"{b}.mlp.fc1.bias"] = (D, I), (I,)
            S[f"{b}.mlp.fc2.weight"], S[f"{b}.mlp.fc2.bias"] = (I, D), (D,)

    def _check(self):
        c = self.config
        self.head_dim = c.hidden_size // c.num_attention_heads
        if self.head_dim * c.num_attention_heads != c.hidden_size:
            raise ValueError(f"embed_dim must be divisible by num_heads (got `embed_dim`: {c.hidden_size} and `num_heads`:"
                             f" {c.num_attention_heads}).")
        if self.head_dim not in (64, 128):
            raise NotImplementedError("CLIP(b200): head_dim must be 64 or 128")
        if c.hidden_act not in _ACTS:
            raise NotImplementedError(f"CLIP(b200): hidden_act {c.hidden_act}")
        self.device, self.dtype = None, bf16

    def _load_layers(self, P, dev):
        c = self.config

        def W(n):  # Paddle Linear [in, out] -> [out, in] bf16
            return _to_t(P[n + ".weight"]).t().contiguous()

        def V(n):
            return _to_t(P[n]).to(dev)

        self.layers = []
        for i in range(c.num_hidden_layers):
            b = f"{self.prefix}.encoder.layers.{i}"
            a = b + ".self_attn"
            wqkv = torch.cat([W(a + ".q_proj"), W(a + ".k_proj"), W(a + ".v_proj")], 0)
            bqkv = torch.cat([_to_t(P[a + f".{n}.bias"]) for n in ("q_proj", "k_proj", "v_proj")], 0)
            self.layers.append(dict(
                ln1=(V(b + ".layer_norm1.weight"), V(b + ".layer_norm1.bias")), ln2=(V(b + ".layer_norm2.weight"), V(b + ".layer_norm2.bias")),
                qkv=(wqkv.to(dev, bf16).contiguous(), bqkv.to(dev)), o=(W(a + ".out_proj").to(dev, bf16), V(a + ".out_proj.bias")),
                fc1=(W(b + ".mlp.fc1").to(dev, bf16), V(b + ".mlp.fc1.bias")), fc2=(W(b + ".mlp.fc2").to(dev, bf16), V(b + ".mlp.fc2.bias"))))

    def _encoder(self, x, causal, mask):
        """CLIPEncoder.forward (:644-723): x bf16 [B,S,D] -> (last, [input of every layer..., last])."""
        from .. import ops
        c = self.config
        B, S, D = x.shape
        H, d, act, eps = c.num_attention_heads, self.head_dim, _ACTS[c.hidden_act], c.layer_norm_eps
        hidden = []
        for L in self.layers:
            hidden.append(x)
            n = ops.layernorm(x, *L["ln1"], eps=eps)
            qkv = ops.linear(n, *L["qkv"])
            q, k, v = (qkv[:, :, i * D:(i + 1) * D].unflatten(-1, (H, d)) for i in range(3))
            o = ops.sdpa(q, k, v, scale=d ** -0.5, causal=causal and mask is None, attn_mask=mask)
            x = ops.linear(o.reshape(B, S, D), *L["o"], residual=x)
            n = ops.layernorm(x, *L["ln2"], eps=eps)
            x = ops.linear(ops.linear(n, *L["fc1"], act=act), *L["fc2"], residual=x)
        hidden.append(x)
        return x, hidden

    def init_synthetic_weights(self, seed: int = 1, device: Union[int, str] = 0):
        dev = torch.device("cuda", device) if isinstance(device, int) else torch.device(device)
        g = torch.Generator(device=dev).manual_seed(seed)
        P = {}
        for name, shp in sorted(self.state_dict_shapes().items()):
            if name.endswith(".weight") and len(shp) >= 2 and "embedding" not in name:
                fan_in = shp[0] if len(shp) == 2 else shp[1] * shp[2] * shp[3]
                t = (torch.rand(shp, generator=g, device=dev) * 2 - 1) / fan_in ** 0.5
            elif "embedding" in name:
                t = 0.3 * torch.randn(shp, generator=g, device=dev)
            elif name.endswith(".weight"):
                t = 1.0 + 0.1 * torch.randn(shp, generator=g, device=dev)
            else:
                t = 0.05 * torch.randn(shp, generator=g, device=dev)
            P[name] = t.to(bf16)
        return self.load_state_dict(P, device=device)


class CLIPTextModel(_CLIPBase):
    """ppdiffusers CLIPTextModel (modeling.py:845-897). forward(input_ids, attention_mask=None, position_ids=None,
    output_hidden_states=None, return_dict=None) -> BaseModelOutputWithPooling-like namespace."""
    prefix = "text_model"
    with_projection = False

    def __init__(self, config: Union[Dict[str, Any], Any] = None, **kw):
        cfg = dict(vocab_size=49408, hidden_size=768, intermediate_size=3072, num_hidden_layers=12, num_attention_heads=12,
                   max_position_embeddings=77, hidden_act="quick_gelu", layer_norm_eps=1e-5, eos_token_id=2, projection_dim=768)
        cfg.update(dict(config or {}))
        cfg.update(kw)
        self.config = FrozenDict(cfg)
        self._check()

    def state_dict_shapes(self) -> Dict[str, tuple]:
        c = self.config
        D = c.hidden_size
        S = {"text_model.embeddings.token_embedding.weight": (c.vocab_size, D),
             "text_model.embeddings.position_embedding.weight": (c.max_position_embeddings, D),
             "text_model.final_layer_norm.weight": (D,), "text_model.final_layer_norm.bias": (D,)}
        self._layer_shapes(S)
        if self.with_projection:
            S["text_projection.weight"] = (D, c.projection_dim)
        return S

    EMBEDDING_KEYS = ("token_embedding.weight", "position_embedding.weight")

    def load_state_dict(self, P: Dict[str, Any], device: Union[int, str] = 0):
        from .. import ops
        dev = torch.device("cuda", device) if isinstance(device, int) else torch.device(device)
        ops.init(dev.index or 0)
        self.device = dev
        missing = [k for k in self.state_dict_shapes() if k not in P]
        if missing:
            raise KeyError(f"state dict is missing {len(missing)} parameters, e.g. {missing[:3]}")
        self.tok = _to_t(P["text_model.embeddings.token_embedding.weight"]).to(dev, bf16).contiguous()
        self.pos = _to_t(P["text_model.embeddings.position_embedding.weight"]).to(dev, bf16).contiguous()
        self.final_ln = (_to_t(P["text_model.final_layer_norm.weight"]).to(dev), _to_t(P["text_model.final_layer_norm.bias"]).to(dev))
        self._load_layers(P, dev)
        self.proj = None
        if self.with_projection:
            self.proj = _to_t(P["text_projection.weight"]).t().contiguous().to(dev, bf16)
        return self

    def forward(self, input_ids=None, attention_mask=None, position_ids=None, output_attentions=None,
                output_hidden_states=None, return_dict=None):
        from .. import ops
        if input_ids is None:
            raise ValueError("You have to specify input_ids")
        if self.device is None:
            raise RuntimeError("load_state_dict() must be called before forward()")
        c, dev = self.config, self.device
        ids_host = input_ids.detach().cpu().reshape(-1, input_ids.shape[-1]).to(torch.int64)
        B, S = ids_host.shape
        ids = ids_host.to(dev)
        x = ops.gather_rows(self.tok, ids.reshape(-1)).reshape(B, 1, S, c.hidden_size)
        pidx = torch.arange(S) if position_ids is None else position_ids.detach().cpu().reshape(-1)[:S].to(torch.int64)
        pos = self.pos[pidx.to(dev)].unsqueeze(0).expand(B, S, c.hidden_size).contiguous().reshape(B, 1, S, c.hidden_size)
        x = ops.add_residual_nhwc(x, pos, r_nchw=False).reshape(B, S, c.hidden_size)  # token + position embeddings (:214-231)
        mask = None
        if attention_mask is not None:  # causal mask + _expand_mask(attention_mask) as one additive bias (:768-776)
            big = torch.finfo(torch.float32).min
            m = torch.full((S, S), big).triu(1)[None, None].expand(B, 1, S, S).clone()
            inv = 1.0 - attention_mask.detach().cpu().reshape(B, 1, 1, S).to(torch.float32)
            m = m + inv.masked_fill(inv.bool(), big)
            mask = torch.clamp(m, min=big).to(dev).contiguous()
        x, hidden = self._encoder(x, causal=True, mask=mask)
        last = ops.layernorm(x, *self.final_ln, eps=c.layer_norm_eps)
        if c.eos_token_id == 2:  # :800-806
            eos = ids_host.argmax(-1)
        else:
            eos = (ids_host == c.eos_token_id).int().argmax(-1)
        rows = (torch.arange(B) * S + eos).to(dev)
        pooled = ops.gather_rows(last.reshape(B * S, -1), rows)
        out = SimpleNamespace(last_hidden_state=last, pooler_output=pooled,
                              hidden_states=tuple(hidden) if output_hidden_states else None, attentions=None)
        if self.proj is not None:
            out.text_embeds = ops.linear(pooled, self.proj)
        if return_dict is False:
            first = (out.text_embeds, last) if self.proj is not None else (last, pooled)
            return first + ((out.hidden_states,) if output_hidden_states else ())
        return out

    __call__ = forward


class CLIPTextModelWithProjection(CLIPTextModel):
    """modeling.py:1231-1304: pooled output through text_projection (no bias) -> text_embeds (SDXL's text_encoder_2)."""
    with_projection = True


class CLIPVisionModel(_CLIPBase):
    """CLIPVisionModel (modeling.py:956-1006; LLaVA's tower, paddlemix/models/llava/clip_model.py:945-1078)."""
    prefix = "vision_model"

    def __init__(self, config: Union[Dict[str, Any], Any] = None, **kw):
        cfg = dict(hidden_size=1024, intermediate_size=4096, num_hidden_layers=24, num_attention_heads=16, image_size=336,
                   patch_size=14, num_channels=3, hidden_act="quick_gelu", layer_norm_eps=1e-5)
        cfg.update(dict(config or {}))
        cfg.update(kw)
        self.config = FrozenDict(cfg)
        self._check()

    def state_dict_shapes(self) -> Dict[str, tuple]:
        c = self.config
        D, p = c.hidden_size, c.patch_size
        S = {"vision_model.embeddings.class_embedding": (D,),
             "vision_model.embeddings.patch_embedding.weight": (D, c.num_channels, p, p),
             "vision_model.embeddings.position_embedding.weight": ((c.image_size // p) ** 2 + 1, D),
             "vision_model.pre_layrnorm.weight": (D,), "vision_model.pre_layrnorm.bias": (D,),
             "vision_model.post_layernorm.weight": (D,), "vision_model.post_layernorm.bias": (D,)}
        self._layer_shapes(S)
        return S

    EMBEDDING_KEYS = ("position_embedding.weight",)

    def load_state_dict(self, P: Dict[str, Any], device: Union[int, str] = 0):
        from .. import ops
        dev = torch.device("cuda", device) if isinstance(device, int) else torch.device(device)
        ops.init(dev.index or 0)
        self.device = dev
        missing = [k for k in self.state_dict_shapes() if k not in P]
        if missing:
            raise KeyError(f"state dict is missing {len(missing)} parameters, e.g. {missing[:3]}")
        c = self.config
        D = c.hidden_size
        w = _to_t(P["vision_model.embeddings.patch_embedding.weight"]).reshape(D, -1)  # [D, C*p*p], columns (c, ph, pw)
        self.k_patch = w.shape[1]
        self.k_pad = (self.k_patch + 7) // 8 * 8  # TMA rows are 16-byte multiples: 3*14*14 = 588 -> 592 (zero columns)
        wp = torch.zeros(D, self.k_pad)
        wp[:, : self.k_patch] = w
        self.w_patch = wp.to(dev, bf16).contiguous()
        self.cls = _to_t(P["vision_model.embeddings.class_embedding"]).to(dev, bf16)
        self.pos = _to_t(P["vision_model.embeddings.position_embedding.weight"]).to(dev, bf16).contiguous()
        self.pre_ln = (_to_t(P["vision_model.pre_layrnorm.weight"]).to(dev), _to_t(P["vision_model.pre_layrnorm.bias"]).to(dev))
        self.post_ln = (_to_t(P["vision_model.post_layernorm.weight"]).to(dev), _to_t(P["vision_model.post_layernorm.bias"]).to(dev))
        self._load_layers(P, dev)
        return self

    def forward(self, pixel_values=None, output_attentions=None, output_hidden_states=None, return_dict=None):
        from .. import ops
        if pixel_values is None:
            raise ValueError("You have to specify pixel_values")
        if self.device is None:
            raise RuntimeError("load_state_dict() must be called before forward()")
        c, dev = self.config, self.device
        x = pixel_values.to(dev)
        if x.dtype not in (torch.float32, bf16):
            x = x.float()
        B, D, p = x.shape[0], c.hidden_size, c.patch_size
        n = (x.shape[2] // p) * (x.shape[3] // p)
        patches = ops.patchify(x.contiguous(), p)  # [B, n, C*p*p] bf16: the stride-p conv as a row gather (:172-179)
        a = torch.zeros(B * n, self.k_pad, device=dev, dtype=bf16)
        a[:, : self.k_patch] = patches.reshape(B * n, self.k_patch)
        pe = ops.linear(a, self.w_patch).reshape(B, n, D)  # patch_embedding has no bias
        emb = torch.empty(B, n + 1, D, device=dev, dtype=bf16)
        emb[:, 0] = self.cls
        emb[:, 1:] = pe
        pos = self.pos[: n + 1].unsqueeze(0).expand(B, n + 1, D).contiguous()
        h = ops.add_residual_nhwc(emb.reshape(B, 1, n + 1, D), pos.reshape(B, 1, n + 1, D), r_nchw=False).reshape(B, n + 1, D)
        h = ops.layernorm(h, *self.pre_ln, eps=c.layer_norm_eps)
        last, hidden = self._encoder(h, causal=False, mask=None)
        pooled = ops.layernorm(last[:, 0].contiguous(), *self.post_ln, eps=c.layer_norm_eps)
        out = SimpleNamespace(last_hidden_state=last, pooler_output=pooled,
                              hidden_states=tuple(hidden) if output_hidden_states else None, attentions=None)
        if return_dict is False:
            return (last, pooled) + ((out.hidden_states,) if output_hidden_states else ())
        return out

    __call__ = forward
