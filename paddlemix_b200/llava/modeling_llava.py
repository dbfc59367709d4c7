"""LLaVA on the sm_90a kernels: the Llama decoder prefill (PaddleNLP/paddlenlp/transformers/llama/modeling.py: RMSNorm
:386-420, rotary :534-555, attention :197-330, decoder layers, lm head) and the LLaVA composition around it
(paddlemix/models/llava/modeling.py:47-120, base_model.py:136-330): CLIP vision tower -> feature_select
(clip_encoder.py:49-57) -> mm_projector mlp2x_gelu (mm_projector.py:45-58) -> image features spliced in place of each
sample's IMAGE_TOKEN_INDEX placeholder -> causal prefill -> fp32 logits.

The decoder is paddlemix_b200.decoder.CausalDecoder without the qkv bias, run as its prefill. Device graph per decoder
layer: RMSNorm -> fused q|k|v GEMM -> RoPE in place (rotate_half, fp32 math) -> causal GQA flash attention (d = 128) ->
o_proj GEMM (+residual) -> RMSNorm -> gate|up GEMM with the SwiGLU epilogue (interleaved rows) -> down GEMM
(+residual). SURVEY.md §8 row a19.
"""
from types import SimpleNamespace
from typing import Any, Dict, Union

import torch

from ..clip import CLIPVisionModel
from ..decoder import CausalDecoder, rope_cos_sin
from ..modeling import FrozenDict, bind, device_linear

bf16 = torch.bfloat16
IMAGE_TOKEN_INDEX = -200  # paddlemix/models/llava/constants.py


class LlamaForCausalLM:
    """Prefill-only mirror of PaddleNLP's LlamaForCausalLM: forward(input_ids | inputs_embeds) -> logits (fp32)."""
    PREFIX = "llama"

    def __init__(self, config: Union[Dict[str, Any], Any] = None, **kw):
        cfg = dict(vocab_size=32000, hidden_size=4096, intermediate_size=11008, num_hidden_layers=32, num_attention_heads=32,
                   num_key_value_heads=32, rms_norm_eps=1e-5, rope_theta=10000.0, quant_type=None)
        cfg.update(dict(config or {}))
        cfg.update(kw)
        self.config = FrozenDict(cfg)
        c = self.config
        self.head_dim = c.hidden_size // c.num_attention_heads
        if self.head_dim * c.num_attention_heads != c.hidden_size:
            raise ValueError(f"hidden_size must be divisible by num_heads (got `hidden_size`: {c.hidden_size} and "
                             f"`num_heads`: {c.num_attention_heads}).")
        if self.head_dim not in (64, 128):
            raise NotImplementedError("Llama(b200): head_dim must be 64 or 128")
        self.decoder = CausalDecoder(c, self.PREFIX, qkv_bias=False)
        self.device, self.dtype = None, bf16

    EMBEDDING_KEYS = ("embed_tokens.weight",)

    def state_dict_shapes(self) -> Dict[str, tuple]:
        return self.decoder.state_dict_shapes()

    def load_state_dict(self, P: Dict[str, Any], device: Union[int, str] = 0):
        self.decoder.load_state_dict(P, bind(self, P, device))
        return self

    def _rope_tables(self, S):
        """LlamaRotaryEmbedding: cos / sin fp32 [S, head_dim] for positions 0..S-1 (host index math)."""
        cos, sin = rope_cos_sin(self.config.rope_theta, self.head_dim, S)
        return cos.to(self.device), sin.to(self.device)

    def prefill_embeds(self, x):
        """x: bf16 [B, S, H] input embeddings -> fp32 logits [B, S, vocab] (causal, positions 0..S-1)."""
        B, S, H = x.shape
        cos, sin = self._rope_tables(S)
        # one cos / sin row per token of the flattened [B*S] axis
        return self.decoder.prefill(x.reshape(B * S, H).contiguous(), B, S, cos.repeat(B, 1), sin.repeat(B, 1))

    def embed_tokens(self, ids_dev):
        from .. import ops
        return ops.gather_rows(self.decoder.embed, ids_dev.reshape(-1))

    def forward(self, input_ids=None, inputs_embeds=None, attention_mask=None, return_dict=True):
        if self.device is None:
            raise RuntimeError("load_state_dict() must be called before forward()")
        if attention_mask is not None and not bool(torch.as_tensor(attention_mask).all()):
            raise NotImplementedError("Llama(b200) prefill: padded batches are outside this path")
        if inputs_embeds is None:
            B, S = input_ids.shape
            inputs_embeds = self.embed_tokens(input_ids.to(self.device)).reshape(B, S, -1)
        logits = self.prefill_embeds(inputs_embeds.to(self.device, bf16))
        return SimpleNamespace(logits=logits) if return_dict else (logits,)

    __call__ = forward


class LlavaLlamaForCausalLM(LlamaForCausalLM):
    """paddlemix LlavaLlamaForCausalLM (modeling.py:47-120): forward(input_ids, images) -> logits over the merged sequence.
    Every sample must hold the same number of IMAGE_TOKEN_INDEX placeholders at positions that give equal merged lengths
    (one image per sample in the LLaVA-1.5 prompt format); ragged merges need the padded-batch path, which is refused."""

    def __init__(self, config=None, vision_config=None, mm_vision_select_layer=-2, mm_vision_select_feature="patch",
                 mm_projector_type="mlp2x_gelu", **kw):
        super().__init__(config, **kw)
        if mm_projector_type != "mlp2x_gelu":
            raise NotImplementedError(f"mm_projector_type={mm_projector_type}")
        self.vision_tower = CLIPVisionModel(vision_config)
        self.select_layer, self.select_feature = mm_vision_select_layer, mm_vision_select_feature

    VT = "llama.vision_tower.vision_tower."

    def state_dict_shapes(self):
        S = super().state_dict_shapes()
        for k, v in self.vision_tower.state_dict_shapes().items():
            S[self.VT + k] = v
        Dv, H = self.vision_tower.config.hidden_size, self.config.hidden_size
        S["llama.mm_projector.0.weight"], S["llama.mm_projector.0.bias"] = (Dv, H), (H,)
        S["llama.mm_projector.2.weight"], S["llama.mm_projector.2.bias"] = (H, H), (H,)
        return S

    def load_state_dict(self, P, device=0):
        super().load_state_dict(P, device)  # binds and checks every key of this class's shapes, the vision tower's too
        self.vision_tower.load_state_dict({k[len(self.VT):]: v for k, v in P.items() if k.startswith(self.VT)}, device)
        self.proj0 = device_linear(P, "llama.mm_projector.0", self.device)
        self.proj2 = device_linear(P, "llama.mm_projector.2", self.device)
        return self

    def encode_images(self, images):
        """vision tower -> feature_select -> mm_projector (base_model.py:106-116)."""
        from .. import ops
        from .._lib import ACT_GELU_ERF
        hs = self.vision_tower(pixel_values=images, output_hidden_states=True).hidden_states
        f = hs[self.select_layer]
        if self.select_feature == "patch":
            f = f[:, 1:]
        elif self.select_feature != "cls_patch":
            raise ValueError(f"Unexpected select feature: {self.select_feature}")
        f = f.contiguous()
        return ops.linear(ops.linear(f, *self.proj0, act=ACT_GELU_ERF), *self.proj2)

    def forward(self, input_ids=None, images=None, attention_mask=None, return_dict=True):
        if images is None:
            return super().forward(input_ids=input_ids, attention_mask=attention_mask, return_dict=return_dict)
        if attention_mask is not None and not bool(torch.as_tensor(attention_mask).all()):
            raise NotImplementedError("Llava(b200) prefill: padded batches are outside this path")
        ids = input_ids.detach().cpu()
        feats = self.encode_images(images)  # [B, n_img, H]
        rows = []
        for b in range(ids.shape[0]):  # prepare_inputs_labels_for_multimodal (base_model.py:225-290)
            pos = (ids[b] == IMAGE_TOKEN_INDEX).nonzero().flatten().tolist()
            parts, prev = [], 0
            for i, p in enumerate(pos):
                if p > prev:
                    parts.append(self.embed_tokens(ids[b, prev:p].to(self.device)))
                if len(pos) != 1:
                    raise NotImplementedError("Llava(b200): one image per sample")
                parts.append(feats[b])
                prev = p + 1
            if prev < ids.shape[1]:
                parts.append(self.embed_tokens(ids[b, prev:].to(self.device)))
            rows.append(torch.cat(parts, 0))
        if len({r.shape[0] for r in rows}) != 1:
            raise NotImplementedError("Llava(b200) prefill: merged sequences of different lengths need the padded-batch path")
        logits = self.prefill_embeds(torch.stack(rows, 0))
        return SimpleNamespace(logits=logits) if return_dict else (logits,)

    __call__ = forward
