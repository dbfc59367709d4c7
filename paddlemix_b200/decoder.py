"""The Llama-family causal decoder shared by Qwen2-VL's LLM (with a qkv bias) and Llama (without): parameter names, the
device weight layout, the 1-D RoPE table and one layer loop on the sm_90a kernels.

Per layer: RMSNorm -> fused q|k|v GEMM (+bias) -> attention -> o_proj GEMM (+residual) -> RMSNorm -> gate|up GEMM with
SwiGLU epilogue (interleaved rows) -> down GEMM (+residual); then the final RMSNorm and the lm_head GEMM with fp32
output. Only the attention differs between prefill() (RoPE in place, optional KV-cache fill, causal or masked flash
attention) and decode() (one token per sequence, every position on the device: CUDA-graph capturable).

config.quant_type = "weight_only_int8" (PaddleNLP's inference models, qwen/modeling.py:73-85,194-235) quantizes the four
projection matrices of every layer to int8 with one scale per output row at load time; ops.linear takes them in place
of the bf16 weights, so the layer loop is the same. The embedding, lm_head, norms and biases stay as they are.
"""
from typing import Dict

import torch

from .modeling import device_vector, linear_bias, linear_weight, to_f32

bf16 = torch.bfloat16


def rope_cos_sin(theta: float, head_dim: int, n_positions: int):
    """Rotary table (rotate_half convention) for positions 0 .. n_positions - 1: fp32 host cos, sin
    [n_positions, head_dim], each row cat([f, f]) of position * inv_freq."""
    inv_freq = 1.0 / (theta ** (torch.arange(0, head_dim, 2, dtype=torch.float32) / head_dim))
    freqs = torch.arange(n_positions, dtype=torch.float32)[:, None] * inv_freq[None]
    emb = torch.cat([freqs, freqs], -1)
    return emb.cos(), emb.sin()


def decode_attention(qkv, cache_k, cache_v, heads: int, kv_heads: int, head_dim: int, kv_lens, key_bias=None, out=None):
    """Attention of one token per sequence over its KV cache: qkv bf16 [B, (heads + 2 * kv_heads) * head_dim] row view
    (q heads after RoPE), cache_k / cache_v bf16 [B, max_len, kv_heads, head_dim], kv_lens int32 [B] (keys [0, kv_len)
    are read), key_bias fp32 [B, max_len] additive key mask or None. The G = heads / kv_heads query heads that share a
    KV head are presented to the attention kernel as G query rows of ONE head (Sq = G, Hq = kv_heads): one K / V stream
    per KV head instead of one per query head. Returns bf16 [B, heads * head_dim], written into `out` (a row view with a
    contiguous last axis) when it is given."""
    from . import ops
    B, G, qd = qkv.shape[0], heads // kv_heads, heads * head_dim
    kb = None if key_bias is None else key_bias[:, None, None, :]
    if out is not None and (tuple(out.shape) != (B, qd) or out.stride(1) != 1):
        raise ValueError(f"out must be a [{B}, {qd}] view with a contiguous last axis, got {tuple(out.shape)}")
    a = torch.empty(B, qd, device=qkv.device, dtype=bf16) if out is None else out
    qg = qkv.as_strided((B, G, kv_heads, head_dim), (qkv.stride(0), head_dim, G * head_dim, 1), qkv.storage_offset())
    ag = a.as_strided((B, G, kv_heads, head_dim), (a.stride(0), head_dim, G * head_dim, 1), a.storage_offset())
    ops.sdpa(qg, cache_k, cache_v, scale=head_dim ** -0.5, kv_lens=kv_lens, attn_mask=kb, out=ag)
    return a


class CausalDecoder:
    """Embedding table, decoder layers, final norm and lm_head. Parameters are `{prefix}.embed_tokens`,
    `{prefix}.layers.{i}.*`, `{prefix}.norm` and `lm_head` in the Paddle Linear layout ([in, out]); on the device q|k|v
    rows are fused, up / gate rows interleaved, GEMM weights bf16 [N, K] (the layers' four matrices ops.Int8Weight with
    config.quant_type = "weight_only_int8"), norm weights and biases fp32."""

    QUANT_TYPES = (None, "weight_only_int8")

    def __init__(self, config, prefix: str, qkv_bias: bool):
        self.config, self.prefix, self.qkv_bias = config, prefix, qkv_bias
        self.head_dim = config.hidden_size // config.num_attention_heads
        self.quant_type = config.get("quant_type")
        if self.quant_type not in self.QUANT_TYPES:
            raise ValueError(f"quant_type must be one of {self.QUANT_TYPES}, got {self.quant_type!r}")

    def state_dict_shapes(self) -> Dict[str, tuple]:
        c, p = self.config, self.prefix
        H, I = c.hidden_size, c.intermediate_size
        kv = c.num_key_value_heads * self.head_dim
        S = {f"{p}.embed_tokens.weight": (c.vocab_size, H)}
        for i in range(c.num_hidden_layers):
            b = f"{p}.layers.{i}"
            S[b + ".input_layernorm.weight"] = S[b + ".post_attention_layernorm.weight"] = (H,)
            for name, out in (("q_proj", H), ("k_proj", kv), ("v_proj", kv)):
                S[f"{b}.self_attn.{name}.weight"] = (H, out)
                if self.qkv_bias:
                    S[f"{b}.self_attn.{name}.bias"] = (out,)
            S[b + ".self_attn.o_proj.weight"] = (H, H)
            S[b + ".mlp.gate_proj.weight"] = S[b + ".mlp.up_proj.weight"] = (H, I)
            S[b + ".mlp.down_proj.weight"] = (I, H)
        S[f"{p}.norm.weight"] = (H,)
        S["lm_head.weight"] = (H, c.vocab_size)
        return S

    def load_state_dict(self, P: Dict[str, object], dev: torch.device):
        from . import ops
        c, p = self.config, self.prefix
        self.embed = to_f32(P[f"{p}.embed_tokens.weight"]).contiguous().to(dev, bf16)
        if self.quant_type == "weight_only_int8":
            # quantized after fusing (the scales are per output row) from the fp32 values; one bf16 workspace, as large
            # as the largest of the four matrices, serves every layer's GEMMs above the weight-streaming range
            H, I, kv = c.hidden_size, c.intermediate_size, c.num_key_value_heads * self.head_dim
            ws = torch.empty(max((H + 2 * kv) * H, H * H, 2 * I * H, H * I), device=dev, dtype=bf16)
            weight = lambda w: ops.quantize_w8(w.to(dev), ws)  # noqa: E731
        else:
            weight = lambda w: w.to(dev, bf16)  # noqa: E731
        self.layers = []
        for i in range(c.num_hidden_layers):
            b = f"{p}.layers.{i}"
            qkv = [f"{b}.self_attn.{n}_proj" for n in "qkv"]
            gate, up = linear_weight(P, b + ".mlp.gate_proj"), linear_weight(P, b + ".mlp.up_proj")  # [I, H] each
            gu = torch.stack([up, gate], 1).reshape(2 * up.shape[0], -1)  # interleave: 2j = up (value), 2j+1 = gate
            self.layers.append(dict(
                ln1=device_vector(P, b + ".input_layernorm.weight", dev),
                ln2=device_vector(P, b + ".post_attention_layernorm.weight", dev),
                qkv=weight(torch.cat([linear_weight(P, n) for n in qkv], 0)),
                qkv_bias=torch.cat([linear_bias(P, n) for n in qkv], 0).to(dev) if self.qkv_bias else None,
                o=weight(linear_weight(P, b + ".self_attn.o_proj")), gu=weight(gu),
                down=weight(linear_weight(P, b + ".mlp.down_proj"))))
        self.norm_w = device_vector(P, f"{p}.norm.weight", dev)
        self.lm_head = linear_weight(P, "lm_head").to(dev, bf16)
        return self

    def _layers(self, x, attention):
        """x bf16 [M, hidden] -> fp32 logits [M, vocab]; attention(layer index, qkv [M, q|k|v]) -> bf16 [M, heads *
        head_dim]. Kernel launches only."""
        from . import ops
        from ._lib import GLU_SWIGLU
        eps = self.config.rms_norm_eps
        for li, L in enumerate(self.layers):
            h1 = ops.layernorm(x, L["ln1"], None, eps=eps, rms=True)
            a = attention(li, ops.linear(h1, L["qkv"], L["qkv_bias"]))
            x = ops.linear(a, L["o"], residual=x)
            h2 = ops.layernorm(x, L["ln2"], None, eps=eps, rms=True)
            x = ops.linear(ops.linear(h2, L["gu"], glu=GLU_SWIGLU), L["down"], residual=x)  # silu(gate) * up
        hN = ops.layernorm(x, self.norm_w, None, eps=eps, rms=True)
        return ops.linear(hN, self.lm_head, out_fp32=True)

    def prefill(self, x, B, S, cos, sin, cache=None, attn_bias=None):
        """x bf16 [B*S, hidden] input embeddings, cos / sin fp32 [B*S, head_dim]; cache: a KVCache to fill with the RoPE'd
        K and V (its length becomes S); attn_bias: additive [B, 1, S, S] mask of a padded batch (causality included) or
        None for the causal mask. Returns fp32 logits [B, S, vocab]."""
        from . import ops
        c, hd = self.config, self.head_dim
        nh, nkv = c.num_attention_heads, c.num_key_value_heads
        qd, kvd = nh * hd, nkv * hd
        if cache is not None:
            if cache.batch != B or cache.max_len < S:
                raise ValueError(f"KV cache [{cache.batch}, {cache.max_len}] cannot hold a [{B}, {S}] prefill")
            cache.length = S

        def attention(li, qkv):
            q = qkv[:, :qd].unflatten(-1, (nh, hd))
            k = qkv[:, qd:qd + kvd].unflatten(-1, (nkv, hd))
            v = qkv[:, qd + kvd:].unflatten(-1, (nkv, hd))
            ops.rope_inplace(q, cos, sin)
            ops.rope_inplace(k, cos, sin)
            if cache is not None:
                cache.k[li][:, :S].copy_(k.unflatten(0, (B, S)))
                cache.v[li][:, :S].copy_(v.unflatten(0, (B, S)))
            a = ops.sdpa(q.unflatten(0, (B, S)), k.unflatten(0, (B, S)), v.unflatten(0, (B, S)), scale=hd ** -0.5,
                         causal=attn_bias is None, attn_mask=attn_bias)
            return a.reshape(B * S, qd)
        return self._layers(x, attention).reshape(B, S, c.vocab_size)

    def decode(self, ids, cos, sin, cache, rows, kv_lens):
        """One token per sequence against `cache`: ids int64 [B], cos / sin fp32 [B, head_dim] for its position, rows
        int64 [B] = b * max_len + position (the flattened cache row its K / V go to), kv_lens int32 [B] = position + 1,
        all on the device. Attention is decode_attention() over the cache. Returns fp32 logits [B, vocab]; advancing
        cache.length is the caller's job."""
        from . import ops
        c, hd = self.config, self.head_dim
        nh, nkv = c.num_attention_heads, c.num_key_value_heads
        kvd = nkv * hd

        def attention(li, qkv):
            ops.decode_rope_cache(qkv, nh, nkv, hd, cos, sin, rows, cache.k[li].view(-1, kvd), cache.v[li].view(-1, kvd))
            return decode_attention(qkv, cache.k[li], cache.v[li], nh, nkv, hd, kv_lens, cache.key_bias)
        return self._layers(ops.gather_rows(self.embed, ids), attention)
