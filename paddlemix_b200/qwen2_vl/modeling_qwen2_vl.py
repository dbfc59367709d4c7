"""Qwen2VLForConditionalGeneration — host-side mirror of paddlemix/models/qwen2_vl/modeling_qwen2_vl.py for the
PREFILL path (forward signature :1382-1399; logits over all positions in fp32, :1474-1475) on sm_90a kernels.

Device graph (one process per GPU, every arithmetic op is a libb200mix kernel):
  ViT (:916-986): PatchEmbed Conv3D == GEMM [T,1176]x[1176,E]; 32 x { LayerNorm -> fused qkv GEMM (+bias) -> 2-D RoPE
  in place (fp32 math, rotate_half) -> varlen block-diagonal flash attention (cu_seqlens) -> proj GEMM (+bias,
  +residual) -> LayerNorm -> fc1 GEMM + quick_gelu -> fc2 GEMM (+residual) }; PatchMerger LN -> GEMM+GELU -> GEMM.
  ViT heads are 80 wide: q/k/v rows and proj columns are zero-padded to 128 once at load time (exact).
  LLM (:813-889): paddlemix_b200.decoder.CausalDecoder with the qkv bias: 28 x { RMSNorm -> fused q|k|v GEMM (+bias)
  -> M-RoPE in place -> causal GQA flash attention (28 q heads / 4 kv heads, d=128) -> o_proj GEMM (+residual) ->
  RMSNorm -> gate|up GEMM with SwiGLU epilogue (interleaved rows) -> down GEMM (+residual) }; final RMSNorm; lm_head
  GEMM with fp32 output. Prefill, eager decode and the CUDA-graph decode step all run that one layer loop; both decode
  paths run the same single-token body (fused RoPE + cache write, GQA-folded attention over the cache).
Host side (pure index math, no arithmetic on activations): get_rope_index (:1217-1360), rot_pos_emb (:940-971),
the cos/sin tables of both rotary embeddings.
"""
from dataclasses import dataclass
from typing import Any, Dict, List, Optional, Union

import torch

from ..decoder import CausalDecoder, rope_cos_sin
from ..modeling import (FrozenDict, bind, device_linear, device_vector, linear_bias, linear_weight, pad_head_cols,
                        pad_head_rows, pad_head_vec, pad_head_width, synthetic_state_dict, to_f32)

bf16 = torch.bfloat16


class Qwen2VLConfig(FrozenDict):
    """Subset of paddlemix's Qwen2VLConfig (configuration_qwen2_vl.py) that the prefill path reads."""

    def __init__(self, hidden_size=3584, intermediate_size=18944, num_hidden_layers=28, num_attention_heads=28,
                 num_key_value_heads=4, vocab_size=152064, rms_norm_eps=1e-6, rope_theta=1000000.0,
                 mrope_section=(16, 24, 24), image_token_id=151655, video_token_id=151656,
                 vision_start_token_id=151652, vision_end_token_id=151653, vision=None, tie_word_embeddings=False,
                 quant_type=None, **kw):
        vision = dict(depth=32, embed_dim=1280, num_heads=16, mlp_ratio=4, in_channels=3, patch_size=14,
                      temporal_patch_size=2, spatial_merge_size=2, hidden_act="quick_gelu") if vision is None else dict(vision)
        super().__init__(hidden_size=hidden_size, intermediate_size=intermediate_size,
                         num_hidden_layers=num_hidden_layers, num_attention_heads=num_attention_heads,
                         num_key_value_heads=num_key_value_heads, vocab_size=vocab_size, rms_norm_eps=rms_norm_eps,
                         rope_theta=rope_theta, mrope_section=tuple(mrope_section), image_token_id=image_token_id,
                         video_token_id=video_token_id, vision_start_token_id=vision_start_token_id,
                         vision_end_token_id=vision_end_token_id, vision=FrozenDict(vision),
                         tie_word_embeddings=bool(tie_word_embeddings), quant_type=quant_type)


@dataclass
class Qwen2VLCausalLMOutputWithPast:
    """modeling_qwen2_vl.py:96-133."""
    loss: Optional[torch.Tensor] = None
    logits: torch.Tensor = None
    past_key_values: Any = None
    hidden_states: Any = None
    attentions: Any = None
    rope_deltas: Optional[torch.Tensor] = None


class KVCache:
    """past_key_values of the LLM (modeling_qwen2_vl.py:591-596 appends along the sequence axis): one preallocated
    [B, max_len, kv_heads, head_dim] bf16 buffer per layer for K (after RoPE) and V, plus the number of valid positions
    (the same for every sequence of the batch). A padded prompt batch keeps its padding inside the cache: `key_bias`
    (fp32 [B, max_len], 0 on real tokens and on the positions still to be generated, -inf on the prompt's padding) is the
    additive key mask every later decode step applies."""

    def __init__(self, n_layers, B, max_len, n_kv, head_dim, device):
        # zero-filled: with kv_lens the kernel multiplies the not-yet-written rows of the last key block by probability 0,
        # which is only 0 when those rows are finite (recycled allocator memory may hold inf / nan bit patterns)
        self.k = [torch.zeros(B, max_len, n_kv, head_dim, device=device, dtype=bf16) for _ in range(n_layers)]
        self.v = [torch.zeros(B, max_len, n_kv, head_dim, device=device, dtype=bf16) for _ in range(n_layers)]
        self.length, self.max_len, self.batch = 0, max_len, B
        self.key_bias = None

    def get_seq_length(self):
        return self.length


class GraphedDecodeStep:
    """One decode step of Qwen2-VL as a CUDA graph (weak point of round 1: 11.7 ms per step, eager launches, host syncs).
    Static device state: newest token ids, the cache row to write and the key count per sequence (both advance INSIDE the
    graph), the 1-D rotary position per sequence (after the prompt all three M-RoPE axes carry the same position,
    cache_position + rope_delta, modeling_qwen2_vl.py:1413-1441) with cos / sin gathered from device tables.
    step(ids) = one small H2D copy (or none, with device ids) + one graph replay; logits stay on the device.
    With a `sampler` (sampling.TokenSampler or beam_search.BeamSearcher) the graph also runs its token selection on the
    step's logits, which writes the next ids straight into the static ids buffer (sampler.ids): step() is then a replay
    only."""

    def __init__(self, model, cache: KVCache, rope_deltas, warmup: int = 2, sampler=None):
        from .. import ops
        if cache.length + warmup > cache.max_len:  # the warm-up steps write cache rows length .. length + warmup - 1
            raise ValueError(f"KV cache has {cache.max_len - cache.length} free positions, the graph's warm-up needs {warmup}")
        self.model, self.cache, self.sampler = model, cache, sampler
        dev, B, hd = model.device, cache.batch, model.head_dim
        P = cache.length
        deltas = torch.zeros(B, dtype=torch.long) if rope_deltas is None else rope_deltas.reshape(B).cpu().long()
        n_pos = cache.max_len + int(deltas.max().clamp(min=0)) + 2
        cos, sin = rope_cos_sin(model.config.rope_theta, hd, n_pos)
        self.cos_table, self.sin_table = cos.to(dev), sin.to(dev)
        self.ids = torch.zeros(B, dtype=torch.long, device=dev) if sampler is None else sampler.ids
        self.pos = (P + deltas).clamp(min=0).to(dev)
        self.rows = (torch.arange(B) * cache.max_len + P).to(dev)
        self.kv_lens = torch.full((B,), P + 1, dtype=torch.int32, device=dev)
        self.cos, self.sin = torch.empty(B, hd, device=dev), torch.empty(B, hd, device=dev)
        self._state0 = (self.pos.clone(), self.rows.clone(), self.kv_lens.clone())

        def body():
            torch.index_select(self.cos_table, 0, self.pos, out=self.cos)  # row gathers (no arithmetic on activations)
            torch.index_select(self.sin_table, 0, self.pos, out=self.sin)
            logits = model.decoder.decode(self.ids, self.cos, self.sin, cache, self.rows, self.kv_lens)
            self.pos.add_(1), self.rows.add_(1), self.kv_lens.add_(1)  # index bookkeeping advances on the device
            return logits

        s = torch.cuda.Stream(device=dev)
        s.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(s):
            for _ in range(warmup):
                body()
        torch.cuda.current_stream(dev).wait_stream(s)
        torch.cuda.synchronize(dev)
        for t, t0 in zip((self.pos, self.rows, self.kv_lens), self._state0):  # undo the warm-up steps' advance
            t.copy_(t0)
        self.graph = torch.cuda.CUDAGraph()
        n0 = ops.launches()
        with torch.cuda.graph(self.graph):
            self.logits = body()
            if sampler is not None:
                sampler(self.logits)
        self.launches_per_step = ops.launches() - n0
        for t, t0 in zip((self.pos, self.rows, self.kv_lens), self._state0):
            t.copy_(t0)

    def step(self, ids=None):
        """ids: int64 [B] (host or device) newest token of each sequence -> fp32 logits [B, vocab] (device, reused).
        With a sampler, ids is None: the previous step's sampler output is already in place."""
        from .. import ops
        if self.cache.length + 1 > self.cache.max_len:
            raise ValueError(f"KV cache is full ({self.cache.max_len} positions)")
        if ids is not None:
            self.ids.copy_(ids.reshape(-1), non_blocking=True)
        elif self.sampler is None:
            raise ValueError("step() needs the newest ids when the graph has no sampler")
        self.graph.replay()
        ops._count(self.launches_per_step)
        self.cache.length += 1
        return self.logits


class Qwen2VLForConditionalGeneration:
    def __init__(self, config: Union[Qwen2VLConfig, Dict[str, Any]]):
        self.config = config if isinstance(config, Qwen2VLConfig) else Qwen2VLConfig(**config)
        c = self.config
        if (c.hidden_size // c.num_attention_heads) * c.num_attention_heads != c.hidden_size:
            raise ValueError(f"hidden_size must be divisible by num_heads (got `hidden_size`: {c.hidden_size}"
                             f" and `num_heads`: {c.num_attention_heads}).")
        self.head_dim = c.hidden_size // c.num_attention_heads
        if self.head_dim not in (64, 128):
            raise NotImplementedError("Qwen2VL(b200): LLM head_dim must be 64 or 128")
        self.v_head = c.vision["embed_dim"] // c.vision["num_heads"]
        self.v_pad = pad_head_width(self.v_head)
        self.decoder = CausalDecoder(c, "model", qkv_bias=True)
        self.dtype = bf16
        self.device = None

    # ------------------------------------------------------------------------------------------------------------
    def state_dict_shapes(self) -> Dict[str, tuple]:
        c, v = self.config, self.config.vision
        E, H = v["embed_dim"], c.hidden_size
        S: Dict[str, tuple] = {}

        def lin(name, i, o, bias=True):
            S[name + ".weight"] = (i, o)
            if bias:
                S[name + ".bias"] = (o,)

        S["visual.patch_embed.proj.weight"] = (E, v["in_channels"], v["temporal_patch_size"], v["patch_size"], v["patch_size"])
        for i in range(v["depth"]):
            b = f"visual.blocks.{i}"
            for n in ("norm1", "norm2"):
                S[f"{b}.{n}.weight"], S[f"{b}.{n}.bias"] = (E,), (E,)
            lin(b + ".attn.qkv", E, 3 * E), lin(b + ".attn.proj", E, E)
            lin(b + ".mlp.fc1", E, E * v["mlp_ratio"]), lin(b + ".mlp.fc2", E * v["mlp_ratio"], E)
        m = E * v["spatial_merge_size"] ** 2
        S["visual.merger.ln_q.weight"], S["visual.merger.ln_q.bias"] = (E,), (E,)
        lin("visual.merger.mlp.0", m, m), lin("visual.merger.mlp.2", m, H)
        S.update(self.decoder.state_dict_shapes())
        return S

    def default_missing_parameters(self, sd) -> Dict[str, Any]:
        """config.tie_word_embeddings (Qwen2-VL-2B): the archive has no lm_head.weight and the reference ties it to the
        embedding table (modeling_qwen2_vl.py:1188); in the Paddle Linear layout that is embed_tokens.weight^T."""
        if self.config.tie_word_embeddings and "lm_head.weight" not in sd and "model.embed_tokens.weight" in sd:
            return {"lm_head.weight": sd["model.embed_tokens.weight"].t()}
        return {}

    def init_synthetic_weights(self, seed: int = 1, device: Union[int, str] = 0):
        def special(name, shp, randn):
            return 0.5 * randn(shp) if name == "model.embed_tokens.weight" else None
        return self.load_state_dict(synthetic_state_dict(self.state_dict_shapes(), seed, device, special), device)

    def load_state_dict(self, P: Dict[str, Any], device: Union[int, str] = 0):
        dev = bind(self, P, device)
        v = self.config.vision
        E, nh = v["embed_dim"], v["num_heads"]
        d, dp = self.v_head, self.v_pad

        self.w_patch = to_f32(P["visual.patch_embed.proj.weight"]).reshape(E, -1).contiguous().to(dev, bf16)
        self.vblocks = []
        for i in range(v["depth"]):
            b = f"visual.blocks.{i}"
            # q|k|v rows are (3, heads, d): padded as 3 * heads heads
            wqkv = pad_head_rows(linear_weight(P, b + ".attn.qkv"), 3 * nh, d, dp)
            bqkv = pad_head_vec(linear_bias(P, b + ".attn.qkv"), 3 * nh, d, dp)
            wp = pad_head_cols(linear_weight(P, b + ".attn.proj"), nh, d, dp)  # [E, heads*dp]
            self.vblocks.append(dict(
                n1=(device_vector(P, b + ".norm1.weight", dev), device_vector(P, b + ".norm1.bias", dev)),
                n2=(device_vector(P, b + ".norm2.weight", dev), device_vector(P, b + ".norm2.bias", dev)),
                qkv=(wqkv.to(dev, bf16), bqkv.to(dev)),
                proj=(wp.to(dev, bf16), device_vector(P, b + ".attn.proj.bias", dev)),
                fc1=device_linear(P, b + ".mlp.fc1", dev), fc2=device_linear(P, b + ".mlp.fc2", dev)))
        self.merger = dict(ln=(device_vector(P, "visual.merger.ln_q.weight", dev),
                               device_vector(P, "visual.merger.ln_q.bias", dev)),
                           m0=device_linear(P, "visual.merger.mlp.0", dev), m2=device_linear(P, "visual.merger.mlp.2", dev))
        self.decoder.load_state_dict(P, dev)
        return self

    # ------------------------------------------------------------------------------------------------------------
    # host-side index math
    # ------------------------------------------------------------------------------------------------------------
    def rot_pos_emb(self, grid_thw: List[List[int]]) -> torch.Tensor:
        """:940-971 -> freqs [T, head_dim/2] (fp32, host)."""
        v = self.config.vision
        m = v["spatial_merge_size"]
        pos = []
        for t, h, w in grid_thw:
            hp = torch.arange(h).unsqueeze(1).expand(-1, w).reshape(h // m, m, w // m, m).permute(0, 2, 1, 3).flatten()
            wp = torch.arange(w).unsqueeze(0).expand(h, -1).reshape(h // m, m, w // m, m).permute(0, 2, 1, 3).flatten()
            pos.append(torch.stack([hp, wp], -1).repeat(t, 1))
        pos = torch.cat(pos, 0)
        dim = self.v_head // 2
        inv_freq = 1.0 / 10000.0 ** (torch.arange(0, dim, 2, dtype=torch.float32) / dim)
        freqs = torch.outer(torch.arange(max(max(h, w) for _, h, w in grid_thw), dtype=torch.float32), inv_freq)
        return freqs[pos].flatten(1)

    def get_rope_index(self, input_ids, image_grid_thw=None, video_grid_thw=None, attention_mask=None):
        """:1217-1360 (image inputs). input_ids host/device int tensor [B,S]. Returns (position_ids [3,B,S], deltas [B,1])."""
        if video_grid_thw is not None:
            raise NotImplementedError("video inputs are outside the hot path")
        c = self.config
        ids_all = input_ids.cpu()
        B, S = ids_all.shape
        if image_grid_thw is None:
            if attention_mask is not None:
                am = attention_mask.cpu().long()
                pos = am.cumsum(-1) - 1
                pos.masked_fill_(am == 0, 1)
                pos = pos.unsqueeze(0).expand(3, -1, -1)
                mx = pos.max(0)[0].max(-1, keepdim=True)[0]
                return pos, mx + 1 - S
            return torch.arange(S).reshape(1, 1, -1).expand(3, B, -1), torch.zeros(B, 1, dtype=torch.long)
        grids = image_grid_thw.tolist() if torch.is_tensor(image_grid_thw) else image_grid_thw
        m = c.vision["spatial_merge_size"]
        position_ids = torch.ones(3, B, S, dtype=torch.long)
        deltas, image_index = [], 0
        for i in range(B):
            keep = torch.ones(S, dtype=torch.bool) if attention_mask is None else attention_mask[i].cpu() == 1
            toks = ids_all[i][keep].tolist()
            starts = [j for j, t in enumerate(toks) if t == c.vision_start_token_id]
            image_nums = sum(1 for j in starts if j + 1 < len(toks) and toks[j + 1] == c.image_token_id)
            plist, st = [], 0
            for _ in range(image_nums):
                ed = toks.index(c.image_token_id, st)
                t, h, w = grids[image_index]
                image_index += 1
                gh, gw = h // m, w // m
                text_len = ed - st
                st_idx = int(plist[-1].max()) + 1 if plist else 0
                plist.append(torch.arange(text_len).reshape(1, -1).expand(3, -1) + st_idx)
                ti = torch.arange(t).reshape(-1, 1).expand(-1, gh * gw).flatten()
                hi = torch.arange(gh).reshape(1, -1, 1).expand(t, -1, gw).flatten()
                wi = torch.arange(gw).reshape(1, 1, -1).expand(t, gh, -1).flatten()
                plist.append(torch.stack([ti, hi, wi]) + text_len + st_idx)
                st = ed + t * gh * gw
            if st < len(toks):
                st_idx = int(plist[-1].max()) + 1 if plist else 0
                plist.append(torch.arange(len(toks) - st).reshape(1, -1).expand(3, -1) + st_idx)
            llm = torch.cat(plist, 1).reshape(3, -1)
            position_ids[:, i, keep] = llm
            deltas.append(int(llm.max()) + 1 - S)
        return position_ids, torch.tensor(deltas).unsqueeze(1)

    def _mrope_tables(self, position_ids):
        """Qwen2RotaryEmbedding (:136-166) + section gather (:212-220) -> cos, sin fp32 [B*S, head_dim] on device."""
        c, hd = self.config, self.head_dim
        cos, sin = rope_cos_sin(c.rope_theta, hd, int(position_ids.max()) + 1)
        cos, sin = cos[position_ids], sin[position_ids]
        sec = list(c.mrope_section) * 2
        cos = torch.cat([x[i % 3] for i, x in enumerate(cos.split(sec, -1))], -1)
        sin = torch.cat([x[i % 3] for i, x in enumerate(sin.split(sec, -1))], -1)
        return cos.reshape(-1, hd).contiguous().to(self.device), sin.reshape(-1, hd).contiguous().to(self.device)

    # ------------------------------------------------------------------------------------------------------------
    def visual(self, pixel_values, grid_thw):
        """Qwen2VisionTransformerPretrainedModel.forward :973-986. pixel_values [T, C*tp*p*p] -> [T/m^2, hidden] bf16."""
        from .. import ops
        from .._lib import ACT_GELU_ERF, ACT_QUICK_GELU
        v = self.config.vision
        E, nh, d, dp = v["embed_dim"], v["num_heads"], self.v_head, self.v_pad
        grids = grid_thw.tolist() if torch.is_tensor(grid_thw) else grid_thw
        x = ops.linear(pixel_values.to(device=self.device, dtype=bf16).contiguous(), self.w_patch)  # [T, E]
        T = x.shape[0]
        freqs = self.rot_pos_emb(grids)
        cos = torch.cat([freqs.cos(), freqs.cos()], -1).contiguous().to(self.device)  # apply_rotary_pos_emb_vision :227-238
        sin = torch.cat([freqs.sin(), freqs.sin()], -1).contiguous().to(self.device)
        cu = [0]
        for t, h, w in grids:
            for _ in range(t):
                cu.append(cu[-1] + h * w)
        cu_t = torch.tensor(cu, dtype=torch.int32, device=self.device)
        inner = nh * dp
        for blk in self.vblocks:
            h1 = ops.layernorm(x, *blk["n1"], eps=1e-6)
            qkv = ops.linear(h1, *blk["qkv"])  # [T, 3*nh*dp]
            q = qkv[:, :inner].unflatten(-1, (nh, dp))
            k = qkv[:, inner:2 * inner].unflatten(-1, (nh, dp))
            vv = qkv[:, 2 * inner:].unflatten(-1, (nh, dp))
            ops.rope_inplace(q, cos, sin, rot_dim=d)
            ops.rope_inplace(k, cos, sin, rot_dim=d)
            a = ops.sdpa(q.unsqueeze(0), k.unsqueeze(0), vv.unsqueeze(0), scale=d ** -0.5, cu_seqlens=cu_t)
            x = ops.linear(a.reshape(T, inner), *blk["proj"], residual=x)
            h2 = ops.layernorm(x, *blk["n2"], eps=1e-6)
            f = ops.linear(h2, *blk["fc1"], act=ACT_QUICK_GELU)
            x = ops.linear(f, *blk["fc2"], residual=x)
        m2 = v["spatial_merge_size"] ** 2
        hq = ops.layernorm(x, *self.merger["ln"], eps=1e-6).reshape(T // m2, E * m2)
        return ops.linear(ops.linear(hq, *self.merger["m0"], act=ACT_GELU_ERF), *self.merger["m2"])

    def forward(self, input_ids=None, attention_mask=None, position_ids=None, past_key_values=None, inputs_embeds=None,
                labels=None, use_cache=None, output_attentions=None, output_hidden_states=None, return_dict=None,
                pixel_values=None, pixel_values_videos=None, image_grid_thw=None, video_grid_thw=None,
                rope_deltas=None):
        """Same signature as the reference (:1382-1399). Prefill (optionally filling a KV cache: use_cache=True) and
        single-token decode (past_key_values = the KVCache a previous call returned; position = past length +
        rope_deltas, :1413-1441). A padded batch (attention_mask [B, S] with zeros, either side) runs with the reference's
        causal + key-padding mask (:403-444, applied at :604-607) and its mask-aware M-RoPE positions; the rows of padding
        tokens carry no meaning (as in the reference). During decode the padding recorded in the cache is used; a mask
        passed then only has to be consistent in shape."""
        if self.device is None:
            raise RuntimeError("load_state_dict() must be called before forward()")
        for name, val in (("labels", labels), ("pixel_values_videos", pixel_values_videos),
                          ("video_grid_thw", video_grid_thw), ("inputs_embeds", inputs_embeds)):
            if val is not None:
                raise NotImplementedError(f"Qwen2VL(b200).forward: `{name}` is outside the inference hot path")
        if output_attentions or output_hidden_states:
            raise NotImplementedError("output_attentions / output_hidden_states are outside the inference hot path")
        c, dev = self.config, self.device
        ids_host = input_ids.cpu()
        B, S = ids_host.shape
        ids_dev = ids_host.to(dev).reshape(-1).contiguous()
        if past_key_values is not None and past_key_values.length > 0:
            # ---- decode: one new token per sequence against the cache, the body GraphedDecodeStep captures ----
            cache, P = past_key_values, past_key_values.length
            if S != 1 or pixel_values is not None:
                raise NotImplementedError("decode takes exactly one new token per sequence and no new images")
            if B != cache.batch:
                raise ValueError(f"decode got {B} sequences for a KV cache of {cache.batch}")
            if position_ids is None:
                if rope_deltas is None:
                    raise ValueError("decode needs the rope_deltas returned by the prefill call (or explicit position_ids)")
                pos = P + rope_deltas.reshape(B, 1).cpu().long()  # arange(1) + cache_position + delta
                position_ids = pos.unsqueeze(0).expand(3, -1, -1)
            if P + 1 > cache.max_len:
                raise ValueError(f"KV cache is full ({cache.max_len} positions)")
            cos, sin = self._mrope_tables(position_ids.cpu())
            rows = (torch.arange(B) * cache.max_len + P).to(dev)
            kv_lens = torch.full((B,), P + 1, dtype=torch.int32, device=dev)
            logits = self.decoder.decode(ids_dev, cos, sin, cache, rows, kv_lens).reshape(B, 1, c.vocab_size)
            cache.length = P + 1
            if return_dict is False:
                return (logits, past_key_values)
            return Qwen2VLCausalLMOutputWithPast(logits=logits, past_key_values=past_key_values, rope_deltas=rope_deltas)
        image_idx = None
        if pixel_values is not None:
            image_idx = (ids_host.reshape(-1) == c.image_token_id).nonzero().reshape(-1).to(dev)
        if position_ids is None:
            position_ids, rope_deltas = self.get_rope_index(ids_host, image_grid_thw, None, attention_mask)
        cos, sin = self._mrope_tables(position_ids.cpu())
        cache = None
        if use_cache:
            cache = past_key_values if past_key_values is not None else KVCache(
                c.num_hidden_layers, B, S + int(getattr(self, "cache_headroom", 256)), c.num_key_value_heads, self.head_dim, dev)
        attn_bias = None
        if attention_mask is not None and not bool((attention_mask == 1).all()):
            if tuple(attention_mask.shape) != (B, S):
                raise ValueError(f"attention_mask {tuple(attention_mask.shape)} does not match input_ids {(B, S)}")
            key_ok = attention_mask.to(dev) == 1
            allowed = torch.ones(S, S, dtype=torch.bool, device=dev).tril()[None] & key_ok[:, None, :]
            attn_bias = torch.zeros(B, 1, S, S, device=dev, dtype=bf16).masked_fill_(~allowed[:, None], float("-inf"))
            if cache is not None:
                cache.key_bias = torch.zeros(B, cache.max_len, device=dev, dtype=torch.float32)
                cache.key_bias[:, :S].masked_fill_(~key_ok, float("-inf"))
        logits = self.prefill_device(ids_dev, B, S, cos, sin, pixel_values, image_grid_thw, image_idx, cache=cache,
                                     attn_bias=attn_bias)
        if return_dict is False:
            return (logits,) if cache is None else (logits, cache)
        return Qwen2VLCausalLMOutputWithPast(logits=logits, past_key_values=cache, rope_deltas=rope_deltas)

    def prefill_device(self, ids_dev, B, S, cos, sin, pixel_values=None, image_grid_thw=None, image_idx=None, cache=None,
                       attn_bias=None):
        """The device part of forward(): everything below is kernel launches on the current stream (no host sync).
        ids_dev int64 [B*S]; cos/sin fp32 [B*S, head_dim] (M-RoPE tables); image_idx int64 [n_image_tokens]; attn_bias =
        additive [B, 1, S, S] mask of a padded batch (causality included) or None for the plain causal mask."""
        from .. import ops
        x = ops.gather_rows(self.decoder.embed, ids_dev)  # [B*S, H]  (embed_tokens, :1443)
        if pixel_values is not None:
            image_embeds = self.visual(pixel_values, image_grid_thw)
            if image_idx.numel() != image_embeds.shape[0]:
                raise ValueError(f"Image features and image tokens do not match: tokens: {image_idx.numel()}, "
                                 f"features {image_embeds.shape[0]}")
            ops.scatter_rows(image_embeds, image_idx, x)  # inputs_embeds[image_mask] = image_embeds (:1449-1452)
        # the cache holds key_states / value_states after RoPE, as the reference's does (:591-596); fp32 logits over all
        # positions (:1474-1475)
        return self.decoder.prefill(x, B, S, cos, sin, cache=cache, attn_bias=attn_bias)

    @torch.no_grad()
    def generate(self, input_ids, pixel_values=None, image_grid_thw=None, max_new_tokens: int = 16, eos_token_id=None,
                 attention_mask=None, *, decode_strategy: str = "greedy_search", do_sample: bool = False,
                 temperature: float = 1.0, top_k: int = 50, top_p: float = 1.0, repetition_penalty: float = 1.0,
                 pad_token_id: Optional[int] = None, generator: Optional[torch.Generator] = None,
                 num_beams: int = 1, length_penalty: float = 1.0, early_stopping: bool = False,
                 num_return_sequences: int = 1, diversity_rate: float = 0.0, num_beam_groups: int = 1,
                 return_scores: bool = False):
        """PaddleNLP GenerationMixin.generate for greedy search, sampling and beam search (generation/utils.py): prefill
        with use_cache, then one decode step per token; returns [B, S + n_new] token ids. Prompts of different lengths
        are LEFT-padded (attention_mask zeros in front), so that every prompt ends at column S - 1.

        Greedy search (the default) takes the argmax. do_sample=True or decode_strategy="sampling" draws from
        softmax(logits / temperature) after top_k / top_p filtering; repetition_penalty applies to both. eos_token_id is
        an int or a list of ints; a sequence that has produced one of them is continued with pad_token_id (default: an
        int eos_token_id) and generation stops at the step where the last sequence finished. The random numbers come
        from a Philox key drawn from `generator` (torch's default CPU generator when None): the same generator state
        gives the same tokens. Everything after the prefill runs as CUDA-graph replays with next-token selection on
        the device (b200mix_sample_tokens).

        Calls that use none of penalty, sampling, an eos list or pad_token_id keep plain greedy decoding, which does
        not pad sequences that have finished.

        decode_strategy="beam_search" keeps num_beams (2 .. 16) beams per prompt (BeamSearchScorer, GNMT length penalty
        ((len + 5) / 6) ** length_penalty, early_stopping, diversity_rate for diverse sibling search) and returns the
        num_return_sequences best hypotheses of prompt b in rows b * num_return_sequences ... (b + 1) *
        num_return_sequences - 1, each ended by eos_token_id (one int or None) when it fits and padded with
        pad_token_id (default eos_token_id); return_scores=True also returns their fp32 scores [B *
        num_return_sequences]. Beam search applies repetition_penalty and ignores do_sample, temperature, top_k, top_p
        and generator, as the reference's beam branch does. The prompt is prefilled once per prompt; after that, token
        selection and KV-cache reordering run on the device inside the graphed decode step
        (b200mix_beam_search_step, b200mix_kv_reorder)."""
        if decode_strategy == "beam_search" or num_beams != 1:
            from ..beam_search import resolve_beam_search_args
            if decode_strategy != "beam_search":
                raise ValueError(f"num_beams={num_beams} needs decode_strategy='beam_search'")
            bargs = resolve_beam_search_args(num_beams, num_return_sequences, length_penalty, early_stopping,
                                             diversity_rate, num_beam_groups, repetition_penalty, eos_token_id,
                                             pad_token_id)
            if attention_mask is not None and not bool((attention_mask[:, -1] == 1).all()):
                raise ValueError("generate(): pad on the left (the last column of attention_mask must be all ones)")
            ids, scores = self._generate_beam_search(input_ids, pixel_values, image_grid_thw, max_new_tokens,
                                                     attention_mask, bargs)
            return (ids, scores) if return_scores else ids
        if return_scores:
            raise ValueError("return_scores=True needs decode_strategy='beam_search'")
        from ..sampling import FINISH_CHECK_INTERVAL, resolve_generation_args, seed_from
        args = resolve_generation_args(decode_strategy, do_sample, temperature, top_k, top_p, repetition_penalty,
                                       eos_token_id, pad_token_id)
        if attention_mask is not None and not bool((attention_mask[:, -1] == 1).all()):
            raise ValueError("generate(): pad on the left (the last column of attention_mask must be all ones)")
        if args.on_device:
            return self._generate_on_device(input_ids, pixel_values, image_grid_thw, max_new_tokens, attention_mask,
                                            args, seed_from(generator) if args.do_sample else 0)
        # plain greedy: graph replays with a device argmax. With an int eos the host reads the tokens back once every
        # FINISH_CHECK_INTERVAL steps; the result ends at the first step by which every row has produced the eos
        self.cache_headroom = max_new_tokens
        out = self.forward(input_ids=input_ids, attention_mask=attention_mask, pixel_values=pixel_values,
                           image_grid_thw=image_grid_thw, use_cache=True)
        toks = [out.logits[:, -1].argmax(-1)]
        if max_new_tokens > 1:
            stepper = GraphedDecodeStep(self, out.past_key_values, out.rope_deltas)
            for i in range(1, max_new_tokens):
                if (eos_token_id is not None and i % FINISH_CHECK_INTERVAL == 0
                        and bool((torch.stack(toks, 1) == eos_token_id).any(1).all())):
                    break
                toks.append(stepper.step(toks[-1]).argmax(-1))
        new = torch.stack(toks, 1).cpu()
        if eos_token_id is not None:
            all_seen = ((new == eos_token_id).cumsum(1) > 0).all(0)  # [n]: every row has an eos among its first j + 1
            if bool(all_seen.any()):
                new = new[:, :int(all_seen.nonzero()[0, 0]) + 1]
        return torch.cat([input_ids.cpu(), new], 1)

    def _generate_on_device(self, input_ids, pixel_values, image_grid_thw, max_new_tokens, attention_mask, args, seed):
        """generate() with b200mix_sample_tokens: the prefill's last logits row gives the first token, then every
        decode step and its token selection is one graph replay; the host reads the all-finished flag once every
        FINISH_CHECK_INTERVAL steps."""
        from ..sampling import FINISH_CHECK_INTERVAL, TokenSampler
        if max_new_tokens < 1:
            raise ValueError(f"max_new_tokens must be >= 1, got {max_new_tokens}")
        self.cache_headroom = max_new_tokens
        out = self.forward(input_ids=input_ids, attention_mask=attention_mask, pixel_values=pixel_values,
                           image_grid_thw=image_grid_thw, use_cache=True)
        sampler = TokenSampler(input_ids, self.config.vocab_size, max_new_tokens, args, seed, self.device)
        sampler(out.logits[:, -1])
        if max_new_tokens > 1:
            stepper = GraphedDecodeStep(self, out.past_key_values, out.rope_deltas, sampler=sampler)
            for i in range(1, max_new_tokens):
                if i % FINISH_CHECK_INTERVAL == 0 and sampler.all_finished():
                    break
                stepper.step()
        n = sampler.n_generated()
        return torch.cat([input_ids.cpu(), sampler.out[:, :n].cpu()], 1)

    def _generate_beam_search(self, input_ids, pixel_values, image_grid_thw, max_new_tokens, attention_mask, args):
        """generate() with beam search: one prefill at B rows, the cache, key mask and rope deltas expanded to B * nb
        rows, selection step 0 on the expanded last logits row, then graph replays of decode + selection + cache
        reorder; the host reads the all-done flag once every FINISH_CHECK_INTERVAL steps."""
        from ..beam_search import BeamSearcher, expand_cache
        from ..sampling import FINISH_CHECK_INTERVAL
        if max_new_tokens < 1:
            raise ValueError(f"max_new_tokens must be >= 1, got {max_new_tokens}")
        nb = args.num_beams
        self.cache_headroom = max_new_tokens
        out = self.forward(input_ids=input_ids, attention_mask=attention_mask, pixel_values=pixel_values,
                           image_grid_thw=image_grid_thw, use_cache=True)
        cache = expand_cache(out.past_key_values, nb)
        deltas = out.rope_deltas.repeat_interleave(nb, 0)
        searcher = BeamSearcher(input_ids, self.config.vocab_size, max_new_tokens, args, cache, self.device)
        searcher(out.logits[:, -1].repeat_interleave(nb, 0))
        del out
        if max_new_tokens > 1:
            stepper = GraphedDecodeStep(self, cache, deltas, sampler=searcher)
            for i in range(1, max_new_tokens):
                if i % FINISH_CHECK_INTERVAL == 0 and searcher.all_done():
                    break
                stepper.step()
        return searcher.finalize()

    __call__ = forward
