"""Qwen2VLForConditionalGeneration — host-side mirror of paddlemix/models/qwen2_vl/modeling_qwen2_vl.py for the
PREFILL path (forward signature :1382-1399; logits over all positions in fp32, :1474-1475) on sm_90a kernels.

Device graph (one process per GPU, every arithmetic op is a libb200mix kernel):
  ViT (:916-986): PatchEmbed Conv3D == GEMM [T,1176]x[1176,E]; 32 x { LayerNorm -> fused qkv GEMM (+bias) -> 2-D RoPE
  in place (fp32 math, rotate_half) -> varlen block-diagonal flash attention (cu_seqlens) -> proj GEMM (+bias,
  +residual) -> LayerNorm -> fc1 GEMM + quick_gelu -> fc2 GEMM (+residual) }; PatchMerger LN -> GEMM+GELU -> GEMM.
  ViT heads are 80 wide: q/k/v rows and proj columns are zero-padded to 128 once at load time (exact).
  LLM (:813-889): 28 x { RMSNorm -> fused q|k|v GEMM (+bias) -> M-RoPE in place -> causal GQA flash attention
  (28 q heads / 4 kv heads, d=128) -> o_proj GEMM (+residual) -> RMSNorm -> gate|up GEMM with SwiGLU epilogue
  (interleaved rows) -> down GEMM (+residual) }; final RMSNorm; lm_head GEMM with fp32 output.
Host side (pure index math, no arithmetic on activations): get_rope_index (:1217-1360), rot_pos_emb (:940-971),
the cos/sin tables of both rotary embeddings.
"""
import math
from dataclasses import dataclass
from typing import Any, Dict, List, Optional, Union

import torch

from ..ppdiffusers.unet_2d_condition import FrozenDict, _to_t

bf16 = torch.bfloat16


class Qwen2VLConfig(FrozenDict):
    """Subset of paddlemix's Qwen2VLConfig (configuration_qwen2_vl.py) that the prefill path reads."""

    def __init__(self, hidden_size=3584, intermediate_size=18944, num_hidden_layers=28, num_attention_heads=28,
                 num_key_value_heads=4, vocab_size=152064, rms_norm_eps=1e-6, rope_theta=1000000.0,
                 mrope_section=(16, 24, 24), image_token_id=151655, video_token_id=151656,
                 vision_start_token_id=151652, vision_end_token_id=151653, vision=None, tie_word_embeddings=False,
                 **kw):
        vision = dict(depth=32, embed_dim=1280, num_heads=16, mlp_ratio=4, in_channels=3, patch_size=14,
                      temporal_patch_size=2, spatial_merge_size=2, hidden_act="quick_gelu") if vision is None else dict(vision)
        super().__init__(hidden_size=hidden_size, intermediate_size=intermediate_size,
                         num_hidden_layers=num_hidden_layers, num_attention_heads=num_attention_heads,
                         num_key_value_heads=num_key_value_heads, vocab_size=vocab_size, rms_norm_eps=rms_norm_eps,
                         rope_theta=rope_theta, mrope_section=tuple(mrope_section), image_token_id=image_token_id,
                         video_token_id=video_token_id, vision_start_token_id=vision_start_token_id,
                         vision_end_token_id=vision_end_token_id, vision=FrozenDict(vision),
                         tie_word_embeddings=bool(tie_word_embeddings))


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
    step(ids) = one small H2D copy (or none, with device ids) + one graph replay; logits stay on the device."""

    def __init__(self, model, cache: KVCache, rope_deltas, warmup: int = 2):
        from .. import ops
        self.model, self.cache = model, cache
        dev, B, hd = model.device, cache.batch, model.head_dim
        c = model.config
        P = cache.length
        deltas = torch.zeros(B, dtype=torch.long) if rope_deltas is None else rope_deltas.reshape(B).cpu().long()
        n_pos = cache.max_len + int(deltas.max().clamp(min=0)) + 2
        inv_freq = 1.0 / (c.rope_theta ** (torch.arange(0, hd, 2, dtype=torch.float32) / hd))
        fr = torch.arange(n_pos, dtype=torch.float32)[:, None] * inv_freq[None]
        emb = torch.cat([fr, fr], -1)
        self.cos_table, self.sin_table = emb.cos().contiguous().to(dev), emb.sin().contiguous().to(dev)
        self.ids = torch.zeros(B, dtype=torch.long, device=dev)
        self.pos = (P + deltas).clamp(min=0).to(dev)
        self.rows = (torch.arange(B) * cache.max_len + P).to(dev)
        self.kv_lens = torch.full((B,), P + 1, dtype=torch.int32, device=dev)
        self.cos, self.sin = torch.empty(B, hd, device=dev), torch.empty(B, hd, device=dev)
        self._state0 = (self.pos.clone(), self.rows.clone(), self.kv_lens.clone())

        def body():
            torch.index_select(self.cos_table, 0, self.pos, out=self.cos)  # row gathers (no arithmetic on activations)
            torch.index_select(self.sin_table, 0, self.pos, out=self.sin)
            logits = model.decode_body_static(self.ids, self.cos, self.sin, cache, self.rows, self.kv_lens)
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
        self.launches_per_step = ops.launches() - n0
        for t, t0 in zip((self.pos, self.rows, self.kv_lens), self._state0):
            t.copy_(t0)

    def step(self, ids):
        """ids: int64 [B] (host or device) newest token of each sequence -> fp32 logits [B, vocab] (device, reused)."""
        from .. import ops
        if self.cache.length + 1 > self.cache.max_len:
            raise ValueError(f"KV cache is full ({self.cache.max_len} positions)")
        self.ids.copy_(ids.reshape(-1), non_blocking=True)
        self.graph.replay()
        ops._count(self.launches_per_step)
        self.cache.length += 1
        return self.logits


def _pad_rows(w, heads, d, dp):  # [heads*d, in] -> [heads*dp, in]
    if d == dp:
        return w
    out = torch.zeros(heads, dp, w.shape[-1], device=w.device)
    out[:, :d] = w.reshape(heads, d, -1)
    return out.reshape(heads * dp, -1)


def _pad_vec(b, heads, d, dp):
    if d == dp:
        return b
    out = torch.zeros(heads, dp, device=b.device)
    out[:, :d] = b.reshape(heads, d)
    return out.reshape(-1)


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
        self.v_pad = 64 if self.v_head <= 64 else 128
        self.dtype = bf16
        self.device = None

    # ------------------------------------------------------------------------------------------------------------
    def state_dict_shapes(self) -> Dict[str, tuple]:
        c, v = self.config, self.config.vision
        E, H, I = v["embed_dim"], c.hidden_size, c.intermediate_size
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
        S["model.embed_tokens.weight"] = (c.vocab_size, H)
        kv = c.num_key_value_heads * self.head_dim
        for i in range(c.num_hidden_layers):
            b = f"model.layers.{i}"
            S[b + ".input_layernorm.weight"] = (H,)
            S[b + ".post_attention_layernorm.weight"] = (H,)
            lin(b + ".self_attn.q_proj", H, H), lin(b + ".self_attn.k_proj", H, kv), lin(b + ".self_attn.v_proj", H, kv)
            lin(b + ".self_attn.o_proj", H, H, bias=False)
            lin(b + ".mlp.gate_proj", H, I, bias=False), lin(b + ".mlp.up_proj", H, I, bias=False)
            lin(b + ".mlp.down_proj", I, H, bias=False)
        S["model.norm.weight"] = (H,)
        lin("lm_head", H, c.vocab_size, bias=False)
        return S

    def default_missing_parameters(self, sd) -> Dict[str, Any]:
        """config.tie_word_embeddings (Qwen2-VL-2B): the archive has no lm_head.weight and the reference ties it to the
        embedding table (modeling_qwen2_vl.py:1188); in the Paddle Linear layout that is embed_tokens.weight^T."""
        if self.config.tie_word_embeddings and "lm_head.weight" not in sd and "model.embed_tokens.weight" in sd:
            return {"lm_head.weight": sd["model.embed_tokens.weight"].t()}
        return {}

    def init_synthetic_weights(self, seed: int = 1, device: Union[int, str] = 0):
        dev = torch.device("cuda", device) if isinstance(device, int) else torch.device(device)
        g = torch.Generator(device=dev).manual_seed(seed)
        P = {}
        for name, shp in sorted(self.state_dict_shapes().items()):
            if name == "model.embed_tokens.weight":
                t = 0.5 * torch.randn(shp, generator=g, device=dev)
            elif name.endswith(".weight") and len(shp) >= 2:
                fan_in = shp[0] if len(shp) == 2 else math.prod(shp[1:])
                t = (torch.rand(shp, generator=g, device=dev) * 2 - 1) / fan_in ** 0.5
            elif name.endswith(".weight"):
                t = 1.0 + 0.1 * torch.randn(shp, generator=g, device=dev)
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
        c, v = self.config, self.config.vision
        E, nh = v["embed_dim"], v["num_heads"]
        d, dp = self.v_head, self.v_pad

        def W(name):
            return _to_t(P[name + ".weight"]).t().contiguous()

        def Bv(name):
            return _to_t(P[name + ".bias"])

        def dv(t, dtype=None):
            return t.contiguous().to(dev, dtype) if dtype is not None else t.contiguous().to(dev)

        self.w_patch = dv(_to_t(P["visual.patch_embed.proj.weight"]).reshape(E, -1), bf16)
        self.vblocks = []
        for i in range(v["depth"]):
            b = f"visual.blocks.{i}"
            wqkv, bqkv = W(b + ".attn.qkv"), Bv(b + ".attn.qkv")  # [3E, E] rows ordered (3, heads, d)
            wq = torch.cat([_pad_rows(wqkv[j * E:(j + 1) * E], nh, d, dp) for j in range(3)], 0)
            bq = torch.cat([_pad_vec(bqkv[j * E:(j + 1) * E], nh, d, dp) for j in range(3)], 0)
            wp = W(b + ".attn.proj")  # [E, heads*d] -> [E, heads*dp]
            if d != dp:
                wp3 = torch.zeros(E, nh, dp, device=wp.device)
                wp3[:, :, :d] = wp.reshape(E, nh, d)
                wp = wp3.reshape(E, nh * dp)
            self.vblocks.append(dict(
                n1=(dv(_to_t(P[b + ".norm1.weight"])), dv(Bv(b + ".norm1"))), n2=(dv(_to_t(P[b + ".norm2.weight"])), dv(Bv(b + ".norm2"))),
                qkv=(dv(wq, bf16), dv(bq)), proj=(dv(wp, bf16), dv(Bv(b + ".attn.proj"))),
                fc1=(dv(W(b + ".mlp.fc1"), bf16), dv(Bv(b + ".mlp.fc1"))), fc2=(dv(W(b + ".mlp.fc2"), bf16), dv(Bv(b + ".mlp.fc2")))))
        self.merger = dict(ln=(dv(_to_t(P["visual.merger.ln_q.weight"])), dv(Bv("visual.merger.ln_q"))),
                           m0=(dv(W("visual.merger.mlp.0"), bf16), dv(Bv("visual.merger.mlp.0"))),
                           m2=(dv(W("visual.merger.mlp.2"), bf16), dv(Bv("visual.merger.mlp.2"))))
        self.embed = dv(_to_t(P["model.embed_tokens.weight"]), bf16)
        self.layers = []
        for i in range(c.num_hidden_layers):
            b = f"model.layers.{i}"
            wqkv = torch.cat([W(b + ".self_attn.q_proj"), W(b + ".self_attn.k_proj"), W(b + ".self_attn.v_proj")], 0)
            bqkv = torch.cat([Bv(b + ".self_attn.q_proj"), Bv(b + ".self_attn.k_proj"), Bv(b + ".self_attn.v_proj")], 0)
            gate, up = W(b + ".mlp.gate_proj"), W(b + ".mlp.up_proj")  # [I, H] each
            gu = torch.stack([up, gate], 1).reshape(2 * up.shape[0], -1)  # interleave: 2j = up (value), 2j+1 = gate
            self.layers.append(dict(ln1=dv(_to_t(P[b + ".input_layernorm.weight"])), ln2=dv(_to_t(P[b + ".post_attention_layernorm.weight"])),
                                    qkv=(dv(wqkv, bf16), dv(bqkv)), o=dv(W(b + ".self_attn.o_proj"), bf16),
                                    gu=dv(gu, bf16), down=dv(W(b + ".mlp.down_proj"), bf16)))
        self.norm_w = dv(_to_t(P["model.norm.weight"]))
        self.lm_head = dv(W("lm_head"), bf16)
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
        inv_freq = 1.0 / (c.rope_theta ** (torch.arange(0, hd, 2, dtype=torch.float32) / hd))
        n = int(position_ids.max()) + 1
        freqs = torch.einsum("i,j->ij", torch.arange(n, dtype=torch.float32), inv_freq)
        emb = torch.cat([freqs, freqs], -1)
        cos, sin = emb.cos()[position_ids], emb.sin()[position_ids]
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
            # ---- decode: one new token per sequence against the cache ----
            if S != 1 or pixel_values is not None:
                raise NotImplementedError("decode takes exactly one new token per sequence and no new images")
            if position_ids is None:
                if rope_deltas is None:
                    raise ValueError("decode needs the rope_deltas returned by the prefill call (or explicit position_ids)")
                pos = past_key_values.length + rope_deltas.reshape(B, 1).cpu().long()  # arange(1) + cache_position + delta
                position_ids = pos.unsqueeze(0).expand(3, -1, -1)
            cos, sin = self._mrope_tables(position_ids.cpu())
            logits = self.decode_device(ids_dev, B, cos, sin, past_key_values).reshape(B, 1, c.vocab_size)
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
        from .._lib import GLU_SWIGLU
        c, hd = self.config, self.head_dim
        nh, nkv = c.num_attention_heads, c.num_key_value_heads
        x = ops.gather_rows(self.embed, ids_dev)  # [B*S, H]  (embed_tokens, :1443)
        if pixel_values is not None:
            image_embeds = self.visual(pixel_values, image_grid_thw)
            if image_idx.numel() != image_embeds.shape[0]:
                raise ValueError(f"Image features and image tokens do not match: tokens: {image_idx.numel()}, "
                                 f"features {image_embeds.shape[0]}")
            ops.scatter_rows(image_embeds, image_idx, x)  # inputs_embeds[image_mask] = image_embeds (:1449-1452)
        qd, kvd = nh * hd, nkv * hd
        if cache is not None:
            if cache.batch != B or cache.max_len < S:
                raise ValueError(f"KV cache [{cache.batch}, {cache.max_len}] cannot hold a [{B}, {S}] prefill")
            cache.length = S
        for li, L in enumerate(self.layers):
            h1 = ops.layernorm(x, L["ln1"], None, eps=c.rms_norm_eps, rms=True)
            qkv = ops.linear(h1, *L["qkv"])  # [B*S, qd + 2*kvd]
            q = qkv[:, :qd].unflatten(-1, (nh, hd))
            k = qkv[:, qd:qd + kvd].unflatten(-1, (nkv, hd))
            vv = qkv[:, qd + kvd:].unflatten(-1, (nkv, hd))
            ops.rope_inplace(q, cos, sin)
            ops.rope_inplace(k, cos, sin)
            if cache is not None:  # key_states / value_states after RoPE are what the reference caches (:591-596)
                cache.k[li][:, :S].copy_(k.unflatten(0, (B, S)))
                cache.v[li][:, :S].copy_(vv.unflatten(0, (B, S)))
            a = ops.sdpa(q.unflatten(0, (B, S)), k.unflatten(0, (B, S)), vv.unflatten(0, (B, S)), scale=hd ** -0.5,
                         causal=attn_bias is None, attn_mask=attn_bias)
            x = ops.linear(a.reshape(B * S, qd), L["o"], residual=x)
            h2 = ops.layernorm(x, L["ln2"], None, eps=c.rms_norm_eps, rms=True)
            g = ops.linear(h2, L["gu"], glu=GLU_SWIGLU)  # silu(gate) * up
            x = ops.linear(g, L["down"], residual=x)
        hN = ops.layernorm(x, self.norm_w, None, eps=c.rms_norm_eps, rms=True)
        return ops.linear(hN, self.lm_head, out_fp32=True).reshape(B, S, c.vocab_size)  # fp32 logits (:1474-1475)

    def decode_device(self, ids_dev, B, cos, sin, cache: KVCache):
        """One decode step (Qwen2VLDecoderLayer.forward :829-889 with a cache): ids_dev int64 [B] = the newest token of each
        sequence, cos / sin fp32 [B, head_dim] for its position. Appends K / V at cache.length, attends over the
        cache.length + 1 cached positions (GQA, no mask needed: everything cached is in the past), returns fp32 logits
        [B, vocab] and advances the cache. Kernel launches only."""
        from .. import ops
        from .._lib import GLU_SWIGLU
        c, hd = self.config, self.head_dim
        nh, nkv = c.num_attention_heads, c.num_key_value_heads
        P = cache.length
        if P + 1 > cache.max_len:
            raise ValueError(f"KV cache is full ({cache.max_len} positions)")
        x = ops.gather_rows(self.embed, ids_dev)  # [B, H]
        qd, kvd = nh * hd, nkv * hd
        for li, L in enumerate(self.layers):
            h1 = ops.layernorm(x, L["ln1"], None, eps=c.rms_norm_eps, rms=True)
            qkv = ops.linear(h1, *L["qkv"])  # [B, qd + 2*kvd]
            q = qkv[:, :qd].unflatten(-1, (nh, hd))
            k = qkv[:, qd:qd + kvd].unflatten(-1, (nkv, hd))
            vv = qkv[:, qd + kvd:].unflatten(-1, (nkv, hd))
            ops.rope_inplace(q, cos, sin)
            ops.rope_inplace(k, cos, sin)
            cache.k[li][:, P].copy_(k)
            cache.v[li][:, P].copy_(vv)
            kb = None if cache.key_bias is None else cache.key_bias[:, None, None, :P + 1]
            a = ops.sdpa(q.unsqueeze(1), cache.k[li][:, :P + 1], cache.v[li][:, :P + 1], scale=hd ** -0.5, attn_mask=kb)  # [B,1,nh,hd]
            x = ops.linear(a.reshape(B, qd), L["o"], residual=x)
            h2 = ops.layernorm(x, L["ln2"], None, eps=c.rms_norm_eps, rms=True)
            g = ops.linear(h2, L["gu"], glu=GLU_SWIGLU)
            x = ops.linear(g, L["down"], residual=x)
        cache.length = P + 1
        hN = ops.layernorm(x, self.norm_w, None, eps=c.rms_norm_eps, rms=True)
        return ops.linear(hN, self.lm_head, out_fp32=True)

    def decode_body_static(self, ids_dev, cos, sin, cache: KVCache, rows, kv_lens):
        """decode_device with every position-dependent quantity on the DEVICE (CUDA-graph capturable): `rows` int64 [B] =
        b * max_len + position of the new token (row of the flattened cache to write), `kv_lens` int32 [B] = keys to attend
        to (position + 1). The G = heads / kv_heads query heads that share a KV head are presented to the attention kernel
        as G query rows of ONE head (Sq = G, Hq = Hkv): one K / V stream per KV head instead of one per query head."""
        from .. import ops
        from .._lib import GLU_SWIGLU
        c, hd = self.config, self.head_dim
        nh, nkv = c.num_attention_heads, c.num_key_value_heads
        G = nh // nkv
        B = ids_dev.shape[0]
        x = ops.gather_rows(self.embed, ids_dev)
        qd, kvd = nh * hd, nkv * hd
        for li, L in enumerate(self.layers):
            h1 = ops.layernorm(x, L["ln1"], None, eps=c.rms_norm_eps, rms=True)
            qkv = ops.linear(h1, *L["qkv"])
            ops.decode_rope_cache(qkv, nh, nkv, hd, cos, sin, rows, cache.k[li].view(-1, kvd), cache.v[li].view(-1, kvd))
            a = torch.empty(B, qd, device=x.device, dtype=bf16)
            qg = qkv.as_strided((B, G, nkv, hd), (qkv.stride(0), hd, G * hd, 1), qkv.storage_offset())
            ag = a.as_strided((B, G, nkv, hd), (qd, hd, G * hd, 1))
            kb = None if cache.key_bias is None else cache.key_bias[:, None, None, :]
            ops.sdpa(qg, cache.k[li], cache.v[li], scale=hd ** -0.5, kv_lens=kv_lens, attn_mask=kb, out=ag)
            x = ops.linear(a, L["o"], residual=x)
            h2 = ops.layernorm(x, L["ln2"], None, eps=c.rms_norm_eps, rms=True)
            x = ops.linear(ops.linear(h2, L["gu"], glu=GLU_SWIGLU), L["down"], residual=x)
        hN = ops.layernorm(x, self.norm_w, None, eps=c.rms_norm_eps, rms=True)
        return ops.linear(hN, self.lm_head, out_fp32=True)

    @torch.no_grad()
    def generate(self, input_ids, pixel_values=None, image_grid_thw=None, max_new_tokens: int = 16, eos_token_id=None,
                 attention_mask=None):
        """Greedy decoding (generation_utils' default `do_sample=False`): prefill with use_cache, then one decode step per
        token; returns [B, S + n_new] token ids (generation stops early when every sequence has produced EOS). Prompts of
        different lengths are LEFT-padded (attention_mask zeros in front), so that every prompt ends at column S - 1."""
        B, S = input_ids.shape
        if attention_mask is not None and not bool((attention_mask[:, -1] == 1).all()):
            raise ValueError("generate(): pad on the left (the last column of attention_mask must be all ones)")
        self.cache_headroom = max_new_tokens
        out = self.forward(input_ids=input_ids, attention_mask=attention_mask, pixel_values=pixel_values,
                           image_grid_thw=image_grid_thw, use_cache=True)
        cache, deltas = out.past_key_values, out.rope_deltas
        nxt = out.logits[:, -1].argmax(-1)
        seq = [input_ids.cpu(), nxt.cpu().unsqueeze(1)]
        done = torch.zeros(B, dtype=torch.bool)
        if eos_token_id is None:
            # no early stop: the whole continuation stays on the device (graph replays, device argmax, ONE final D2H)
            stepper = GraphedDecodeStep(self, cache, deltas)
            toks = [nxt]
            for _ in range(max_new_tokens - 1):
                toks.append(stepper.step(toks[-1]).argmax(-1))
            return torch.cat([input_ids.cpu(), torch.stack(toks, 1).cpu()], 1)
        for _ in range(max_new_tokens - 1):
            done |= seq[-1].squeeze(1) == eos_token_id
            if bool(done.all()):
                break
            out = self.forward(input_ids=seq[-1], past_key_values=cache, rope_deltas=deltas, use_cache=True)
            seq.append(out.logits[:, -1].argmax(-1).cpu().unsqueeze(1))
        return torch.cat(seq, 1)

    __call__ = forward
