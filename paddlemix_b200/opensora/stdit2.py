"""STDiT2 — host-side mirror of ppdiffusers/examples/Open-Sora/models/stdit/stdit2.py (STDiT2.forward :334-448,
STDiT2Block.forward :119-191) on sm_90a kernels; inference path (x_mask = None).

Device graph per block (tokens are [B, T*S, D] with row = (b*T + t)*S + s, never transposed):
  LN+modulate (one kernel) -> spatial qkv GEMM -> [q/k RMSNorm per head] -> flash attention over S per (b, t)
  -> proj GEMM with fused gate*(.)+residual;  LN+modulate -> temporal qkv GEMM -> `small_attention` kernel along the
  frame axis (strided reads, RoPE + q/k norm fused; a 16x16 problem per head does not fill a tensor-core tile) -> proj
  GEMM with gate+residual;  q GEMM -> cross attention against the per-sample text keys/values (kv_lens = the
  reference's block-diagonal mask) -> proj GEMM + residual;  LN+modulate -> fc1 GEMM + tanh-GELU -> fc2 GEMM with
  gate+residual.  Spatial / cross heads (72 wide) are zero-padded to 128 at load; the temporal path uses 72 directly.
  The 28 x (6+3) modulation vectors come from two GEMMs and one table-broadcast kernel per forward; all 28 cross-attn
  k|v projections of the text are one GEMM per forward.
"""
import math
from typing import Any, Dict, Union

import torch

from ..ppdiffusers.unet_2d_condition import FrozenDict, _to_t

bf16 = torch.bfloat16


class STDiT2Config(FrozenDict):
    """STDiT2Config (stdit2.py:194-238), the fields the forward reads."""

    def __init__(self, input_sq_size=32, in_channels=4, patch_size=(1, 2, 2), hidden_size=1152, depth=28, num_heads=16,
                 mlp_ratio=4.0, pred_sigma=True, caption_channels=4096, model_max_length=120, qk_norm=False, **kw):
        super().__init__(input_sq_size=input_sq_size, in_channels=in_channels, patch_size=tuple(patch_size),
                         hidden_size=hidden_size, depth=depth, num_heads=num_heads, mlp_ratio=mlp_ratio,
                         pred_sigma=pred_sigma, caption_channels=caption_channels, model_max_length=model_max_length,
                         qk_norm=qk_norm)


class STDiT2:
    def __init__(self, config: Union[STDiT2Config, Dict[str, Any]]):
        self.config = config if isinstance(config, STDiT2Config) else STDiT2Config(**config)
        c = self.config
        assert c.hidden_size % 3 == 0, "hidden_size must be divisible by 3"
        if c.patch_size[0] != 1 or c.patch_size[1] != c.patch_size[2]:
            raise NotImplementedError("STDiT2(b200): patch_size must be (1, p, p)")
        self.head_dim = c.hidden_size // c.num_heads
        self.head_pad = 64 if self.head_dim <= 64 else 128
        if self.head_dim > 128 or self.head_dim % 8:
            raise NotImplementedError("STDiT2(b200): head_dim must be a multiple of 8 and <= 128")
        self.out_channels = c.in_channels * 2 if c.pred_sigma else c.in_channels
        self.dtype = bf16
        self.device = None

    def state_dict_shapes(self) -> Dict[str, tuple]:
        c = self.config
        D, hd = c.hidden_size, self.head_dim
        pt, ph, pw = c.patch_size
        hidden = int(D * c.mlp_ratio)
        S: Dict[str, tuple] = {}

        def lin(name, i, o):
            S[name + ".weight"], S[name + ".bias"] = (i, o), (o,)

        S["x_embedder.proj.weight"], S["x_embedder.proj.bias"] = (D, c.in_channels, pt, ph, pw), (D,)
        lin("t_embedder.mlp.0", 256, D), lin("t_embedder.mlp.2", D, D)
        lin("t_block.1", D, 6 * D), lin("t_block_temp.1", D, 3 * D)
        lin("y_embedder.y_proj.fc1", c.caption_channels, D), lin("y_embedder.y_proj.fc2", D, D)
        for name, d in (("csize_embedder", D // 3), ("ar_embedder", D // 3), ("fl_embedder", D), ("fps_embedder", D)):
            lin(name + ".mlp.0", 256, d), lin(name + ".mlp.2", d, d)
        for i in range(c.depth):
            b = f"blocks.{i}"
            S[b + ".scale_shift_table"], S[b + ".scale_shift_table_temporal"] = (6, D), (3, D)
            for a in ("attn", "attn_temp"):
                lin(f"{b}.{a}.qkv", D, 3 * D), lin(f"{b}.{a}.proj", D, D)
                if c.qk_norm:
                    S[f"{b}.{a}.q_norm.weight"], S[f"{b}.{a}.k_norm.weight"] = (hd,), (hd,)
            lin(b + ".cross_attn.q_linear", D, D), lin(b + ".cross_attn.kv_linear", D, 2 * D), lin(b + ".cross_attn.proj", D, D)
            lin(b + ".mlp.fc1", D, hidden), lin(b + ".mlp.fc2", hidden, D)
        S["final_layer.scale_shift_table"] = (2, D)
        lin("final_layer.linear", D, pt * ph * pw * self.out_channels)
        return S

    def init_synthetic_weights(self, seed: int = 1, device: Union[int, str] = 0):
        dev = torch.device("cuda", device) if isinstance(device, int) else torch.device(device)
        g = torch.Generator(device=dev).manual_seed(seed)
        P = {}
        D = self.config.hidden_size
        for name, shp in sorted(self.state_dict_shapes().items()):
            if "scale_shift_table" in name:
                t = torch.randn(shp, generator=g, device=dev) / D ** 0.5
            elif name.endswith(".weight") and len(shp) >= 2:
                fan_in = shp[0] if len(shp) == 2 else math.prod(shp[1:])
                t = (torch.rand(shp, generator=g, device=dev) * 2 - 1) / fan_in ** 0.5
            elif name.endswith(".weight"):
                t = 1.0 + 0.1 * torch.randn(shp, generator=g, device=dev)
            else:
                t = 0.05 * torch.randn(shp, generator=g, device=dev)
            P[name] = t.to(bf16)
        return self.load_state_dict(P, device=device)

    # ------------------------------------------------------------------------------------------------------------
    def _pad_heads_rows(self, w):  # [H*d, in] -> [H*dp, in]
        H, d, dp = self.config.num_heads, self.head_dim, self.head_pad
        if d == dp:
            return w
        out = torch.zeros(H, dp, w.shape[-1], device=w.device)
        out[:, :d] = w.reshape(H, d, -1)
        return out.reshape(H * dp, -1)

    def _pad_heads_vec(self, b):
        H, d, dp = self.config.num_heads, self.head_dim, self.head_pad
        if d == dp:
            return b
        out = torch.zeros(H, dp, device=b.device)
        out[:, :d] = b.reshape(H, d)
        return out.reshape(-1)

    def _pad_heads_cols(self, w):  # [out, H*d] -> [out, H*dp]
        H, d, dp = self.config.num_heads, self.head_dim, self.head_pad
        if d == dp:
            return w
        out = torch.zeros(w.shape[0], H, dp, device=w.device)
        out[:, :, :d] = w.reshape(w.shape[0], H, d)
        return out.reshape(w.shape[0], H * dp)

    def load_state_dict(self, P: Dict[str, Any], device: Union[int, str] = 0):
        from .. import ops
        dev = torch.device("cuda", device) if isinstance(device, int) else torch.device(device)
        ops.init(dev.index or 0)
        self.device = dev
        missing = [k for k in self.state_dict_shapes() if k not in P]
        if missing:
            raise KeyError(f"state dict is missing {len(missing)} parameters, e.g. {missing[:3]}")
        c, D = self.config, self.config.hidden_size

        def W(name):
            return _to_t(P[name + ".weight"]).t().contiguous()

        def Bv(name):
            return _to_t(P[name + ".bias"])

        def lin(name):
            return (W(name).to(dev, bf16).contiguous(), Bv(name).to(dev).contiguous())

        self.w_patch = (_to_t(P["x_embedder.proj.weight"]).reshape(D, -1).contiguous().to(dev, bf16), Bv("x_embedder.proj").to(dev))
        self.t_emb = (lin("t_embedder.mlp.0"), lin("t_embedder.mlp.2"))
        self.size_emb = {n: (lin(n + ".mlp.0"), lin(n + ".mlp.2")) for n in ("csize_embedder", "ar_embedder", "fl_embedder", "fps_embedder")}
        self.t_block, self.t_block_temp = lin("t_block.1"), lin("t_block_temp.1")
        self.y_fc1, self.y_fc2 = lin("y_embedder.y_proj.fc1"), lin("y_embedder.y_proj.fc2")
        self.tab_spc = torch.cat([_to_t(P[f"blocks.{i}.scale_shift_table"]).reshape(1, 6 * D) for i in range(c.depth)], 0).to(dev).contiguous()
        self.tab_tmp = torch.cat([_to_t(P[f"blocks.{i}.scale_shift_table_temporal"]).reshape(1, 3 * D) for i in range(c.depth)], 0).to(dev).contiguous()
        self.tab_final = _to_t(P["final_layer.scale_shift_table"]).reshape(1, 2 * D).to(dev).contiguous()
        self.final = lin("final_layer.linear")
        self.blocks = []
        kv_w, kv_b = [], []
        for i in range(c.depth):
            b = f"blocks.{i}"
            blk = {}
            wqkv, bqkv = W(b + ".attn.qkv"), Bv(b + ".attn.qkv")  # rows (3, H, d)
            blk["s_qkv"] = (torch.cat([self._pad_heads_rows(wqkv[j * D:(j + 1) * D]) for j in range(3)], 0).to(dev, bf16).contiguous(),
                            torch.cat([self._pad_heads_vec(bqkv[j * D:(j + 1) * D]) for j in range(3)], 0).to(dev).contiguous())
            blk["s_proj"] = (self._pad_heads_cols(W(b + ".attn.proj")).to(dev, bf16).contiguous(), Bv(b + ".attn.proj").to(dev))
            blk["t_qkv"], blk["t_proj"] = lin(b + ".attn_temp.qkv"), lin(b + ".attn_temp.proj")
            if c.qk_norm:
                for a, key in (("attn", "s"), ("attn_temp", "t")):
                    blk[key + "_qn"] = _to_t(P[f"{b}.{a}.q_norm.weight"]).to(dev).contiguous()
                    blk[key + "_kn"] = _to_t(P[f"{b}.{a}.k_norm.weight"]).to(dev).contiguous()
            blk["c_q"] = (self._pad_heads_rows(W(b + ".cross_attn.q_linear")).to(dev, bf16).contiguous(),
                          self._pad_heads_vec(Bv(b + ".cross_attn.q_linear")).to(dev).contiguous())
            wkv, bkv = W(b + ".cross_attn.kv_linear"), Bv(b + ".cross_attn.kv_linear")  # rows (2, H, d)
            kv_w.append(torch.cat([self._pad_heads_rows(wkv[:D]), self._pad_heads_rows(wkv[D:])], 0))
            kv_b.append(torch.cat([self._pad_heads_vec(bkv[:D]), self._pad_heads_vec(bkv[D:])], 0))
            blk["c_proj"] = (self._pad_heads_cols(W(b + ".cross_attn.proj")).to(dev, bf16).contiguous(), Bv(b + ".cross_attn.proj").to(dev))
            blk["fc1"], blk["fc2"] = lin(b + ".mlp.fc1"), lin(b + ".mlp.fc2")
            self.blocks.append(blk)
        self.kv_w = torch.cat(kv_w, 0).to(dev, bf16).contiguous()  # all blocks' cross-attn k|v projections: one GEMM
        self.kv_b = torch.cat(kv_b, 0).to(dev).contiguous()
        self._pos_cache = {}
        return self

    # ------------------------------------------------------------------------------------------------------------
    def _embed_scalar(self, pair, s, residual=None):
        """TimestepEmbedder / SizeEmbedder MLP on a flat fp32 vector s (dit_llama.py:68-89); `residual` [rows, D] is
        added in the second GEMM's epilogue (the reference's `t + data_info`, `fl + fps` adds, stdit2.py:357,370-371)."""
        from .. import ops
        from .._lib import ACT_SILU
        f = ops.timestep_embedding(s.contiguous(), 256, flip_sin_to_cos=True, downscale_freq_shift=0.0)  # [cos | sin]
        return ops.linear(ops.linear(f, *pair[0], act=ACT_SILU), *pair[1], residual=residual)

    def _pos_embed(self, H, W, scale, base_size):
        """PositionEmbedding2D (blocks.py:487-545) -> bf16 [S, D], host-computed once per latent size."""
        key = (H, W, float(scale), base_size)
        t = self._pos_cache.get(key)
        if t is None:
            D = self.config.hidden_size
            half = D // 2
            inv_freq = 1.0 / 10000 ** (torch.arange(0, half, 2, dtype=torch.float32) / half)
            gh = torch.arange(H, dtype=torch.float32) / scale * (base_size / H)
            gw = torch.arange(W, dtype=torch.float32) / scale * (base_size / W)
            a, bm = torch.meshgrid(gw, gh, indexing="ij")
            a, bm = a.t().reshape(-1), bm.t().reshape(-1)

            def sincos(v):
                o = torch.einsum("i,d->id", v, inv_freq)
                return torch.cat([torch.sin(o), torch.cos(o)], -1)
            t = torch.cat([sincos(a), sincos(bm)], -1).to(bf16).contiguous().to(self.device)
            self._pos_cache[key] = t
        return t

    def forward(self, x, timestep, y, mask=None, x_mask=None, num_frames=None, height=None, width=None, ar=None, fps=None):
        """Same signature as the reference (stdit2.py:334-336). x [B,C,T,H,W]; y [B,1,L,caption]; returns fp32."""
        from .. import ops
        from .._lib import ACT_GELU_TANH, ACT_SILU
        if self.device is None:
            raise RuntimeError("load_state_dict() must be called before forward()")
        if x_mask is not None:
            raise NotImplementedError("x_mask (frame masking) is outside the hot path")
        c, dev, D = self.config, self.device, self.config.hidden_size
        Hh, hd, dp = c.num_heads, self.head_dim, self.head_pad
        ps = c.patch_size[1]
        x = x.to(dev)
        if x.dtype not in (torch.float32, bf16):
            x = x.float()
        B, _, Tx, Hx, Wx = x.shape
        if Hx % ps or Wx % ps:
            raise NotImplementedError("STDiT2(b200): H and W must be multiples of the patch size")
        T, H, W = Tx, Hx // ps, Wx // ps
        S = H * W
        N = T * S
        f32 = lambda v: v.to(device=dev, dtype=torch.float32)
        height, width, ar, fps, num_frames = f32(height), f32(width), f32(ar), f32(fps), f32(num_frames)
        rs = (float(height[0]) * float(width[0])) ** 0.5
        # size / aspect / length / fps embeddings (:349-358)
        hw = torch.stack([height, width], 1).reshape(-1)
        d3 = D // 3
        csize = self._embed_scalar(self.size_emb["csize_embedder"], hw).reshape(B, 2 * d3)
        ar_e = self._embed_scalar(self.size_emb["ar_embedder"], ar)
        fl = self._embed_scalar(self.size_emb["fl_embedder"], num_frames)
        fl = self._embed_scalar(self.size_emb["fps_embedder"], fps, residual=fl)  # fl + fps_embedder(fps) (:357)
        ts = f32(timestep).reshape(-1).expand(B).contiguous()
        t = self._embed_scalar(self.t_emb, ts)
        data_info = torch.cat([csize, ar_e], 1).contiguous()
        t_spc_in = self._embed_scalar(self.t_emb, ts, residual=data_info)  # t + data_info (:370), add fused in the GEMM
        t_tmp_in = self._embed_scalar(self.t_emb, ts, residual=fl)         # t + fl (:371)
        t_spc = ops.linear(ops.activation(t_spc_in, ACT_SILU), *self.t_block, out_fp32=True)       # [B, 6D]
        t_tmp = ops.linear(ops.activation(t_tmp_in, ACT_SILU), *self.t_block_temp, out_fp32=True)  # [B, 3D]
        mod_s = ops.broadcast_add(t_spc, self.tab_spc)      # [B, depth, 6D]
        mod_t = ops.broadcast_add(t_tmp, self.tab_tmp)      # [B, depth, 3D]
        mod_f = ops.broadcast_add(ops.cast(t, torch.float32).repeat(1, 2), self.tab_final)[:, 0]  # [B, 2D]: table + t[:, None]
        # patch embedding + 2-D position embedding (:361-368)
        pos = self._pos_embed(H, W, rs / c.input_sq_size, round(S ** 0.5))
        h = ops.linear(ops.patchify3d(x.contiguous(), ps), *self.w_patch, residual=pos, residual_row_mod=S)  # [B, N, D]
        # caption embedding (:385-394) and all blocks' cross-attention K/V in one GEMM
        L = y.shape[2]
        ye = ops.linear(ops.linear(y.to(device=dev, dtype=bf16).reshape(B, L, -1).contiguous(), *self.y_fc1, act=ACT_GELU_TANH), *self.y_fc2)
        kv_all = ops.linear(ye, self.kv_w, self.kv_b)  # [B, L, depth*2*H*dp]
        kv_lens = None
        if mask is not None:
            m = mask.to(dev)
            if m.shape[0] != B:
                m = m.repeat(B // m.shape[0], 1)
            kv_lens = m.reshape(B, -1).sum(1).to(torch.int32).contiguous()
            if not bool((m.reshape(B, -1).cumsum(1) == torch.arange(1, L + 1, device=dev)[None]).logical_or(m.reshape(B, -1) == 0).all()):
                raise NotImplementedError("text masks must be prefix masks (valid tokens first)")
        freqs = 1.0 / 10000.0 ** (torch.arange(0, hd, 2)[: hd // 2].float() / hd)
        ang = torch.outer(torch.arange(T, dtype=torch.float32), freqs)
        rcos, rsin = ang.cos().contiguous().to(dev), ang.sin().contiguous().to(dev)
        inner = Hh * dp
        ldm_s, ldm_t = mod_s.stride(0), mod_t.stride(0)
        for i, blk in enumerate(self.blocks):
            ms, mt = mod_s[:, i], mod_t[:, i]  # [B, 6D] / [B, 3D] views with batch stride depth*6D
            # spatial branch: shift_msa, scale_msa, gate_msa = chunks 0, 1, 2
            xm = ops.layernorm(h, eps=1e-6, scale=ms[:, D:], shift=ms[:, 0:], rows_per_group=N)
            qkv = ops.linear(xm, *blk["s_qkv"])  # [B, N, 3*H*dp]
            q = qkv[:, :, :inner].reshape(B * T, S, Hh, dp) if False else qkv.view(B * T, S, 3 * inner)[:, :, :inner].unflatten(-1, (Hh, dp))
            k = qkv.view(B * T, S, 3 * inner)[:, :, inner:2 * inner].unflatten(-1, (Hh, dp))
            v = qkv.view(B * T, S, 3 * inner)[:, :, 2 * inner:].unflatten(-1, (Hh, dp))
            if c.qk_norm:
                rows = qkv.view(B * N, 3 * inner)
                ops.head_rmsnorm_inplace(rows[:, :inner].unflatten(-1, (Hh, dp)), blk["s_qn"], hd)
                ops.head_rmsnorm_inplace(rows[:, inner:2 * inner].unflatten(-1, (Hh, dp)), blk["s_kn"], hd)
            a = ops.sdpa(q, k, v, scale=hd ** -0.5)  # [B*T, S, H, dp]
            h = ops.linear(a.reshape(B, N, inner), *blk["s_proj"], row_gate=ms[:, 2 * D:], rows_per_group=N, residual=h)
            # temporal branch (shift_tmp, scale_tmp, gate_tmp)
            xm = ops.layernorm(h, eps=1e-6, scale=mt[:, D:], shift=mt[:, 0:], rows_per_group=N)
            tqkv = ops.linear(xm, *blk["t_qkv"]).reshape(B * N, 3 * D)
            ta = ops.small_attention(tqkv, B, T, S, Hh, hd, scale=hd ** -0.5, rope_cos=rcos, rope_sin=rsin,
                                     q_norm_w=blk.get("t_qn"), k_norm_w=blk.get("t_kn"))
            h = ops.linear(ta.reshape(B, N, D), *blk["t_proj"], row_gate=mt[:, 2 * D:], rows_per_group=N, residual=h)
            # cross attention (no modulation, no gate) :173-174
            cq = ops.linear(h, *blk["c_q"]).unflatten(-1, (Hh, dp))  # [B, N, H, dp]
            off = i * 2 * inner
            ck = kv_all[:, :, off:off + inner].unflatten(-1, (Hh, dp))
            cv = kv_all[:, :, off + inner:off + 2 * inner].unflatten(-1, (Hh, dp))
            ca = ops.sdpa(cq, ck, cv, scale=hd ** -0.5, kv_lens=kv_lens)
            h = ops.linear(ca.reshape(B, N, inner), *blk["c_proj"], residual=h)
            # MLP (shift_mlp, scale_mlp, gate_mlp = chunks 3, 4, 5)
            xm = ops.layernorm(h, eps=1e-6, scale=ms[:, 4 * D:], shift=ms[:, 3 * D:], rows_per_group=N)
            f = ops.linear(xm, *blk["fc1"], act=ACT_GELU_TANH)
            h = ops.linear(f, *blk["fc2"], row_gate=ms[:, 5 * D:], rows_per_group=N, residual=h)
        # T2IFinalLayer (blocks.py:376-392): shift, scale = (table + t).chunk(2)
        hn = ops.layernorm(h, eps=1e-6, scale=mod_f[:, D:], shift=mod_f[:, 0:], rows_per_group=N)
        out = ops.linear(hn, *self.final)  # [B, N, p*p*C_out]
        return ops.unpatchify3d(out, self.out_channels, T, H, W, ps)

    __call__ = forward

