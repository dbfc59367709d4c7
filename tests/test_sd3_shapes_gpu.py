"""SD3-medium (hidden 1536, 24 heads x 64, 24 layers, joint text 4096, pooled 2048) against fp32 / fp64.

Part 1 checks every kernel the MMDiT calls at its production call site: the AdaLN vectors are views into one fp32
modulation table [B, 286 D] at the model's own offsets (row stride 439 296 floats), every sample carries different
vectors, latents are non-square, and the image token count n = h w is not always a multiple of the 128-row tile, so
group boundaries fall inside tiles. Every reference is plain torch in fp32 or fp64 on the GPU (TF32 off) on the same
bf16 inputs, and it rounds to bf16 where the model rounds. The joint [B, n + L, 3D] qkv buffer is filled with a sentinel
so that a GEMM that stores into the other token range is seen even when the other GEMM would overwrite it. One `slow`
test runs the GEMMs and the attention at shapes whose tensors pass 2^31 elements.

Part 2 runs the model (depth cut to 3: two regular blocks and the context-pre-only last block) against oracle/sd3.py on
the GPU in fp32. The embeddings and the modulation table are compared element by element. Each block is compared with
oracle.joint_block evaluated on the same bf16 input, so the bounds measure one block and not the accumulated drift.
Every LayerNorm the model launches is also captured and checked against the oracle's chunk order of the modulation
vectors, which the block comparison alone cannot see at the last block's context norm.

Block bounds. The residual stream is stored in bf16: one storage rounding is 2^-9 relative, and a value re-rounded after
an update can be off by 2^-8 of itself. Each block output must satisfy |out - ref| <= 2^-8 |ref| + ATOL_RMS * rms(ref),
where ATOL_RMS covers the bf16 rounding of the branch outputs (normalised activations, q/k/v, attention and MLP
intermediates), and the normwise error ||out - ref|| / ||ref|| must stay below L2_MAX.
Measured on an H100 80GB HBM3 (700 W power limit) over the three cases of test_sd3_medium_vs_oracle (largest excess
in units of rms(ref) / largest normwise error), with the bounds and their headroom:
  - image stream, per block: 0.0085 / 2.24e-3; bound 0.02 / 4e-3 (2.4x / 1.8x);
  - context stream, per block: 0.0120 / 2.29e-3; same bound (1.7x / 1.7x);
  - final layer on the same bf16 input: 0.0076 / 2.33e-3; same bound (2.6x / 1.7x);
  - whole forward: 0.0220 / 5.05e-3; bound 0.04 / 9e-3 (1.8x / 1.8x);
  - the 2-step CFG pipeline (guidance 5 scales the difference of two model outputs): 0.0621 / 1.49e-2; bound
    0.1 / 2.5e-2 (1.6x / 1.7x);
  - embeddings: patch + position 2.5e-7 / 1.65e-3, context 6.7e-6 / 1.67e-3, temb 0.0065 / 2.60e-3, modulation table
    0.0059 / 1.35e-3; bound 0.01 / 4e-3 (1.5x / 1.5x for temb).
The earlier model test allowed 4 % of the largest output value.
"""
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import sd3 as O

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16

D, HEADS, HD, DEPTH = 1536, 24, 64, 24
MOD_W = 286 * D                  # 23 blocks x 12 D + last block (6 D + 2 D) + norm_out 2 D = 439 296 floats
BNS = [32, 64, 128, 160, 192, 224, 256]
RTOL_RESID = 2.0 ** -8           # bf16 storage of the residual stream
BLOCK_ATOL_RMS, BLOCK_L2 = 0.02, 4e-3
FINAL_ATOL_RMS, FINAL_L2 = 0.04, 9e-3
PIPE_ATOL_RMS, PIPE_L2 = 0.1, 0.025
EMBED_ATOL_RMS, EMBED_L2 = 0.01, 4e-3
JOINT = [(4032, 333), (4096, 154), (240, 77)]   # (image tokens n, text tokens L): 144x112, 128x128, 40x24 latents


@pytest.fixture(scope="module")
def ops():
    from paddlemix_b200 import ops as _ops
    _ops.init(0)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return _ops


def rnd(*shape, seed=0, scale=1.0, dtype=bf16):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).to(dtype)


def close(a, b, atol, rtol, what):
    err = (a.double() - b.double()).abs()
    bad = (err > atol + rtol * b.double().abs()).sum().item()
    assert bad == 0, f"{what}: {bad}/{a.numel()} mismatches, max err {err.max().item():.4g}"


def mod_offsets(depth=DEPTH):
    """Column offsets into the modulation table, in SD3Transformer2DModel's layout: per block (norm1, norm1_context),
    then norm_out."""
    blocks, off = [], 0
    for i in range(depth):
        blocks.append((off, off + 6 * D))
        off += 6 * D + (2 * D if i == depth - 1 else 6 * D)
    return blocks, off


def mod_table(B, seed):
    """The model's fp32 [B, 286 D] modulation table, clearly different per sample."""
    return (rnd(B, MOD_W, seed=seed, dtype=torch.float32) * 0.5).contiguous()


class knobs:
    """Sets the GEMM / LayerNorm debug selectors for one call and restores the defaults."""

    def __init__(self, bn=0, streamk=None, skinny=1, ln_register=0):
        self.bn, self.streamk, self.skinny, self.ln_register = bn, streamk, skinny, ln_register

    def __enter__(self):
        from paddlemix_b200._lib import lib
        lib.b200mix_debug_force_bn(self.bn)
        if self.streamk is not None:
            lib.b200mix_debug_streamk(self.streamk)
        lib.b200mix_debug_skinny(self.skinny)
        lib.b200mix_debug_ln_register_only(self.ln_register)

    def __exit__(self, *a):
        from paddlemix_b200._lib import lib
        lib.b200mix_debug_force_bn(0)
        lib.b200mix_debug_streamk(int(os.environ.get("B200MIX_STREAMK", 1)))
        lib.b200mix_debug_skinny(1)
        lib.b200mix_debug_ln_register_only(0)


# ---------------------------------------------------------------------------------------------------------------------
# Part 1: the kernels at their call sites
# ---------------------------------------------------------------------------------------------------------------------
def test_mod_table_layout():
    assert mod_offsets()[1] + 2 * D == MOD_W == 439296
    assert mod_offsets()[0][-1] == (276 * D, 282 * D)


@pytest.fixture(scope="module")
def mod_gemm(ops):
    """All 49 AdaLN projections of the 24-layer model as one weight: N = 439 296, K = 1536."""
    w = rnd(MOD_W, D, seed=1, scale=D ** -0.5)
    b = rnd(MOD_W, seed=2, scale=0.05, dtype=torch.float32)
    yield w, b
    del w, b
    torch.cuda.empty_cache()


@pytest.mark.parametrize("M", [1, 2, 3, 4, 5, 8, 16, 32])
def test_modulation_gemm_full_width(ops, mod_gemm, M):
    """mod = silu(temb) @ mod_w^T + mod_b in fp32 at every batch size the benchmark and the CFG pipeline give a rank:
    M = 1, 2, 4, 8 run the four skinny kernels, 3 and 5 their padded forms, 16 and 32 the tiled GEMM. The output is
    prefilled with NaN so an unwritten row cannot pass on stale memory. M <= 8 also runs with the skinny path off."""
    from paddlemix_b200._lib import ACT_SILU
    w, b = mod_gemm
    temb = rnd(M, D, seed=100 + M)
    a = ops.activation(temb, ACT_SILU)
    torch.testing.assert_close(a.float(), F.silu(temb.float()).to(bf16).float(), rtol=2.0 ** -7, atol=0)
    ad = a.double()
    ref = torch.cat([ad @ w[j:j + 65536].double().t() for j in range(0, MOD_W, 65536)], 1) + b.double()
    for skinny in ([1, 0] if M <= 8 else [1]):
        out = torch.full((M, MOD_W), float("nan"), device="cuda", dtype=torch.float32)
        with knobs(skinny=skinny):
            got = ops.linear(a, w, b, out_fp32=True, out=out)
        assert got.data_ptr() == out.data_ptr()
        assert bool(torch.isfinite(out).all()), f"M={M} skinny={skinny}: rows left unwritten"
        close(out, ref, 1e-4, 1e-4, f"modulation GEMM M={M} skinny={skinny}")


def adaln_sites(depth=DEPTH):
    """(name, rows, scale column, shift column, LayerNorm bias?) for every AdaLN LayerNorm of SD3Transformer2DModel,
    with columns relative to the table row; a middle block stands in for all regular blocks."""
    blocks, out_off = mod_offsets(depth)
    (x1, c1), (xl, cl) = blocks[7], blocks[-1]
    return [("norm1", "n", x1 + D, x1, False), ("norm1_context", "L", c1 + D, c1, False),
            ("norm2", "n", x1 + 4 * D, x1 + 3 * D, False), ("norm2_context", "L", c1 + 4 * D, c1 + 3 * D, False),
            ("last norm1", "n", xl + D, xl, False), ("last norm1_context", "L", cl, cl + D, True),
            ("norm_out", "n", out_off, out_off + D, True)]


@pytest.mark.parametrize("path", ["block", "register"])
@pytest.mark.parametrize("n,L", JOINT)
def test_adaln_layernorm_sites(ops, n, L, path):
    """LN + (1 + scale), shift at every AdaLN site, scale / shift read through views of the [B, 286 D] table: the
    AdaLayerNormZero sites (shift, scale order, no LayerNorm bias) and the two AdaLayerNormContinuous sites (scale, shift
    order, LayerNorm bias and no weight). B = 3, rows_per_group = n or L."""
    B = 3
    tab = mod_table(B, seed=200 + n)
    ln_bias = rnd(D, seed=201, scale=0.3, dtype=torch.float32)
    xs = {"n": (rnd(B, n, D, seed=202) * 2 + 0.5).to(bf16), "L": (rnd(B, L, D, seed=203) * 3 - 0.25).to(bf16)}
    for name, rows, sc, sh, has_bias in adaln_sites():
        x = xs[rows]
        with knobs(ln_register=1 if path == "register" else 0):
            out = ops.layernorm(x, None, ln_bias if has_bias else None, eps=1e-6, scale=tab[:, sc:], shift=tab[:, sh:],
                                rows_per_group=x.shape[1])
        ref = F.layer_norm(x.double(), (D,), eps=1e-6)
        if has_bias:
            ref = ref + ln_bias.double()
        ref = ref * (1 + tab[:, sc:sc + D].double()[:, None]) + tab[:, sh:sh + D].double()[:, None]
        close(out, ref, 4e-3, 2.0 ** -7, f"{name} rows={x.shape[1]} {path}")


def joint_qkv_case(n, L, B=3):
    nx, nc = rnd(B, n, D, seed=300 + n), rnd(B, L, D, seed=301 + L)
    w, wc = rnd(3 * D, D, seed=302, scale=D ** -0.5), rnd(3 * D, D, seed=303, scale=D ** -0.5)
    b, bc = rnd(3 * D, seed=304, scale=0.1, dtype=torch.float32), rnd(3 * D, seed=305, scale=0.1, dtype=torch.float32)
    return (nx, w, b), (nc, wc, bc)


SENTINEL = 1000.0


@pytest.mark.parametrize("streamk", [0, 1], ids=["roundrobin", "streamk"])
@pytest.mark.parametrize("bn", BNS)
@pytest.mark.parametrize("n,L", JOINT)
def test_joint_qkv_writes_stay_in_range(ops, n, L, bn, streamk):
    """q|k|v of each stream written by linear_batched into its token range of one sentinel-filled [B, n + L, 3D] buffer:
    the image GEMM alone leaves every text row untouched, the text GEMM alone every image row, and both orders give the
    same buffer."""
    B = 3
    (nx, w, b), (nc, wc, bc) = joint_qkv_case(n, L, B)
    ref_x = nx.float() @ w.float().t() + b
    ref_c = nc.float() @ wc.float().t() + bc
    results = []
    for order in (("x",), ("c",), ("x", "c"), ("c", "x")):
        qkv = torch.full((B, n + L, 3 * D), SENTINEL, device="cuda", dtype=bf16)
        with knobs(bn=bn, streamk=streamk):
            for s in order:
                if s == "x":
                    ops.linear_batched(nx, w, b, out=qkv[:, :n])
                else:
                    ops.linear_batched(nc, wc, bc, out=qkv[:, n:])
        what = f"n={n} L={L} bn={bn} streamk={streamk} order={'+'.join(order)}"
        for s, rng, ref in (("x", slice(0, n), ref_x), ("c", slice(n, n + L), ref_c)):
            if s in order:
                close(qkv[:, rng], ref, 1e-2, 2.0 ** -7, what + f" {s} rows")
            else:
                assert bool((qkv[:, rng] == SENTINEL).all()), what + f": {s} rows written by the other GEMM"
        results.append(qkv)
    assert torch.equal(results[2], results[3])


def attention_ref(q, k, v, b, h):
    qq, kk, vv = (t[b, :, h].float() for t in (q, k, v))
    return torch.softmax(qq @ kk.t() * q.shape[-1] ** -0.5, -1) @ vv


@pytest.mark.parametrize("heads,hd", [(HEADS, HD), (12, 128)], ids=["24x64", "12x128"])
@pytest.mark.parametrize("S", [4250, 4365, 317])
def test_joint_attention_strided_views(ops, S, heads, hd):
    """sdpa on the q / k / v column slices of the joint [B, S, 3D] buffer, exactly as the blocks call it, B = 3 with
    different content per sample; the fp32 reference runs per (sample, head) for the first, middle and last sample."""
    B = 3
    qkv = rnd(B, S, 3 * D, seed=400 + S + hd)
    qkv[1] = qkv[1] * 1.5 + 0.25
    q, k, v = (qkv[:, :, i * D:(i + 1) * D].unflatten(-1, (heads, hd)) for i in range(3))
    out = ops.sdpa(q, k, v, scale=hd ** -0.5)
    assert out.shape == (B, S, heads, hd)
    for b in range(B):
        for h in (0, heads // 2, heads - 1):
            close(out[b, :, h], attention_ref(q, k, v, b, h), 1e-2, 2.0 ** -7, f"S={S} {heads}x{hd} sample {b} head {h}")


@pytest.mark.parametrize("n,L", JOINT)
def test_output_projections_gate_residual(ops, n, L):
    """to_out / to_add_out: linear_batched on the o[:, :n] and o[:, n:] token ranges of the attention output, with the
    per-sample gate a view of the modulation table (gate_msa / c_gate_msa of a middle block) and the stream as residual."""
    B = 3
    o = rnd(B, n + L, D, seed=500 + n)
    tab = mod_table(B, seed=501)
    x1, c1 = mod_offsets()[0][7]
    for rng, off, seed in ((slice(0, n), x1, 502), (slice(n, n + L), c1, 503)):
        a = o[:, rng]
        w = rnd(D, D, seed=seed, scale=D ** -0.5)
        bias = rnd(D, seed=seed + 10, scale=0.1, dtype=torch.float32)
        res = rnd(B, a.shape[1], D, seed=seed + 20)
        gate = tab[:, off + 2 * D:]
        out = torch.empty_like(res)
        ops.linear_batched(a, w, bias, out=out, row_gate=gate, residual=res)
        ref = (a.float() @ w.float().t() + bias) * gate[:, None, :D] + res.float()
        close(out, ref, 1e-2, 2.0 ** -7, f"out projection rows {rng}")


@pytest.mark.parametrize("streamk", [0, 1], ids=["roundrobin", "streamk"])
@pytest.mark.parametrize("bn", BNS)
@pytest.mark.parametrize("n", [4032, 240])
def test_ff2_gate_residual_groups_inside_tiles(ops, n, bn, streamk):
    """ff.net.2: x + gate_mlp * (ff @ W^T + b) with rows_per_group = n (4032 and 240: the sample boundaries fall inside
    128-row tiles) and K = 6144, the gate a view of the modulation table."""
    B = 3
    ff = rnd(B, n, 4 * D, seed=600 + n)
    w = rnd(D, 4 * D, seed=601, scale=(4 * D) ** -0.5)
    bias = rnd(D, seed=602, scale=0.1, dtype=torch.float32)
    res = rnd(B, n, D, seed=603)
    tab = mod_table(B, seed=604)
    gate = tab[:, mod_offsets()[0][7][0] + 5 * D:]
    ref = (ff.float() @ w.float().t() + bias) * gate[:, None, :D] + res.float()
    with knobs(bn=bn, streamk=streamk):
        out = ops.linear(ff, w, bias, row_gate=gate, rows_per_group=n, residual=res)
    close(out, ref, 1e-2, 2.0 ** -7, f"ff2 n={n} bn={bn} streamk={streamk}")


LATENTS = [(144, 112), (96, 168), (40, 24)]   # latent H x W (image 1152x896, 768x1344, 320x192)


@pytest.mark.parametrize("dtype", [torch.float32, bf16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("H,W", LATENTS)
def test_patch_embed_nonsquare(ops, sd3_small, H, W, dtype):
    """PatchEmbed on a non-square latent: patchify against the reshape / permute of a stride-2 conv (exact), the patch
    GEMM with the model's cropped position table through residual_row_mod = n against F.conv2d + the oracle's crop."""
    cfg, model, Pd = sd3_small
    B, C, p = 3, 16, 2
    h, w = H // p, W // p
    x = rnd(B, C, H, W, seed=700 + H, dtype=torch.float32).to(dtype)
    rows = ops.patchify(x.contiguous(), p)
    ref_rows = x.to(bf16).reshape(B, C, h, p, w, p).permute(0, 2, 4, 1, 3, 5).reshape(B, h * w, C * p * p)
    assert torch.equal(rows, ref_rows)
    pos = model._pos(h, w)
    emb = ops.linear(rows, model.w_patch, model.b_patch, residual=pos, residual_row_mod=h * w)
    conv = F.conv2d(x.to(bf16).double(), Pd["pos_embed.proj.weight"].double(), Pd["pos_embed.proj.bias"].double(),
                    stride=p).flatten(2).transpose(1, 2)
    ref = conv + O.sd3_pos_embed(cfg, Pd, h, w).to(bf16).double()
    close(emb, ref, 1e-2, 2.0 ** -7, f"patch embedding {H}x{W}")


@pytest.mark.parametrize("H,W", LATENTS)
def test_unpatchify_nonsquare(ops, H, W):
    """proj_out rows [B, h w, p p C] back to [B, C, H, W]: bit-exact against the oracle's reshape / permute."""
    B, C, p = 3, 16, 2
    h, w = H // p, W // p
    y = rnd(B, h * w, p * p * C, seed=800 + H)
    ref = y.float().reshape(B, h, w, p, p, C).permute(0, 5, 1, 3, 2, 4).reshape(B, C, H, W)
    assert torch.equal(ops.unpatchify(y, C, h, w, p, out_dtype=bf16), ref.to(bf16))
    assert torch.equal(ops.unpatchify(y, C, h, w, p, out_dtype=torch.float32), ref)


def test_timestep_embedding_flowmatch_per_sample(ops):
    """The sinusoidal timestep embedding for six samples at different fractional timesteps of the shift-3 FlowMatch
    schedule (28 steps), against fp64."""
    from paddlemix_b200.ppdiffusers.schedulers import FlowMatchEulerDiscreteScheduler
    sch = FlowMatchEulerDiscreteScheduler(shift=3.0)
    sch.set_timesteps(28)
    ts = torch.tensor([float(sch.timesteps[i]) for i in (0, 3, 11, 19, 26, 27)], device="cuda")
    assert len(set(ts.tolist())) == 6 and any(t != round(t) for t in ts.tolist())
    out = ops.timestep_embedding(ts, 256, flip_sin_to_cos=True, downscale_freq_shift=0.0)
    half = 128
    freqs = torch.exp(-torch.log(torch.tensor(10000.0, dtype=torch.float64)) * torch.arange(half, dtype=torch.float64)
                      / half).cuda()
    arg = ts.double()[:, None] * freqs[None]
    ref = torch.cat([arg.cos(), arg.sin()], -1)
    close(out, ref, 2e-3, 2.0 ** -8, "timestep embedding")


def sampled_rows(first, total, seed):
    """Rows around `first`, random rows after it and the whole last 128-row tile."""
    g = torch.Generator().manual_seed(seed)
    return torch.cat([torch.arange(first, first + 4), torch.randint(first, total - 128, (64,), generator=g),
                      torch.arange(total - 128, total)]).cuda()


def big_ff1_ff2(ops):
    """ff1 with GELU-tanh writing [88 * 4096, 6144] (2.21e9 elements), then ff2 reading it as A with the per-sample gate
    and the residual."""
    from paddlemix_b200._lib import ACT_GELU_TANH
    B, n = 88, 4096
    M = B * n
    a = rnd(M, D, seed=900)
    w1, b1 = rnd(4 * D, D, seed=901, scale=D ** -0.5), rnd(4 * D, seed=902, scale=0.1, dtype=torch.float32)
    ff = ops.linear(a, w1, b1, act=ACT_GELU_TANH)
    assert ff.numel() > 1 << 31
    rows = sampled_rows((1 << 31) // (4 * D), M, seed=0)
    ref = F.gelu(a[rows].double() @ w1.double().t() + b1.double(), approximate="tanh")
    close(ff[rows], ref, 1e-2, 2.0 ** -7, "ff1 output past 2^31 elements")
    del a
    w2, b2 = rnd(D, 4 * D, seed=903, scale=(4 * D) ** -0.5), rnd(D, seed=904, scale=0.1, dtype=torch.float32)
    res = rnd(M, D, seed=905)
    gate = mod_table(B, seed=906)[:, 5 * D:]
    out = ops.linear(ff, w2, b2, row_gate=gate, rows_per_group=n, residual=res)
    ref = (ff[rows].double() @ w2.double().t() + b2.double()) * gate[rows // n, :D].double() + res[rows].double()
    close(out[rows], ref, 1e-2, 2.0 ** -7, "ff2 reading A past 2^31 elements")


def big_joint_qkv_sdpa(ops):
    """q|k|v of both streams into a joint [112, 4250, 4608] buffer (2.19e9 elements; the last sample starts past 2^31),
    then attention over the whole batch, checked on the last sample."""
    B, n, L = 112, 4096, 154
    S = n + L
    nx, nc = rnd(B, n, D, seed=910), rnd(B, L, D, seed=911)
    w, wc = rnd(3 * D, D, seed=912, scale=D ** -0.5), rnd(3 * D, D, seed=913, scale=D ** -0.5)
    b, bc = (rnd(3 * D, seed=s, scale=0.1, dtype=torch.float32) for s in (914, 915))
    qkv = torch.empty(B, S, 3 * D, device="cuda", dtype=bf16)
    last = B - 1
    assert last * S * 3 * D > 1 << 31
    ops.linear_batched(nx, w, b, out=qkv[:, :n])
    ops.linear_batched(nc, wc, bc, out=qkv[:, n:])
    rows = sampled_rows(0, n, seed=1)
    close(qkv[last, rows], nx[last, rows].double() @ w.double().t() + b.double(), 1e-2, 2.0 ** -7,
          "image qkv of the last sample")
    close(qkv[last, n:], nc[last].double() @ wc.double().t() + bc.double(), 1e-2, 2.0 ** -7, "text qkv of the last sample")
    del nx, nc
    q, k, v = (qkv[:, :, i * D:(i + 1) * D].unflatten(-1, (HEADS, HD)) for i in range(3))
    o = ops.sdpa(q, k, v, scale=HD ** -0.5)
    for h in (0, HEADS - 1):
        close(o[last, :, h], attention_ref(q, k, v, last, h), 1e-2, 2.0 ** -7, f"attention, last sample, head {h}")


@pytest.mark.slow
@pytest.mark.parametrize("op", ["ff1_ff2", "joint_qkv_sdpa"])
def test_beyond_2_31_elements(ops, op):
    """The GEMMs and the attention where a tensor passes 2^31 elements (1024^2 latents at 88 or 112 images per GPU, or
    2048^2 at 22 or 28): only rows past the 2^31 boundary, including the last tile, are checked against fp64. The
    helpers hold every large tensor, so returning from them frees it (peak about 12 GB)."""
    try:
        (big_ff1_ff2 if op == "ff1_ff2" else big_joint_qkv_sdpa)(ops)
    finally:
        torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------------
# Part 2: the model against the oracle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sd3_small(ops):
    """SD3-medium with depth cut to 3: two regular blocks and the context-pre-only last block."""
    from paddlemix_b200.ppdiffusers.transformer_sd3 import SD3Transformer2DModel
    cfg = dict(O.SD3_CONFIGS["sd3_medium"])
    cfg["num_layers"] = 3
    P = O.init_sd3_params(cfg, seed=1)
    model = SD3Transformer2DModel(**cfg).load_state_dict(P, device=0)
    Pd = {k: v.cuda() for k, v in P.items()}
    return cfg, model, Pd


def make_inputs(cfg, B, H, W, L, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 16, H, W, generator=g).to(bf16).float()
    ctx = torch.randn(B, L, cfg["joint_attention_dim"], generator=g).to(bf16).float()
    pooled = torch.randn(B, cfg["pooled_projection_dim"], generator=g).to(bf16).float()
    ts = torch.tensor([981.25, 402.5, 17.75, 655.0][:B])
    return x.cuda(), ctx.cuda(), pooled.cuda(), ts.cuda()


def errors(out, ref):
    """(excess over the bf16 storage bound in units of rms(ref), normwise relative error)."""
    o, r = out.double(), ref.double()
    d = (o - r).abs()
    rms = r.pow(2).mean().sqrt()
    return ((d - RTOL_RESID * r.abs()).clamp_min(0).max() / rms).item(), (d.norm() / r.norm()).item()


def check(out, ref, atol_rms, l2_max, what):
    assert out.shape == ref.shape and bool(torch.isfinite(out.float()).all()), what
    excess, l2 = errors(out, ref)
    print(f"{what}: excess {excess:.4g} rms, l2 {l2:.4g}")
    assert excess <= atol_rms and l2 <= l2_max, (what, excess, l2)


def oracle_mod(cfg, Pd, temb):
    """The modulation table in the model's column order, from the oracle's per-site Linear layers."""
    s = F.silu(temb)
    parts = []
    for i in range(cfg["num_layers"]):
        for key in ("norm1", "norm1_context"):
            parts.append(O.linear(s, Pd, f"transformer_blocks.{i}.{key}.linear"))
    parts.append(O.linear(s, Pd, "norm_out.linear"))
    return torch.cat(parts, 1)


CASES = {  # B, latent H x W, text tokens L
    "nonsquare_144x112_L333_B3": (3, 144, 112, 333),
    "bench_128x128_L154_B2": (2, 128, 128, 154),
    "odd_40x24_L77_B4": (4, 40, 24, 77),
}


@pytest.mark.parametrize("case", list(CASES))
def test_sd3_medium_vs_oracle(sd3_small, case):
    cfg, model, Pd = sd3_small
    B, H, W, L = CASES[case]
    x, ctx, pooled, ts = make_inputs(cfg, B, H, W, L, seed=7)
    blocks, end = mod_offsets(3)
    assert [(b["norm1_off"], b["norm1_context_off"]) for b in model.blocks] == blocks and model.norm_out_off == end
    xe, cst, temb, mod, (h, w) = model._embed(x, ctx, pooled, ts)
    n = h * w
    assert (h, w) == (H // 2, W // 2) and xe.shape == (B, n, D) and cst.shape == (B, L, D) and mod.shape == (B, end + 2 * D)
    with torch.device("cuda"), torch.no_grad():
        rx, rc, rt = O.sd3_embed(cfg, Pd, x, ctx, pooled, ts)
        rmod = oracle_mod(cfg, Pd, temb.float())
    for name, o, r in (("patch + position embedding", xe, rx), ("context", cst, rc), ("temb", temb, rt),
                       ("modulation table", mod, rmod)):
        check(o, r, EMBED_ATOL_RMS, EMBED_L2, f"{case} {name}")
    for i in range(3):
        last = i == 2
        with torch.device("cuda"), torch.no_grad():
            ref_c, ref_x = O.joint_block(xe.float(), cst.float(), temb.float(), Pd, f"transformer_blocks.{i}", HEADS,
                                         last)
        xe, cst_new = model._block(i, xe, cst, mod, n, L)
        check(xe, ref_x, BLOCK_ATOL_RMS, BLOCK_L2, f"{case} block {i} x")
        if last:
            assert cst_new is cst
        else:
            check(cst_new, ref_c, BLOCK_ATOL_RMS, BLOCK_L2, f"{case} block {i} context")
        cst = cst_new
    out = model._final(xe, mod, h, w)
    with torch.device("cuda"), torch.no_grad():
        ref = O.sd3_final(cfg, Pd, xe.float(), temb.float(), h, w)
    check(out, ref, BLOCK_ATOL_RMS, BLOCK_L2, f"{case} final layer")
    out = model(x, ctx, pooled, ts).sample
    with torch.device("cuda"), torch.no_grad():
        ref = O.sd3_forward(cfg, Pd, x, ctx, pooled, ts)
    check(out, ref, FINAL_ATOL_RMS, FINAL_L2, f"{case} output")


def test_sd3_adaln_call_sites_follow_the_oracle_chunk_order(sd3_small, monkeypatch):
    """Every LayerNorm the model launches, captured with its input and output, against LN(x) [+ b] * (1 + scale) +
    shift in fp64 with scale and shift taken from the model's own modulation table in the oracle's chunk order:
    AdaLayerNormZero (shift, scale, gate, ...) in the regular blocks, AdaLayerNormContinuous (scale, shift) for the last
    block's context and for norm_out. In the last block the context stream only feeds k and v, so a swapped order there
    moves the block output by less than the block bound; this test sees it directly."""
    from paddlemix_b200 import ops
    cfg, model, Pd = sd3_small
    x, ctx, pooled, ts = make_inputs(cfg, 3, 40, 24, 333, seed=14)
    xe, cst, _, mod, (h, w) = model._embed(x, ctx, pooled, ts)
    n, L = h * w, ctx.shape[1]
    calls = []
    real = ops.layernorm

    def spy(inp, weight=None, bias=None, **kw):
        out = real(inp, weight, bias, **kw)
        calls.append((inp.clone(), bias, out.clone()))
        return out
    monkeypatch.setattr(ops, "layernorm", spy)
    expected = []
    for i, (o1, oc) in enumerate(mod_offsets(3)[0]):
        e = mod[:, o1:o1 + 6 * D].chunk(6, dim=1)             # shift_msa, scale_msa, gate_msa, shift_mlp, scale_mlp, ...
        if i == 2:
            c_scale, c_shift = mod[:, oc:oc + 2 * D].chunk(2, dim=1)
            expected += [(e[1], e[0], None, "norm1"), (c_scale, c_shift, Pd["transformer_blocks.2.norm1_context.norm.bias"],
                                                        "last norm1_context"), (e[4], e[3], None, "norm2")]
        else:
            ec = mod[:, oc:oc + 6 * D].chunk(6, dim=1)
            expected += [(e[1], e[0], None, "norm1"), (ec[1], ec[0], None, "norm1_context"), (e[4], e[3], None, "norm2"),
                         (ec[4], ec[3], None, "norm2_context")]
        xe, cst = model._block(i, xe, cst, mod, n, L)
    model._final(xe, mod, h, w)
    scale, shift = mod[:, model.norm_out_off:model.norm_out_off + 2 * D].chunk(2, dim=1)
    expected.append((scale, shift, Pd["norm_out.norm.bias"], "norm_out"))
    assert len(calls) == len(expected) == 12
    for k, ((inp, bias, out), (sc, sh, b, name)) in enumerate(zip(calls, expected)):
        ref = F.layer_norm(inp.double(), (D,), eps=1e-6)
        if b is not None:
            assert bias is not None
            ref = ref + b.double()
        ref = ref * (1 + sc.double()[:, None]) + sh.double()[:, None]
        close(out, ref, 4e-3, 2.0 ** -7, f"call {k} ({name})")


def test_sd3_forward_is_embed_blocks_final(sd3_small):
    """forward() is _embed, then _block for every block, then _final: the same launches, bit for bit."""
    from paddlemix_b200 import ops
    cfg, model, _ = sd3_small
    x, ctx, pooled, ts = make_inputs(cfg, 3, 144, 112, 333, seed=8)
    ops.reset_launches()
    out = model(x, ctx, pooled, ts).sample
    n_forward = ops.launches()
    ops.reset_launches()
    xe, cst, _, mod, (h, w) = model._embed(x, ctx, pooled, ts)
    for i in range(len(model.blocks)):
        xe, cst = model._block(i, xe, cst, mod, h * w, ctx.shape[1])
    ref = model._final(xe, mod, h, w)
    assert ops.launches() == n_forward
    assert torch.equal(out, ref)


def test_sd3_sample_independence(sd3_small):
    """Permuting the batch permutes the outputs, and each sample run alone matches its row. Not bit for bit: the
    modulation GEMM takes the skinny M = 1 kernel alone and the M = 3 kernel in the batch, and stream-K splits depend on
    the row position. On an H100 the largest difference was 0.57 % of max |out| (one bf16 step of the largest outputs);
    the bound allows a few (2^-6 of max |out|), far below what a sample mix-up gives."""
    cfg, model, _ = sd3_small
    B = 3
    x, ctx, pooled, ts = make_inputs(cfg, B, 144, 112, 333, seed=9)
    out = model(x, ctx, pooled, ts).sample
    scale = out.abs().max().item()
    perm = [2, 0, 1]
    outp = model(x[perm], ctx[perm], pooled[perm], ts[perm]).sample
    dp = (outp - out[perm]).abs().max().item()
    print(f"permuted batch: max diff {dp / scale:.4g} of max |out|")
    assert dp <= 2.0 ** -6 * scale, dp / scale
    for b in range(B):
        one = model(x[b:b + 1], ctx[b:b + 1], pooled[b:b + 1], ts[b:b + 1]).sample
        d1 = (one[0] - out[b]).abs().max().item()
        print(f"sample {b} alone: max diff {d1 / scale:.4g} of max |out|")
        assert d1 <= 2.0 ** -6 * scale, (b, d1 / scale)
    for b in range(1, B):
        assert (out[b] - out[0]).abs().max().item() > 0.1 * scale, "different samples gave the same output"


def test_sd3_scalar_timestep_equals_vector(sd3_small):
    cfg, model, _ = sd3_small
    x, ctx, pooled, _ = make_inputs(cfg, 2, 40, 24, 77, seed=10)
    a = model(x, ctx, pooled, 500.0).sample
    b = model(x, ctx, pooled, torch.full((2,), 500.0, device="cuda")).sample
    c = model(x, ctx, pooled, torch.tensor(500.0)).sample
    assert torch.equal(a, b) and torch.equal(a, c)


@pytest.mark.slow
def test_sd3_medium_cfg_pipeline_vs_oracle(sd3_small):
    """StableDiffusion3Pipeline with CFG (batch 2 -> 4 model rows: the skinny M = 4 modulation GEMM) on a 48 x 32 latent,
    2 FlowMatchEuler steps, against the oracle's restatement of the loop in fp32."""
    from oracle.schedulers import FlowMatchEulerDiscreteScheduler as OFM
    from paddlemix_b200.ppdiffusers.pipelines import StableDiffusion3Pipeline
    from paddlemix_b200.ppdiffusers.schedulers import FlowMatchEulerDiscreteScheduler
    cfg, model, Pd = sd3_small
    B, steps, gs = 2, 2, 5.0
    lat, ctx, pooled, _ = make_inputs(cfg, B, 48, 32, 154, seed=11)
    g = torch.Generator().manual_seed(12)
    nctx = (torch.randn(B, 154, cfg["joint_attention_dim"], generator=g) * 0.1).to(bf16).float().cuda()
    npooled = (torch.randn(B, cfg["pooled_projection_dim"], generator=g) * 0.1).to(bf16).float().cuda()
    pipe = StableDiffusion3Pipeline(model, FlowMatchEulerDiscreteScheduler(shift=3.0))
    lat0 = lat.clone()
    out = pipe(prompt_embeds=ctx, pooled_prompt_embeds=pooled, negative_prompt_embeds=nctx,
               negative_pooled_prompt_embeds=npooled, latents=lat, num_inference_steps=steps, guidance_scale=gs)
    assert torch.equal(lat, lat0), "the pipeline wrote into the caller's latents"
    sch = OFM(shift=3.0)
    sch.set_timesteps(steps)
    cur = lat.cpu().clone()
    with torch.device("cuda"), torch.no_grad():
        for t in sch.timesteps:
            v = O.sd3_forward(cfg, Pd, torch.cat([cur, cur], 0).cuda(), torch.cat([nctx, ctx], 0),
                              torch.cat([npooled, pooled], 0), t.expand(2 * B).cuda())
            vu, vc = v.cpu().chunk(2)
            cur = sch.step(vu + gs * (vc - vu), t, cur)
    check(out, cur.cuda(), PIPE_ATOL_RMS, PIPE_L2, "CFG pipeline, 2 steps")


def test_sd3_pipeline_leaves_device_latents_alone(sd3_small):
    """Latents passed as an fp32 tensor already on the device are the caller's: the loop must work on a copy, and the
    result must be the same as for the same latents passed from the host."""
    from paddlemix_b200.ppdiffusers.pipelines import StableDiffusion3Pipeline
    from paddlemix_b200.ppdiffusers.schedulers import FlowMatchEulerDiscreteScheduler
    cfg, model, _ = sd3_small
    lat, ctx, pooled, _ = make_inputs(cfg, 2, 16, 24, 77, seed=13)
    lat0 = lat.clone()
    pipe = StableDiffusion3Pipeline(model, FlowMatchEulerDiscreteScheduler(shift=3.0))
    kw = dict(prompt_embeds=ctx, pooled_prompt_embeds=pooled, num_inference_steps=3, guidance_scale=4.0)
    out = pipe(latents=lat, **kw)
    assert torch.equal(lat, lat0), "the pipeline wrote into the caller's latents"
    assert out.data_ptr() != lat.data_ptr()
    assert torch.equal(out, pipe(latents=lat0.cpu(), **kw))


def test_arguments_the_kernels_would_misread_are_refused(ops):
    """A weight with the wrong K, a joint-buffer output or residual of the wrong shape, a per-group vector with fewer
    groups or columns than the output needs, or several groups without rows_per_group: refused before any launch."""
    B, n = 3, 240
    tab = mod_table(B, seed=1000)
    a, w = rnd(B, n, D, seed=1001), rnd(D, D, seed=1002, scale=D ** -0.5)
    res = rnd(B, n, D, seed=1003)
    with pytest.raises(ValueError, match="weight must be"):
        ops.linear(a, rnd(D, D + 64, seed=1004))
    with pytest.raises(ValueError, match="weight must be"):
        ops.linear_batched(a, rnd(D, D + 64, seed=1004), out=torch.empty_like(res))
    with pytest.raises(ValueError, match="out must be"):
        ops.linear_batched(a, w, out=torch.empty(B, n + 1, D, device="cuda", dtype=bf16)[:, 1:-1])
    with pytest.raises(ValueError, match="residual must be"):
        ops.linear_batched(a, w, out=torch.empty_like(res), residual=res[:, :-1])
    with pytest.raises(ValueError, match="rows_per_group is not set"):
        ops.linear(a, w, row_gate=tab[:, 2 * D:], residual=res)
    with pytest.raises(ValueError, match="does not cover"):
        ops.linear(a, w, row_gate=tab[:2, 2 * D:], rows_per_group=n, residual=res)
    with pytest.raises(ValueError, match="does not cover"):
        ops.linear_batched(a, w, out=torch.empty_like(res), row_gate=tab[:2, 2 * D:], residual=res)
    with pytest.raises(ValueError, match="does not cover"):
        ops.layernorm(a, eps=1e-6, scale=tab[:, MOD_W - D // 2:], shift=tab[:, 0:], rows_per_group=n)
    with pytest.raises(ValueError, match="rows_per_group is not set"):
        ops.layernorm(a, eps=1e-6, scale=tab[:, D:], shift=tab[:, 0:])
    # the model's own calls are accepted
    ops.layernorm(a, eps=1e-6, scale=tab[:, D:], shift=tab[:, 0:], rows_per_group=n)
    ops.linear(a, w, row_gate=tab[:, 5 * D:], rows_per_group=n, residual=res)
    ops.linear_batched(a, w, out=torch.empty_like(res), row_gate=tab[:, 2 * D:], residual=res)
