"""SD / SDXL VAE decoder (AutoencoderKL.decode: block_out_channels 128 / 256 / 512 / 512, 32 groups, eps 1e-6) at its
production geometry against fp32 / fp64.

Bounds. A bf16 value stored once is off by up to 2^-9 of itself, and by 2^-8 after it is re-rounded, so every check is
|out - ref| <= 2^-8 |ref| + ATOL_RMS * rms(ref) plus a normwise ||out - ref|| / ||ref|| <= L2_MAX for the model-level
ones. Measured on an H100 80GB HBM3 (700 W power limit), as the largest excess over 2^-8 |ref| in units of rms(ref) /
the largest normwise error, with the bounds and their headroom:
  - kernels per call (conv3x3, upsample conv, shortcut, small-Cin convs, GroupNorm, P.V GEMM): 4.9e-5 (P.V with
    K = 15808 split on 7 clusters; convs 1.7e-5, GroupNorm 2.1e-5); bound 1e-4 (2.0x);
  - GroupNorm at its range edges (|mean| / std 0 to 2^8, RMS 1e-3 to 1e4, on the two longest chains): 3.9e-5; same
    bound (2.6x). The kernel before this suite summed x and x^2 about 0 and added the int64 partials in int64: at RMS 1
    it was at 4.9e-3 / 0.13 / 4.8 for |mean| / std = 16 / 64 / 2^8, and at RMS 1e4 the totals of the squares wrapped
    (excess 6e7 at |mean| / std = 0);
  - fp32 score GEMM against fp64, as max |out - ref| / rms(ref): 4.8e-6; bound 1e-5 (2.1x);
  - softmax_rows: within 2^-8 |ref| everywhere (excess 0); bound 1e-4;
  - the whole mid attention against fp64: 6.0e-4 / 1.66e-3; bound 1.5e-3 / 3.5e-3 (2.5x / 2.1x);
  - per block (resnet, mid attention, upsampler) against the fp32 oracle: 0.0238 / 3.20e-3; bound 0.05 / 6e-3
    (2.1x / 1.9x);
  - final output against the fp32 oracle decode: 0.118 / 1.19e-2 (Open-Sora frames; 0.092 to 0.106 on the batch-8 and
    bucket decodes; one sample alone against its row of the batch 0.109 / 1.17e-2); bound 0.25 / 0.025 (2.1x / 2.1x).
    With the mid attention replaced by the identity the output is at 0.385 / 0.040 and fails both.

Part 1 checks the kernels at their call sites, derived from oracle.vae.vae_decoder_layout for the latent size: every
conv3x3 with the epilogue the model gives it, the fused upsample convs, the 1x1 shortcut GEMMs, conv_out (Cout = 3),
post_quant_conv / conv_in on the small-Cin kernel, nhwc_to_nchw, every GroupNorm, and the one-head mid attention in
pieces (fp32 score GEMM, softmax_rows, the P.V GEMM under every schedule) and whole. The geometries are SD 512^2 at
batch 8 (4096 tokens), SDXL 1024^2 at batch 8 (the benchmark's batch), the 1216 x 832 and 1344 x 768 buckets at batch 3
(ragged tiles, 15808 / 16128 tokens) and Open-Sora's 64 frames at 512^2 decoded in one call. GroupNorm is also run at
the range edges of its statistics on the two longest per-thread chains, and the calls whose tensors reach 2^31 (SDXL,
batch 8) and 2^32 elements (Open-Sora, 64 frames) are checked on the batch elements before, at and after the boundary.
Every reference is plain torch in fp32 (TF32 off) or fp64 on the same bf16 inputs, rounded to bf16 where the model
rounds. Weights of the fused upsample conv are multiples of 2^-12 with small integer numerators, so their per-parity
fold is exact and the reference nearest-2x + conv3x3 is the same operation as the kernel's.

Part 2 runs the whole decoder (synthetic weights from oracle.vae.init_vae_params) against oracle/vae.py evaluated on the
GPU in fp32. Every resnet, the mid attention and every upsampler is compared with the oracle on its own bf16 input, so
the bounds measure one block and not the accumulated drift; the final output is compared with the whole oracle decode.
"""
import pytest
import torch
import torch.nn.functional as F

from oracle import vae as OV
from test_sdxl_shapes_gpu import SCHEDULES, check_kernel, errors, exact_fold_weight, knobs, ops, record, rnd  # noqa: F401

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16

KERNEL_ATOL_RMS = 1e-4
SCORE_ATOL_RMS = 1e-5
ATTN_ATOL_RMS, ATTN_L2 = 1.5e-3, 3.5e-3
BLOCK_ATOL_RMS, BLOCK_L2 = 0.05, 6e-3
FINAL_ATOL_RMS, FINAL_L2 = 0.25, 0.025
EPS = 1e-6
KEYS = ("latent_channels", "out_channels", "block_out_channels", "layers_per_block", "norm_num_groups", "scaling_factor")
# name: (config, batch, latent H, latent W)
GEOMS = {"sd_512_b8": ("sd_vae", 8, 64, 64), "sdxl_1024_b8": ("sdxl_vae", 8, 128, 128),
         "bucket_152x104_b3": ("sdxl_vae", 3, 152, 104), "bucket_168x96_b3": ("sdxl_vae", 3, 168, 96)}
OPENSORA = ("sd_vae", 64, 64, 64)


@pytest.fixture(autouse=True)
def peak_memory():
    if torch.cuda.is_available():
        torch.cuda.reset_peak_memory_stats()
    yield
    if torch.cuda.is_available():
        print(f"MEASURE peak memory: {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
        torch.cuda.empty_cache()


def nchw(t):
    return t.float().permute(0, 3, 1, 2)


def nhwc(t):
    return t.permute(0, 2, 3, 1)


def batch_errors(out, ref_fn, idx):
    """Largest (excess, normwise error) over the batch elements idx of out against ref_fn(b) (NHWC, one element)."""
    worst = [0.0, 0.0]
    for b in idx:
        ref = ref_fn(b)
        assert out[b:b + 1].shape == ref.shape, (out.shape, ref.shape)
        assert bool(torch.isfinite(out[b].float()).all()), f"non-finite output in element {b}"
        e = errors(out[b:b + 1], ref)
        worst = [max(worst[0], e[0]), max(worst[1], e[1])]
        del ref
    return worst


def check_batch(out, ref_fn, what, atol_rms=KERNEL_ATOL_RMS, l2_max=None, idx=None):
    excess, l2 = batch_errors(out, ref_fn, range(out.shape[0]) if idx is None else idx)
    record(what, excess, l2)
    assert excess <= atol_rms and (l2_max is None or l2 <= l2_max), (what, excess, l2)


def rnd_nhwc(B, H, W, C, seed):
    """bf16 [B, H, W, C], generated one element at a time (the fp32 temporary of a 2^31-element tensor is 8 GB)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.empty(B, H, W, C, device="cuda", dtype=bf16)
    for b in range(B):
        x[b] = torch.randn(H, W, C, generator=g, device="cuda")
    return x


def sites(geom, ops_=None):
    cfg, B, h, w = GEOMS[geom]
    out, seen = [], set()
    for s in OV.vae_decoder_layout(OV.VAE_CONFIGS[cfg], B, h, w):
        key = (s["op"], s["H"], s["W"], s["cin"], s["cout"], s.get("residual"), s.get("silu"))
        if (ops_ is None or s["op"] in ops_) and key not in seen:
            seen.add(key)
            out.append(s)
    return out


def site_id(s):
    extra = {True: "+res", False: ""}.get(s.get("residual"), "") + {True: "+silu", False: ""}.get(s.get("silu"), "")
    return f"{s['op']}{extra}_{s['cin']}-{s['cout']}@{s['H']}x{s['W']}"


def site_params(ops_):
    return [pytest.param(g, s, id=f"{g}-{site_id(s)}") for g in GEOMS for s in sites(g, ops_)]


# ---------------------------------------------------------------------------------------------------------------------
# Part 1: the kernels at their VAE call sites
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("geom,s", site_params(("conv3x3", "shortcut")))
def test_conv_sites(ops, geom, s):
    """Every conv3x3 (conv2 adds the block input or its shortcut; conv_out has Cout = 3 and takes the direct epilogue)
    and every 1x1 shortcut GEMM (M = B H W rows)."""
    B, H, W, cin, cout = s["B"], s["H"], s["W"], s["cin"], s["cout"]
    x = rnd_nhwc(B, H, W, cin, seed=cin + H)
    bias = rnd(cout, seed=cout + 4, scale=0.05, dtype=torch.float32)
    what = f"{geom} {s['name']} {site_id(s)}"
    if s["op"] == "shortcut":
        w = rnd(cout, cin, seed=cout + 3, scale=cin ** -0.5)
        out = ops.linear(x, w, bias)
        check_batch(out, lambda b: (x[b:b + 1].float() @ w.float().t() + bias), what)
        return
    w = rnd(cout, 3, 3, cin, seed=cout + 3, scale=(9 * cin) ** -0.5)
    res = rnd_nhwc(B, H, W, cout, seed=cout + 6) if s["residual"] else None
    out = ops.conv3x3(x, w, bias, residual=res)
    wf = w.float().permute(0, 3, 1, 2)

    def ref(b):
        r = nhwc(F.conv2d(nchw(x[b:b + 1]), wf, bias, padding=1))
        return r if res is None else r + res[b:b + 1].float()
    check_batch(out, ref, what)
    if s["name"] == "decoder.conv_out":
        y = ops.nhwc_to_nchw(out, out_dtype=torch.float32)
        assert y.dtype == torch.float32 and torch.equal(y, out.float().permute(0, 3, 1, 2)), "nhwc_to_nchw"


@pytest.mark.parametrize("geom,s", site_params(("up2x",)))
def test_upsample_conv_sites(ops, geom, s):
    B, H, W, C = s["B"], s["H"], s["W"], s["cin"]
    w = exact_fold_weight(C, C, seed=C + H)
    bias = rnd(C, seed=C + H + 1, scale=0.05, dtype=torch.float32)
    x = rnd_nhwc(B, H, W, C, seed=C + H + 2)
    out = ops.conv3x3_up2x(x, ops.fold_upsample_conv_weight(w), bias)
    wf = w.float().permute(0, 3, 1, 2)
    check_batch(out, lambda b: nhwc(F.conv2d(F.interpolate(nchw(x[b:b + 1]), scale_factor=2.0, mode="nearest"), wf,
                                             bias, padding=1)), f"{geom} {s['name']} {site_id(s)}")


@pytest.mark.parametrize("x_dtype", [torch.float32, bf16], ids=["fp32_in", "bf16_in"])
@pytest.mark.parametrize("geom", list(GEOMS))
def test_small_cin_sites(ops, geom, x_dtype):
    """post_quant_conv (1x1 on 4 channels, run as a centre-tap 3x3 with the output padded to 8 channels) and conv_in
    (8 -> 512) on the small-Cin kernel, plus the nchw_to_nhwc cast of the latents that feeds them."""
    cfg, B, h, w = GEOMS[geom]
    g = torch.Generator(device="cuda").manual_seed(h + w)
    z = torch.randn(B, 4, h, w, generator=g, device="cuda") / OV.VAE_CONFIGS[cfg]["scaling_factor"]
    zn = ops.nchw_to_nhwc(z)
    assert torch.equal(zn, z.permute(0, 2, 3, 1).to(bf16)), "nchw_to_nhwc"
    x = zn.to(x_dtype) if x_dtype == bf16 else z.permute(0, 2, 3, 1).contiguous()
    wpq = torch.zeros(8, 3, 3, 4, device="cuda", dtype=bf16)
    wpq[:4, 1, 1, :] = rnd(4, 4, seed=1, scale=0.5)
    bpq = torch.zeros(8, device="cuda")
    bpq[:4] = rnd(4, seed=2, scale=0.05, dtype=torch.float32)
    y = ops.conv3x3_small_cin(x, wpq, bpq)
    # the kernel rounds fp32 inputs to bf16, as every other conv sees bf16 activations
    check_batch(y, lambda b: nhwc(F.conv2d(nchw(x[b:b + 1].to(bf16)), wpq.float().permute(0, 3, 1, 2), bpq, padding=1)),
                f"{geom} post_quant_conv {x_dtype}")
    assert not bool(y[..., 4:].any()), "post_quant_conv padding channels must be zero"
    win = torch.zeros(512, 3, 3, 8, device="cuda", dtype=bf16)
    win[..., :4] = rnd(512, 3, 3, 4, seed=3, scale=36 ** -0.5)
    bin_ = rnd(512, seed=4, scale=0.05, dtype=torch.float32)
    x8 = y if x_dtype == bf16 else y.float()
    out = ops.conv3x3_small_cin(x8, win, bin_)
    check_batch(out, lambda b: nhwc(F.conv2d(nchw(x8[b:b + 1].to(bf16)), win.float().permute(0, 3, 1, 2), bin_, padding=1)),
                f"{geom} conv_in {x_dtype}")


def groupnorm_ref(x, gamma, beta, G, silu):
    """fp64 GroupNorm (+ SiLU) of one NHWC element."""
    y = F.group_norm(x.double().permute(0, 3, 1, 2), G, gamma.double(), beta.double(), EPS)
    return nhwc(F.silu(y) if silu else y)


def channel_offsets(C, seed):
    """Per-channel offsets and scales, so the channels of a group do not share one distribution."""
    return (0.5 * rnd(C, seed=seed, dtype=torch.float32), 1.0 + 0.5 * rnd(C, seed=seed + 1, dtype=torch.float32).abs())


@pytest.mark.parametrize("geom,s", site_params(("groupnorm",)))
def test_groupnorm_sites(ops, geom, s):
    """Every GroupNorm: 4 (128 channels) to 16 (512) channels per group, up to 8.4 M elements per group."""
    B, H, W, C, G = s["B"], s["H"], s["W"], s["cin"], s["groups"]
    off, sc = channel_offsets(C, seed=C + H)
    x = rnd_nhwc(B, H, W, C, seed=C + H + 2)
    for b in range(B):
        x[b] = (x[b].float() * sc + off).to(bf16)
    gamma = 1.0 + 0.1 * rnd(C, seed=3, dtype=torch.float32)
    beta = 0.1 * rnd(C, seed=4, dtype=torch.float32)
    out = ops.groupnorm_nhwc(x, gamma, beta, groups=G, eps=EPS, silu=s["silu"])
    check_batch(out, lambda b: groupnorm_ref(x[b:b + 1], gamma, beta, G, s["silu"]), f"{geom} {s['name']} {site_id(s)}")


# ---- GroupNorm at the edges of its statistics ------------------------------------------------------------------------
RATIOS = (0.0, 16.0, 64.0, 256.0)   # |mean| / std of a group
RMSS = (1e-3, 1.0, 1e4)
EDGE_CASES = [(r, q) for r in RATIOS for q in RMSS]
# the two longest per-thread chains: up_blocks.3.resnets.0.norm1 (256 channels at full resolution) of the SDXL decode at
# batch 8 (8.4 M elements per group, ~2000 values per thread) and of Open-Sora's 64 frames at 512^2 (~3600 per thread)
LONG_CHAINS = {"sdxl_1024_b8": (8, 1024, 1024), "opensora_64f": (64, 512, 512)}


def edge_input(B, H, W, C, G, seed):
    """Group g of element b holds the case EDGE_CASES[(b * G + g) % 12]: N(ratio, 1) scaled to the case's RMS. Returns
    the bf16 tensor and the case of each (element, group)."""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.empty(B, H, W, C, device="cuda", dtype=bf16)
    case = torch.tensor([[(b * G + g) % len(EDGE_CASES) for g in range(G)] for b in range(B)])
    ratio = torch.tensor([r for r, _ in EDGE_CASES], device="cuda")
    rms = torch.tensor([q for _, q in EDGE_CASES], device="cuda")
    for b in range(B):
        cg = case[b].cuda().repeat_interleave(C // G)
        x[b] = ((torch.randn(H, W, C, generator=gen, device="cuda") + ratio[cg]) * (rms[cg] / (ratio[cg] ** 2 + 1).sqrt())).to(bf16)
    return x, case


@pytest.mark.parametrize("silu", [False, True], ids=["plain", "silu"])
@pytest.mark.parametrize("chain", list(LONG_CHAINS))
def test_groupnorm_range_edges(ops, chain, silu):
    """Every (|mean| / std, RMS) combination on both long-chain geometries, each as whole groups of the real call, with
    eps 1e-6; per case the largest excess over all checked groups. Two runs are bit-identical."""
    B, H, W = LONG_CHAINS[chain]
    C, G = 256, 32
    x, case = edge_input(B, H, W, C, G, seed=B + H)
    gamma = 1.0 + 0.1 * rnd(C, seed=5, dtype=torch.float32)
    beta = 0.1 * rnd(C, seed=6, dtype=torch.float32)
    out = ops.groupnorm_nhwc(x, gamma, beta, groups=G, eps=EPS, silu=silu)
    again = ops.groupnorm_nhwc(x, gamma, beta, groups=G, eps=EPS, silu=silu)
    assert all(torch.equal(out[b], again[b]) for b in range(B)), "two runs differ"
    del again
    worst = {}
    for b in sorted({0, 1, B // 2, B - 1}):
        ref = groupnorm_ref(x[b:b + 1], gamma, beta, G, silu)
        for g in range(G):
            cs = slice(g * C // G, (g + 1) * C // G)
            e = errors(out[b:b + 1, ..., cs], ref[..., cs])[0]
            k = EDGE_CASES[case[b, g]]
            worst[k] = max(worst.get(k, 0.0), e)
        del ref
    assert len(worst) == len(EDGE_CASES)
    bad = []
    for (r, q), e in sorted(worst.items()):
        record(f"groupnorm edge {chain} silu={silu} mean/std={r:g} rms={q:g}", e)
        if e > KERNEL_ATOL_RMS:
            bad.append((r, q, e))
    assert not bad, f"GroupNorm outside its bound (mean/std, rms, excess): {bad}"


# ---- the mid attention in pieces and whole ---------------------------------------------------------------------------
TOKENS = [4096, 15808, 16128, 16384]
HEAD = 512


@pytest.mark.parametrize("N", TOKENS)
def test_attention_score_gemm(ops, N):
    """scores = q k^T in fp32 (K = 512) against fp64; the output is not rounded to bf16, so the bound is absolute."""
    q, k = rnd(N, HEAD, seed=N), rnd(N, HEAD, seed=N + 1)
    s = ops.linear(q, k, out_fp32=True)
    assert s.dtype == torch.float32 and s.shape == (N, N)
    ref = q.double() @ k.double().t()
    err = ((s.double() - ref).abs().max() / ref.pow(2).mean().sqrt()).item()
    record(f"score gemm N={N}", err)
    assert err <= SCORE_ATOL_RMS, (N, err)


@pytest.mark.parametrize("spread", [1.0, 30.0], ids=["realistic", "large_range"])
@pytest.mark.parametrize("N", TOKENS)
def test_softmax_rows_long(ops, N, spread):
    """softmax_rows on rows of the mid attention's length; scores * scale ~ N(0, spread^2) (30: weights over e^+-90)."""
    M, scale = 512, HEAD ** -0.5
    g = torch.Generator(device="cuda").manual_seed(N)
    x = torch.randn(M, N, generator=g, device="cuda") * (spread / scale)
    y = ops.softmax_rows(x, scale=scale)
    ref = torch.softmax(x.double() * scale, -1)
    check_kernel(y, ref, f"softmax N={N} spread={spread}", KERNEL_ATOL_RMS)
    assert torch.equal(y, ops.softmax_rows(x, scale=scale))


@pytest.mark.parametrize("sched", SCHEDULES, ids=lambda s: f"sk{s[0]}c{s[1]}")
@pytest.mark.parametrize("N", TOKENS)
def test_attention_pv_gemm(ops, N, sched):
    """o = P V with K = N (up to 256 k-blocks): stream-K as shipped, round-robin, forced splits and 7 clusters."""
    g = torch.Generator(device="cuda").manual_seed(N + 7)
    p = torch.softmax(torch.randn(N, N, generator=g, device="cuda") * 2.0, -1).to(bf16)
    v = rnd(N, HEAD, seed=N + 8)
    with knobs(streamk=sched[0], clusters=sched[1]):
        o = ops.linear(p, v.t().contiguous())
    check_kernel(o, p.double() @ v.double(), f"pv gemm N={N} streamk={sched[0]} clusters={sched[1]}")


@pytest.fixture(scope="module")
def vae(ops):
    """Decoders from seeded synthetic weights per config, and the same weights in fp32 on the device for the oracle."""
    from paddlemix_b200.ppdiffusers.autoencoder_kl import AutoencoderKL
    models = {}

    def get(cfg_name):
        if cfg_name not in models:
            cfg = OV.VAE_CONFIGS[cfg_name]
            P = OV.init_vae_params(cfg, seed=3)
            model = AutoencoderKL(**{k: cfg[k] for k in KEYS}).load_state_dict(P, device=0)
            models[cfg_name] = (model, {k: v.cuda() for k, v in P.items()})
        return models[cfg_name]
    yield get
    models.clear()


ATT = "decoder.mid_block.attentions.0"


@pytest.mark.parametrize("geom", list(GEOMS))
def test_mid_attention_vs_fp64(vae, geom):
    """The whole _mid_attention (GroupNorm, fused qkv GEMM, per-image score / softmax / PV, to_out + residual) against
    fp64 attention on the same bf16 input."""
    cfg, B, h, w = GEOMS[geom]
    model, Pd = vae(cfg)
    off, sc = channel_offsets(HEAD, seed=11)
    x = (rnd_nhwc(B, h, w, HEAD, seed=12).float() * sc + off).to(bf16)
    out = model._mid_attention(x)
    P64 = {k: v.double() for k, v in Pd.items() if k.startswith(ATT)}
    check_batch(out, lambda b: nhwc(OV._mid_attention(x[b:b + 1].double().permute(0, 3, 1, 2), P64, ATT, 32)),
                f"{geom} mid attention", ATTN_ATOL_RMS, ATTN_L2)


# ---- tensors past 2^31 elements --------------------------------------------------------------------------------------
BOUNDARY = {"sdxl_1024_b8": (8, 128), "opensora_64f": (64, 64)}   # (batch, latent size): 2^31 / 2^32 elements


@pytest.mark.parametrize("geom", list(BOUNDARY))
def test_boundary_calls(ops, geom):
    """up_blocks.2's upsampler (256 channels at full resolution: 2^31 elements at SDXL batch 8, 2^32 at 64 frames), then
    up_blocks.3.resnets.0 as the model runs it (norm1, conv1 256 -> 128, norm2, the 1x1 shortcut over M = 8.4 M / 16.8 M
    rows, conv2 + shortcut). Checked on the first and last element and on those holding byte offset 2^31, element 2^31 /
    byte offset 2^32; every op is per element, so the fp32 / fp64 reference needs only that element."""
    B, h = BOUNDARY[geom]
    S = 8 * h
    Ci, Co, G = 256, 128, 32
    per = S * S * Ci
    idx = sorted({0, (2 ** 30) // per, min(B - 1, (2 ** 31) // per), B - 1})
    x = rnd_nhwc(B, S // 2, S // 2, Ci, seed=21)
    wu = exact_fold_weight(Ci, Ci, seed=22)
    bu = rnd(Ci, seed=23, scale=0.05, dtype=torch.float32)
    up = ops.conv3x3_up2x(x, ops.fold_upsample_conv_weight(wu), bu)
    assert up.numel() == B * per and up.numel() >= 2 ** 31
    check_batch(up, lambda b: nhwc(F.conv2d(F.interpolate(nchw(x[b:b + 1]), scale_factor=2.0, mode="nearest"),
                                            wu.float().permute(0, 3, 1, 2), bu, padding=1)), f"{geom} up2x", idx=idx)
    del x
    g1, b1 = 1.0 + 0.1 * rnd(Ci, seed=24, dtype=torch.float32), 0.1 * rnd(Ci, seed=25, dtype=torch.float32)
    n1 = ops.groupnorm_nhwc(up, g1, b1, groups=G, eps=EPS, silu=True)
    check_batch(n1, lambda b: groupnorm_ref(up[b:b + 1], g1, b1, G, True), f"{geom} norm1", idx=idx)
    w1, c1 = rnd(Co, 3, 3, Ci, seed=26, scale=(9 * Ci) ** -0.5), rnd(Co, seed=27, scale=0.05, dtype=torch.float32)
    h1 = ops.conv3x3(n1, w1, c1)
    check_batch(h1, lambda b: nhwc(F.conv2d(nchw(n1[b:b + 1]), w1.float().permute(0, 3, 1, 2), c1, padding=1)),
                f"{geom} conv1", idx=idx)
    del n1
    g2, b2 = 1.0 + 0.1 * rnd(Co, seed=28, dtype=torch.float32), 0.1 * rnd(Co, seed=29, dtype=torch.float32)
    n2 = ops.groupnorm_nhwc(h1, g2, b2, groups=G, eps=EPS, silu=True)
    check_batch(n2, lambda b: groupnorm_ref(h1[b:b + 1], g2, b2, G, True), f"{geom} norm2", idx=idx)
    del h1
    ws, cs = rnd(Co, Ci, seed=30, scale=Ci ** -0.5), rnd(Co, seed=31, scale=0.05, dtype=torch.float32)
    res = ops.linear(up, ws, cs)
    check_batch(res, lambda b: up[b:b + 1].float() @ ws.float().t() + cs, f"{geom} shortcut", idx=idx)
    del up
    w2, c2 = rnd(Co, 3, 3, Co, seed=32, scale=(9 * Co) ** -0.5), rnd(Co, seed=33, scale=0.05, dtype=torch.float32)
    out = ops.conv3x3(n2, w2, c2, residual=res)
    check_batch(out, lambda b: nhwc(F.conv2d(nchw(n2[b:b + 1]), w2.float().permute(0, 3, 1, 2), c2, padding=1)) +
                res[b:b + 1].float(), f"{geom} conv2 + shortcut", idx=idx)


# ---------------------------------------------------------------------------------------------------------------------
# Part 2: the decoder against the oracle, block by block
# ---------------------------------------------------------------------------------------------------------------------
def latents(cfg_name, B, h, w, seed):
    """Latents as the pipeline hands them to decode (divided by the scaling factor), rounded to bf16 as decode rounds
    them, so the oracle sees the same input."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    z = torch.randn(B, 4, h, w, generator=g, device="cuda") / OV.VAE_CONFIGS[cfg_name]["scaling_factor"]
    return z.to(bf16).float()


def oracle_decode(cfg_name, Pd, z, b):
    with torch.no_grad():
        return nhwc(OV.vae_decode(OV.VAE_CONFIGS[cfg_name], Pd, z[b:b + 1]))


class Capture:
    """Wraps the decoder's blocks: each call is compared with the oracle on its own bf16 input, per batch element,
    while the call's tensors are alive (keeping them all would not fit at batch 8, 1024^2)."""

    def __init__(self, monkeypatch, Pd, G):
        from paddlemix_b200.ppdiffusers import autoencoder_kl as A
        from paddlemix_b200.ppdiffusers import unet_2d_condition as U
        self.results = []

        def ref_fn(kind, obj, x):
            if kind == "resnet":
                return lambda b: nhwc(OV._resnet(nchw(x[b:b + 1]), Pd, obj.name, G))
            if kind == "attention":
                return lambda b: nhwc(OV._mid_attention(nchw(x[b:b + 1]), Pd, ATT, G))
            return lambda b: nhwc(F.conv2d(F.interpolate(nchw(x[b:b + 1]), scale_factor=2.0, mode="nearest"),
                                           Pd[obj.name + ".weight"], Pd[obj.name + ".bias"], padding=1))

        def wrap(cls, attr, kind):
            real = getattr(cls, attr)

            def spy(self_, x):
                out = real(self_, x)
                with torch.no_grad():
                    e = batch_errors(out, ref_fn(kind, self_, x), range(x.shape[0]))
                self.results.append((kind, getattr(self_, "name", ATT), e))
                return out
            monkeypatch.setattr(cls, attr, spy)

        wrap(A._VaeResnet, "__call__", "resnet")
        wrap(A.AutoencoderKL, "_mid_attention", "attention")
        wrap(U._Conv3x3, "up2x", "up")


DECODE_CASES = ["sd_512_b8", "sdxl_1024_b8", "bucket_152x104_b3"]


@pytest.mark.parametrize("geom", DECODE_CASES)
def test_decoder_blocks_vs_oracle(vae, geom, monkeypatch):
    cfg_name, B, h, w = GEOMS[geom]
    model, Pd = vae(cfg_name)
    cfg = OV.VAE_CONFIGS[cfg_name]
    z = latents(cfg_name, B, h, w, seed=41)
    cap = Capture(monkeypatch, Pd, cfg["norm_num_groups"])
    out = model.decode(z).sample
    monkeypatch.undo()
    kinds = [k for k, _, _ in cap.results]
    n_res = 2 + len(cfg["block_out_channels"]) * (cfg["layers_per_block"] + 1)
    assert kinds.count("resnet") == n_res and kinds.count("attention") == 1
    assert kinds.count("up") == len(cfg["block_out_channels"]) - 1
    bad = []
    for kind, name, (excess, l2) in cap.results:
        record(f"{geom} {name}", excess, l2)
        if not (excess <= BLOCK_ATOL_RMS and l2 <= BLOCK_L2):
            bad.append((name, excess, l2))
    assert not bad, bad
    assert out.shape == (B, 3, 8 * h, 8 * w) and out.dtype == torch.float32
    check_batch(nhwc(out), lambda b: oracle_decode(cfg_name, Pd, z, b), f"{geom} output", FINAL_ATOL_RMS, FINAL_L2)


def test_decoder_negative_control(vae, monkeypatch):
    """The final-output bound bites: with the mid attention replaced by the identity the decode must fail it."""
    from paddlemix_b200.ppdiffusers.autoencoder_kl import AutoencoderKL
    model, Pd = vae("sd_vae")
    z = latents("sd_vae", 2, 64, 64, seed=43)
    monkeypatch.setattr(AutoencoderKL, "_mid_attention", lambda self, x: x)
    out = nhwc(model.decode(z).sample)
    monkeypatch.undo()
    excess, l2 = batch_errors(out, lambda b: oracle_decode("sd_vae", Pd, z, b), range(2))
    record("negative control: identity mid attention", excess, l2)
    assert excess > FINAL_ATOL_RMS or l2 > FINAL_L2, (excess, l2)


def test_decoder_sample_independence_and_determinism(vae):
    """On the 152 x 104 bucket each sample decoded alone matches its row of the batch (within the output bound: the
    GroupNorm partitions and the stream-K splits depend on the batch size), and two runs are bit-identical."""
    cfg_name, B, h, w = GEOMS["bucket_152x104_b3"]
    model, _ = vae(cfg_name)
    z = latents(cfg_name, B, h, w, seed=44)
    out = model.decode(z).sample
    assert torch.equal(out, model.decode(z).sample), "two decodes differ"
    for b in range(B):
        one = model.decode(z[b:b + 1]).sample
        check_batch(nhwc(one), lambda _: nhwc(out[b:b + 1]), f"sample {b} alone vs in the batch", FINAL_ATOL_RMS,
                    FINAL_L2)
    for b in range(1, B):
        assert (out[b] - out[0]).abs().max() > 0.1 * out.abs().max(), "samples collapsed"


def test_opensora_video_decode(vae):
    """VideoAutoencoderKL with micro_batch_size None (the default): all 64 frames of a 512^2 video in one decode call
    (2^32-element tensors at full resolution); frames 0, 31, 32 and 63 against the fp32 oracle."""
    from paddlemix_b200.opensora.vae import SCALING_FACTOR, VideoAutoencoderKL
    cfg_name, T, h, w = OPENSORA
    model, Pd = vae(cfg_name)
    g = torch.Generator(device="cuda").manual_seed(45)
    z = torch.randn(1, 4, T, h, w, generator=g, device="cuda")
    video = VideoAutoencoderKL(model, micro_batch_size=None).decode(z)
    assert video.shape == (1, 3, T, 8 * h, 8 * w)
    frames = (z[0].permute(1, 0, 2, 3) / SCALING_FACTOR).to(bf16).float()
    out = nhwc(video[0].permute(1, 0, 2, 3))
    check_batch(out, lambda b: oracle_decode(cfg_name, Pd, frames, b), "opensora frames", FINAL_ATOL_RMS, FINAL_L2,
                idx=[0, 31, 32, 63])
