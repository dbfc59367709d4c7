"""SDXL-base UNet (channels 320 / 640 / 1280, 1 / 2 / 10 transformer blocks per stack, text context 2048) at its
production geometry against fp32 / fp64.

Part 1 checks the kernels at their SDXL call sites, derived from oracle.unet.unet_layout for the latent size: the
folded-LayerNorm chain of a 1280-wide block (producer statistics feeding the next consumer, FF2 with K = 5120 under
stream-K), the range edges the header states for that fold, the fused upsample convs, every 3x3 conv with the epilogue
the model gives it, the GroupNorm over the virtual concat [h | skip] and the two-GEMM shortcut over it. Batch 8 at
128 x 128 is the benchmark's geometry; 152 x 104 (the 1216 x 832 bucket, 38 x 26 at the 1280 level) gives ragged tiles,
conv boxes that run past the batch and 988-token rows. Every reference is plain torch in fp32 (TF32 off) or fp64 on the
same bf16 inputs, rounded to bf16 where the model rounds. Weights of the fused upsample conv are multiples of 2^-12
with small integer numerators, so their per-parity fold is exact and the reference nearest-2x + conv3x3 is the same
operation as the kernel's.

Part 2 runs the full SDXL UNet (synthetic weights) against oracle/unet.py evaluated on the GPU in fp32. Every resnet,
Transformer2D, BasicTransformerBlock and upsampler is captured with its bf16 input and compared with the oracle on that
same input, so the bounds measure one block and not the accumulated drift; the time embedding, every row-statistics
table entering a block and the final output are compared too.

Bounds. A bf16 value stored once is off by up to 2^-9 of itself, and by 2^-8 after it is re-rounded, so every check is
|out - ref| <= 2^-8 |ref| + ATOL_RMS * rms(ref) plus a normwise ||out - ref|| / ||ref|| <= L2_MAX for the model-level
ones. Measured on an H100 80GB HBM3 (700 W power limit), as the largest excess over 2^-8 |ref| in units of rms(ref) /
the largest normwise error, with the bounds and their headroom:
  - kernels (GEMM, conv, upsample conv, GroupNorm, shortcut), per call: 6.7e-5 (conv1 2560 -> 1280 on 38 x 26);
    bound 1.5e-4 (2.2x);
  - folded-LayerNorm consumers of the block chain against fp64 Linear(LayerNorm(h)): 1.6e-4; bound 4e-4 (2.5x);
  - the same at the range edges: 6.8e-6 at |mean| / std = 0, 3.1e-5 at 16, 5.7e-4 at 2^8 (K = 1280, RMS 1.8e4: the
    fp32 tensor-core sum acc - mean colsum cancels |mean| / std, still under the output's own bf16 step); bound 1e-3
    (1.75x). With the per-row mean / variance rebuilt in fp32, as before this suite, the 2^8 rows were at 3.2e-3 to
    8.1e-3;
  - row statistics against fp64 sums of the stored bf16 rows, after the table's 2^-25 resolution per tile: 1.6e-7 of
    sum |x| / sum x^2; bound 4e-7 (2.5x);
  - per block (resnet, BasicTransformerBlock, upsampler): 0.0280 / 3.20e-3; bound 0.05 / 6e-3 (1.8x / 1.9x);
  - per Transformer2D stack (up to 10 blocks): 0.0363 / 7.01e-3; bound 0.07 / 1.4e-2 (1.9x / 2.0x);
  - time embedding (bf16 MLPs against fp32): 0.0113 / 2.68e-3; bound 0.02 / 5e-3 (1.8x / 1.9x);
  - whole forward, all schedules and the explicit-LayerNorm path: 0.0405 / 7.67e-3; bound 0.07 / 1.4e-2 (1.7x / 1.8x);
  - one sample alone against its row of the batch on 152 x 104: 0.0349 / 8.23e-3; same bound (2.0x / 1.7x).
The earlier model test allowed 4 % of the largest output value.

Part 3 runs the 2-step Euler CFG pipeline at 128 x 128, batch 2 (4 model rows), with and without the CUDA graph: the
graph captures the split GEMMs and the 31-table statistics arenas, and must give the eager result bit for bit.
"""
import ctypes
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import unet as O

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16

CFG = O.UNET_CONFIGS["sdxl"]
LAYOUT = O.unet_layout(CFG)
BNS = [32, 64, 128, 160, 192, 224, 256]
RTOL = 2.0 ** -8
KERNEL_ATOL_RMS = 1.5e-4
LN_ATOL_RMS = 4e-4
EDGE_ATOL_RMS = 1e-3
STATS_RTOL = 4e-7
BLOCK_ATOL_RMS, BLOCK_L2 = 0.05, 6e-3
STACK_ATOL_RMS, STACK_L2 = 0.07, 1.4e-2
EMBED_ATOL_RMS, EMBED_L2 = 0.02, 5e-3
FINAL_ATOL_RMS, FINAL_L2 = 0.07, 1.4e-2
LN_EPS = 1e-5
# (streamk, max clusters): round-robin | stream-K as shipped | every GEMM with >= 8 k-blocks split | the same on 7
# clusters (odd tile counts per cluster)
SCHEDULES = [(0, 0), (1, 0), (2, 0), (2, 7)]
SQUARE, BUCKET = (8, 128, 128), (3, 152, 104)   # (batch, latent H, latent W)


def record(what, excess, l2=None):
    print(f"MEASURE {what}: excess {excess:.4g}" + ("" if l2 is None else f" l2 {l2:.4g}"))


@pytest.fixture(scope="module")
def ops():
    from paddlemix_b200 import ops as _ops
    from paddlemix_b200._lib import lib
    _ops.init(0)
    for f in (lib.b200mix_debug_streamk, lib.b200mix_debug_max_clusters):
        f.argtypes, f.restype = [ctypes.c_int], None
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return _ops


class knobs:
    """Sets the GEMM schedule selectors for the duration of a block and restores the defaults in any case."""

    def __init__(self, streamk=None, clusters=0, bn=0):
        self.streamk, self.clusters, self.bn = streamk, clusters, bn

    def __enter__(self):
        from paddlemix_b200._lib import lib
        try:
            if self.streamk is not None:
                lib.b200mix_debug_streamk(self.streamk)
            lib.b200mix_debug_max_clusters(self.clusters)
            lib.b200mix_debug_force_bn(self.bn)
        except BaseException:
            self.__exit__()
            raise

    def __exit__(self, *a):
        from paddlemix_b200._lib import lib
        torch.cuda.synchronize()
        lib.b200mix_debug_streamk(int(os.environ.get("B200MIX_STREAMK", 1)))
        lib.b200mix_debug_max_clusters(0)
        lib.b200mix_debug_force_bn(0)


def rnd(*shape, seed, scale=1.0, dtype=bf16):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).to(dtype)


def errors(out, ref):
    """(excess over the bf16 storage bound in units of rms(ref), normwise relative error)."""
    o, r = out.double(), ref.double()
    d = (o - r).abs()
    rms = r.pow(2).mean().sqrt()
    return ((d - RTOL * r.abs()).clamp_min(0).max() / rms).item(), (d.norm() / r.norm()).item()


def check(out, ref, atol_rms, l2_max, what):
    assert out.shape == ref.shape, (what, out.shape, ref.shape)
    assert bool(torch.isfinite(out.float()).all()), f"{what}: non-finite output"
    excess, l2 = errors(out, ref)
    record(what, excess, l2)
    assert excess <= atol_rms and l2 <= l2_max, (what, excess, l2)


def check_kernel(out, ref, what, atol_rms=KERNEL_ATOL_RMS):
    assert out.shape == ref.shape, (what, out.shape, ref.shape)
    assert bool(torch.isfinite(out.float()).all()), f"{what}: non-finite output"
    excess = errors(out, ref)[0]
    record(what, excess)
    assert excess <= atol_rms, (what, excess)


def stats_error(st, h):
    """The fixed-point table of a producer against fp64 sums of the bf16 rows it stored: the largest error of the row
    sum and of the row sum of squares, in units of sum |x| and sum x^2 after the table's own resolution is taken off
    (each of the at most N / 32 tiles of a row rounds its partial to 2^-25)."""
    hd = h.reshape(-1, h.shape[-1]).double()
    tot = st.buf.double() / st.SCALE
    assert st.width == hd.shape[1] and tot.shape == (hd.shape[0], 2)
    quantum = hd.shape[1] / 32 * 2.0 ** -25
    e_sum = ((tot[:, 0] - hd.sum(1)).abs() - quantum).clamp_min(0) / hd.abs().sum(1).clamp_min(1e-30)
    e_sq = ((tot[:, 1] - (hd * hd).sum(1)).abs() - quantum).clamp_min(0) / (hd * hd).sum(1).clamp_min(1e-30)
    return max(e_sum.max().item(), e_sq.max().item())


def check_stats(st, h, what):
    err = stats_error(st, h)
    record(what + " stats", err)
    assert err <= STATS_RTOL, (what, err)


def layernorm64(h):
    hd = h.reshape(-1, h.shape[-1]).double()
    return F.layer_norm(hd, (hd.shape[1],), eps=LN_EPS)


# ---------------------------------------------------------------------------------------------------------------------
# Part 1: the kernels at their SDXL call sites
# ---------------------------------------------------------------------------------------------------------------------
C_TOP = LAYOUT["mid"]["ch"]   # 1280: the 10-block stacks
assert C_TOP == 1280 and LAYOUT["mid"]["tlayers"] == 10


@pytest.fixture(scope="module")
def block1280(ops):
    """Weights of one 1280-wide BasicTransformerBlock plus proj_in, with the three LayerNorms folded into their
    consumers the way _BasicTransformerBlock.load folds them."""
    C = C_TOP
    s = C ** -0.5
    W = {}
    W["proj_in"] = (rnd(C, C, seed=1, scale=s), rnd(C, seed=2, scale=0.05, dtype=torch.float32))
    for i, (name, n_out) in enumerate((("qkv", 3 * C), ("q2", C), ("ff1", 8 * C))):
        w = rnd(n_out, C, seed=10 + i, scale=s, dtype=torch.float32)
        gamma = 1.0 + 0.1 * rnd(C, seed=20 + i, dtype=torch.float32)
        beta = 0.05 * rnd(C, seed=30 + i, dtype=torch.float32)
        bias = None if name != "ff1" else 0.05 * rnd(n_out, seed=40, dtype=torch.float32)
        W[name] = ops.fold_layernorm_into_linear(w, gamma, beta, bias)
    for i, (name, k) in enumerate((("out1", C), ("out2", C), ("ff2", 4 * C))):
        W[name] = (rnd(C, k, seed=50 + i, scale=k ** -0.5), rnd(C, seed=60 + i, scale=0.05, dtype=torch.float32))
    return W


def consumer_ref(h, fold, glu=False):
    """fp64 Linear(LayerNorm(h)) with the folded weights the kernel reads (W' = bf16(W gamma), bias' = bias + W beta)."""
    w2, _, b2 = fold
    z = layernorm64(h) @ w2.double().t() + b2.double()
    return z[:, 0::2] * F.gelu(z[:, 1::2]) if glu else z


def ln_chain(ops, W, M, seed, ff2_bn=0):
    """proj_in (producer) -> qkv (consumer), to_out + residual (producer) -> attn2.to_q (consumer), to_out (producer)
    -> GEGLU FF1 (consumer), FF2 + residual (producer) -> the next block's qkv (consumer). The attention outputs are
    random stand-ins. Every consumer is checked against fp64 on the tensor the previous call stored, every table
    against fp64 sums. Returns the four statistics tables."""
    from paddlemix_b200._lib import lib
    C = C_TOP
    tables = ops.RowStats.arena(4, M, "cuda")
    n = rnd(M, C, seed=seed)
    h, st = ops.linear(n, *W["proj_in"], stats=tables[0])
    check_kernel(h, n.float() @ W["proj_in"][0].float().t() + W["proj_in"][1], f"M={M} proj_in")
    check_stats(st, h, f"M={M} proj_in")
    for step, (cons, prod) in enumerate((("qkv", "out1"), ("q2", "out2"), ("ff1", "ff2"))):
        w2, colsum, b2 = W[cons]
        glu = cons == "ff1"
        y = ops.linear(h, w2, b2, glu=ops.GLU_GEGLU if glu else ops.GLU_NONE, ln=(st, colsum, LN_EPS))
        check_kernel(y, consumer_ref(h, W[cons], glu), f"M={M} {cons} (folded LayerNorm)", LN_ATOL_RMS)
        a = y if glu else rnd(M, C, seed=seed + 1 + step)   # FF2 reads the GEGLU output; to_out an attention stand-in
        wp, bp = W[prod]
        lib.b200mix_debug_force_bn(ff2_bn if prod == "ff2" else 0)
        try:
            h2, st = ops.linear(a, wp, bp, residual=h, stats=tables[1 + step])
        finally:
            lib.b200mix_debug_force_bn(0)
        check_kernel(h2, a.float() @ wp.float().t() + bp + h.float(), f"M={M} {prod} + residual")
        check_stats(st, h2, f"M={M} {prod}")
        h = h2
    w2, colsum, b2 = W["qkv"]
    y = ops.linear(h, w2, b2, ln=(st, colsum, LN_EPS))
    check_kernel(y, consumer_ref(h, W["qkv"]), f"M={M} next block qkv (folded LayerNorm)", LN_ATOL_RMS)
    return tables


ROWS = [8 * 1024, 3 * 38 * 26]   # batch 8 at 32 x 32 | batch 3 at 38 x 26 (988 tokens per image)


@pytest.mark.parametrize("streamk,clusters", SCHEDULES)
@pytest.mark.parametrize("M", ROWS)
def test_folded_layernorm_chain_1280(ops, block1280, M, streamk, clusters):
    """The statistics chain of one 1280-wide block under every schedule; FF2 (K = 5120, 80 k-blocks) takes a stream-K
    head at batch 8 with the default schedule. Two runs give the same tables bit for bit."""
    with knobs(streamk=streamk, clusters=clusters):
        t1 = ln_chain(ops, block1280, M, seed=100)
        t2 = ln_chain(ops, block1280, M, seed=100)
    assert torch.equal(t1, t2), "fixed-point row statistics differ between two runs"


@pytest.mark.parametrize("bn", BNS)
@pytest.mark.parametrize("M", ROWS)
def test_folded_layernorm_chain_ff2_tile_widths(ops, block1280, M, bn):
    """The same chain with FF2 (the producer whose statistics feed the next block) forced to every tile width."""
    with knobs(streamk=1):
        ln_chain(ops, block1280, M, seed=200, ff2_bn=bn)


RMS_LIMIT = 0.9 * 2e4   # the header's range: a 1280-wide row of RMS 2e4 fills the int64 totals


def edge_rows(K, rows_per_case, seed):
    """Rows of every (|mean| / std, RMS, outliers) combination: |mean| / std in {0, 16, 2^8} for the bulk of the row,
    RMS in {1e-3, 1, RMS_LIMIT} for the whole row, and optionally three channels at 100x the bulk's std. Returns the
    fp32 rows (not yet rounded) and the case labels."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    parts, labels = [], []
    for ratio in (0.0, 16.0, 256.0):
        for rms in (1e-3, 1.0, RMS_LIMIT):
            for outliers in (False, True):
                z = torch.randn(rows_per_case, K, generator=g, device="cuda", dtype=torch.float64)
                if outliers:
                    idx = torch.randint(0, K, (rows_per_case, 3), generator=g, device="cuda")
                    sign = torch.randint(0, 2, (rows_per_case, 3), generator=g, device="cuda").double() * 2 - 1
                    z.scatter_(1, idx, 100.0 * sign)
                x = ratio + z
                x = x * (rms / x.pow(2).mean(1, keepdim=True).sqrt())
                parts.append(x)
                labels.append(f"mean/std={ratio:g} rms={rms:g}" + (" outliers" if outliers else ""))
    return torch.cat(parts).float(), labels


@pytest.mark.parametrize("K", [320, 640, 1280])
def test_folded_layernorm_range_edges(ops, K):
    """The fold at the edges of its stated range. A producer GEMM stores h = a @ w^T + residual, where the residual
    carries the row pattern and a @ w^T adds a small term of the row's own scale; its statistics then feed a consumer
    whose output is checked per case against fp64 Linear(LayerNorm(h))."""
    R = 70
    x, labels = edge_rows(K, R, seed=K)
    M = x.shape[0]
    res = x.to(bf16)
    scale = res.float().std(1, keepdim=True) * 0.01
    a = (rnd(M, 64, seed=K + 1, dtype=torch.float32) * scale).to(bf16)
    w = rnd(K, 64, seed=K + 2, scale=64 ** -0.5)
    h, st = ops.linear(a, w, None, residual=res, stats=True)
    assert bool(torch.isfinite(h.float()).all())
    N = 256
    wc = rnd(N, K, seed=K + 3, scale=K ** -0.5, dtype=torch.float32)
    gamma = 1.0 + 0.1 * rnd(K, seed=K + 4, dtype=torch.float32)
    beta = 0.05 * rnd(K, seed=K + 5, dtype=torch.float32)
    fold = ops.fold_layernorm_into_linear(wc, gamma, beta, 0.05 * rnd(N, seed=K + 6, dtype=torch.float32))
    y = ops.linear(h, fold[0], fold[2], ln=(st, fold[1], LN_EPS))
    ref = consumer_ref(h, fold)
    bad = []
    for i, lab in enumerate(labels):
        rows = slice(i * R, (i + 1) * R)
        excess, e_st = errors(y[rows], ref[rows])[0], stats_error(ops.RowStats(st.buf[rows], K), h[rows])
        record(f"K={K} {lab}", excess)
        record(f"K={K} {lab} stats", e_st)
        if not (excess <= EDGE_ATOL_RMS and e_st <= STATS_RTOL):
            bad.append((lab, excess, e_st))
    assert not bad, f"K={K}: folded LayerNorm outside its bounds (case, excess, statistics error): {bad}"


def upsample_sites():
    """(channels, low-resolution level) of every Upsample2D: up_blocks.0 at the 1280 level, up_blocks.1 at 640."""
    sites, level = [], len(LAYOUT["down"]) - 1
    for u in LAYOUT["up"]:
        if u["upsample"]:
            sites.append((u["out_ch"], level))
            level -= 1
    return sites


UP_SITES = upsample_sites()
assert UP_SITES == [(1280, 2), (640, 1)]


def exact_fold_weight(Cout, Cin, seed):
    """A 3x3 filter of small integer multiples of a power of two: sums of up to four taps stay exact in bf16, so the
    per-parity fold is exact."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    k = torch.randint(-31, 32, (Cout, 3, 3, Cin), generator=g, device="cuda").float()
    return (k * 2.0 ** -12).to(bf16)


def up2x_case(ops, B, H, W, C, sched, bn):
    w = exact_fold_weight(C, C, seed=C + H)
    w4 = ops.fold_upsample_conv_weight(w)
    bias = rnd(C, seed=C + H + 1, scale=0.05, dtype=torch.float32)
    x = rnd(B, H, W, C, seed=C + H + 2)
    with knobs(streamk=sched[0], clusters=sched[1], bn=bn):
        out = ops.conv3x3_up2x(x, w4, bias)
    wf = w.float().permute(0, 3, 1, 2)
    worst = 0.0
    for b in range(B):
        up = F.interpolate(x[b:b + 1].float().permute(0, 3, 1, 2), scale_factor=2.0, mode="nearest")
        ref = F.conv2d(up, wf, bias, padding=1).permute(0, 2, 3, 1)
        worst = max(worst, errors(out[b:b + 1], ref)[0])
    what = f"up2x B={B} {C}@{H}x{W} streamk={sched[0]} clusters={sched[1]} bn={bn}"
    record(what, worst)
    assert worst <= KERNEL_ATOL_RMS, (what, worst)


UP_CASES = [(B, H >> lvl, W >> lvl, C) for (B, H, W) in (SQUARE, BUCKET) for C, lvl in UP_SITES]


@pytest.mark.parametrize("sched", SCHEDULES, ids=lambda s: f"sk{s[0]}c{s[1]}")
@pytest.mark.parametrize("B,H,W,C", UP_CASES)
def test_upsample_conv_sites(ops, B, H, W, C, sched):
    """conv3x3_up2x at each SDXL upsampler: 1280 -> 1280 at the 1280 level is 4 taps x 20 = 80 k-blocks, so the
    stream-K head runs over the parity-major tile order."""
    up2x_case(ops, B, H, W, C, sched, 0)


@pytest.mark.parametrize("bn", BNS)
@pytest.mark.parametrize("B,H,W,C", [c for c in UP_CASES if c[3] == 1280])
def test_upsample_conv_1280_tile_widths(ops, B, H, W, C, bn):
    up2x_case(ops, B, H, W, C, (1, 0), bn)


def conv_sites():
    """Every 3x3 conv of SDXL as (kind, Cin, Cout, level): conv_in, the resnets' conv1 (per-sample time embedding
    added as row_add) and conv2 (residual, out_scale), the stride-2 downsamplers and conv_out. Duplicates dropped."""
    sites = [("conv_in", CFG["in_channels"], CFG["block_out_channels"][0], 0)]
    level = 0
    for d in LAYOUT["down"]:
        for j in range(d["layers"]):
            sites += [("conv1", d["in_ch"] if j == 0 else d["out_ch"], d["out_ch"], level),
                      ("conv2", d["out_ch"], d["out_ch"], level)]
        if d["downsample"]:
            sites.append(("down", d["out_ch"], d["out_ch"], level))
            level += 1
    m = LAYOUT["mid"]
    sites += [("conv1", m["ch"], m["ch"], level), ("conv2", m["ch"], m["ch"], level)]
    for u in LAYOUT["up"]:
        for j in range(u["layers"]):
            skip = u["in_ch"] if j == u["layers"] - 1 else u["out_ch"]
            rin = u["prev_ch"] if j == 0 else u["out_ch"]
            sites += [("conv1", rin + skip, u["out_ch"], level), ("conv2", u["out_ch"], u["out_ch"], level)]
        if u["upsample"]:
            level -= 1
    sites.append(("conv_out", CFG["block_out_channels"][0], CFG["out_channels"], 0))
    return list(dict.fromkeys(sites))


CONV_SITES = conv_sites()
assert ("conv1", 1920, 1280, 2) in CONV_SITES and ("conv1", 960, 640, 1) in CONV_SITES
assert ("down", 640, 640, 1) in CONV_SITES and ("conv_out", 320, 4, 0) in CONV_SITES


@pytest.mark.parametrize("geom", [SQUARE, BUCKET], ids=["b8_128x128", "b3_152x104"])
@pytest.mark.parametrize("kind,cin,cout,level", CONV_SITES)
def test_conv3x3_sites(ops, kind, cin, cout, level, geom):
    B, H0, W0 = geom
    H, W = H0 >> level, W0 >> level
    x = rnd(B, H, W, cin, seed=cin * 7 + level)
    w = rnd(cout, 3, 3, cin, seed=cout + 3, scale=(9 * cin) ** -0.5)
    bias = rnd(cout, seed=cout + 4, scale=0.05, dtype=torch.float32)
    radd = res = None
    osf = CFG["resnet_out_scale_factor"]
    scale = 1.0
    if kind == "conv_in":
        out = ops.conv3x3_small_cin(x, w, bias)
    elif kind == "conv1":
        radd = rnd(B, cout, seed=cout + 5, scale=0.5, dtype=torch.float32)
        out = ops.conv3x3(x, w, bias, row_add=radd)
    elif kind == "conv2":
        res = rnd(B, H, W, cout, seed=cout + 6)
        scale = 1.0 / osf
        out = ops.conv3x3(x, w, bias, residual=res, out_scale=scale)
    elif kind == "down":
        out = ops.conv3x3(x, w, bias, stride=2)
    else:
        out = ops.conv3x3(x, w, bias)
    wf = w.float().permute(0, 3, 1, 2)
    worst = 0.0
    for b in range(B):
        ref = F.conv2d(x[b:b + 1].float().permute(0, 3, 1, 2), wf, bias, stride=2 if kind == "down" else 1,
                       padding=1).permute(0, 2, 3, 1)
        if radd is not None:
            ref = ref + radd[b]
        if res is not None:
            ref = (ref + res[b:b + 1].float()) * scale
        worst = max(worst, errors(out[b:b + 1], ref)[0])
    what = f"{kind} {cin}->{cout} B={B} {H}x{W}"
    record(what, worst)
    assert worst <= KERNEL_ATOL_RMS, (what, worst)


def concat_sites():
    """(C1, C2, level) of every up-block resnet: GroupNorm over [h | skip] and the shortcut over the same concat."""
    sites, level = [], len(LAYOUT["down"]) - 1
    for u in LAYOUT["up"]:
        for j in range(u["layers"]):
            skip = u["in_ch"] if j == u["layers"] - 1 else u["out_ch"]
            sites.append((u["prev_ch"] if j == 0 else u["out_ch"], skip, u["out_ch"], level))
        if u["upsample"]:
            level -= 1
    return list(dict.fromkeys(sites))


CONCAT_SITES = concat_sites()
assert (1280, 640, 1280, 2) in CONCAT_SITES and (640, 320, 640, 1) in CONCAT_SITES and (640, 320, 320, 0) in CONCAT_SITES


@pytest.mark.parametrize("geom", [SQUARE, BUCKET], ids=["b8_128x128", "b3_152x104"])
@pytest.mark.parametrize("c1,c2,cout,level", CONCAT_SITES)
def test_concat_groupnorm_sites(ops, c1, c2, cout, level, geom):
    """GroupNorm + SiLU over [x1 | x2] with 32 groups: x1 and x2 carry different per-channel offsets (+2 / -1) and
    scales, so a group straddling the boundary computed on a wrong split is off by far more than the bound."""
    B, H0, W0 = geom
    H, W = H0 >> level, W0 >> level
    G = CFG["norm_num_groups"]
    x1 = (rnd(B, H, W, c1, seed=c1 + level) * 1.5 + 2.0).to(bf16)
    x2 = (rnd(B, H, W, c2, seed=c2 + level + 1) * 0.5 - 1.0).to(bf16)
    gamma = 1.0 + 0.1 * rnd(c1 + c2, seed=3, dtype=torch.float32)
    beta = 0.1 * rnd(c1 + c2, seed=4, dtype=torch.float32)
    out = ops.groupnorm_nhwc(x1, gamma, beta, x2=x2, groups=G, eps=CFG["norm_eps"], silu=True)
    worst = 0.0
    for b in range(B):
        xc = torch.cat([x1[b], x2[b]], -1).double().permute(2, 0, 1)[None]
        ref = F.silu(F.group_norm(xc, G, gamma.double(), beta.double(), CFG["norm_eps"])).permute(0, 2, 3, 1)
        worst = max(worst, errors(out[b:b + 1], ref)[0])
    what = f"concat groupnorm {c1}+{c2} B={B} {H}x{W}"
    record(what, worst)
    assert worst <= KERNEL_ATOL_RMS, (what, worst)


@pytest.mark.parametrize("streamk", [0, 2])
@pytest.mark.parametrize("geom", [SQUARE, BUCKET], ids=["b8_128x128", "b3_152x104"])
@pytest.mark.parametrize("c1,c2,cout,level", CONCAT_SITES)
def test_concat_shortcut_sites(ops, c1, c2, cout, level, geom, streamk):
    """The 1x1 shortcut over [x | skip] as the model runs it: res = x @ w[:, :c1]^T + b in bf16, then
    res = skip @ w[:, c1:]^T + res written over res itself."""
    B, H0, W0 = geom
    H, W = H0 >> level, W0 >> level
    x, skip = rnd(B, H, W, c1, seed=c1 + 11), rnd(B, H, W, c2, seed=c2 + 12)
    w = rnd(cout, c1 + c2, seed=cout + 13, scale=(c1 + c2) ** -0.5)
    bias = rnd(cout, seed=cout + 14, scale=0.05, dtype=torch.float32)
    with knobs(streamk=streamk):
        res = ops.linear(x, w[:, :c1], bias)
        res1 = res.clone()
        out = ops.linear(skip, w[:, c1:], None, residual=res, out=res)
    assert out.data_ptr() == res.data_ptr()
    ref1 = x.reshape(-1, c1).float() @ w[:, :c1].float().t() + bias
    check_kernel(res1.reshape(-1, cout), ref1, f"shortcut x half {c1}->{cout} B={B} {H}x{W} streamk={streamk}")
    ref = skip.reshape(-1, c2).float() @ w[:, c1:].float().t() + res1.reshape(-1, cout).float()
    check_kernel(out.reshape(-1, cout), ref, f"shortcut {c1}+{c2}->{cout} B={B} {H}x{W} streamk={streamk}")


# ---------------------------------------------------------------------------------------------------------------------
# Part 2: the model against the oracle, block by block
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sdxl(ops):
    """The full SDXL UNet from seeded synthetic weights, and the same weights in fp32 on the device for the oracle."""
    from paddlemix_b200.ppdiffusers.unet_2d_condition import UNet2DConditionModel
    P = O.init_params(O.unet_param_shapes(CFG), seed=1)
    keys = ("in_channels", "out_channels", "flip_sin_to_cos", "freq_shift", "down_block_types", "up_block_types",
            "block_out_channels", "layers_per_block", "norm_num_groups", "norm_eps", "cross_attention_dim",
            "transformer_layers_per_block", "attention_head_dim", "use_linear_projection", "addition_embed_type",
            "addition_time_embed_dim", "projection_class_embeddings_input_dim", "resnet_out_scale_factor")
    model = UNet2DConditionModel(**{k: CFG[k] for k in keys}).load_state_dict(P, device=0)
    Pd = {}
    for k in list(P):
        Pd[k] = P.pop(k).cuda()
    yield model, Pd
    del model, Pd
    torch.cuda.empty_cache()


CASES = {  # batch, latent H x W, timesteps (None = the scalar 500), time_ids per sample
    "bench_128x128_B2": (2, 128, 128, [981.0, 421.0]),
    "bucket_152x104_B3": (3, 152, 104, [999.0, 500.0, 1.0]),
    "bucket_168x96_B2_scalar_t": (2, 168, 96, None),
}


def make_inputs(B, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, CFG["in_channels"], H, W, generator=g).to(bf16).float()
    ctx = torch.randn(B, 77, CFG["cross_attention_dim"], generator=g).to(bf16).float()
    n_text = CFG["projection_class_embeddings_input_dim"] - 6 * CFG["addition_time_embed_dim"]
    text = torch.randn(B, n_text, generator=g).to(bf16).float()
    # original size, crop offsets, target size: different per sample
    ids = torch.tensor([[8.0 * H + 64 * b, 8.0 * W - 32 * b, 16.0 * b, 8.0 * b, 8.0 * H, 8.0 * W] for b in range(B)])
    return x.cuda(), ctx.cuda(), {"text_embeds": text.cuda(), "time_ids": ids.cuda()}


def oracle_emb(Pd, t, added, B):
    """The oracle's time + added-condition embedding (unet_forward's first step)."""
    t = t.reshape(-1).expand(B)
    emb = O.timestep_embedding_mlp(O.get_timestep_embedding(t, CFG["block_out_channels"][0], CFG["flip_sin_to_cos"],
                                                            CFG["freq_shift"]), Pd, "time_embedding")
    te = O.get_timestep_embedding(added["time_ids"].flatten(), CFG["addition_time_embed_dim"], CFG["flip_sin_to_cos"],
                                  CFG["freq_shift"]).reshape(B, -1)
    return emb + O.timestep_embedding_mlp(torch.cat([added["text_embeds"], te], -1), Pd, "add_embedding")


def nchw(t):
    return t.float().permute(0, 3, 1, 2).contiguous()


class Capture:
    """Wraps the model's block classes: records each call's bf16 inputs, output and entering row statistics."""

    def __init__(self, monkeypatch):
        from paddlemix_b200.ppdiffusers import unet_2d_condition as U
        self.calls = []
        calls = self.calls

        def wrap(cls, attr, kind):
            real = getattr(cls, attr)

            def spy(self_, *args, **kw):
                rec = dict(kind=kind, obj=self_, h=args[0].clone())
                if kind == "resnet":
                    skip = kw.get("skip")
                    rec["temb_all"], rec["skip"] = args[1], None if skip is None else skip.clone()
                if kind == "block":
                    hs = kw.get("h_stats")
                    rec["stats"] = None if hs is None else (hs.buf.clone(), hs.width)
                out = real(self_, *args, **kw)
                rec["out"] = (out[0] if isinstance(out, tuple) else out).clone()
                calls.append(rec)
                return out
            monkeypatch.setattr(cls, attr, spy)

        wrap(U._Resnet, "__call__", "resnet")
        wrap(U._Transformer2D, "__call__", "transformer")
        wrap(U._BasicTransformerBlock, "__call__", "block")
        wrap(U._Conv3x3, "up2x", "up")


_REF_CACHE = {}


def oracle_output(Pd, case):
    if case not in _REF_CACHE:
        B, H, W, ts = CASES[case]
        x, ctx, added = make_inputs(B, H, W, seed=7)
        t = torch.tensor(500.0, device="cuda") if ts is None else torch.tensor(ts, device="cuda")
        with torch.no_grad():
            _REF_CACHE[case] = O.unet_forward(CFG, Pd, x, t, ctx, added).cpu()
    return _REF_CACHE[case].cuda()


def run_model(model, case):
    B, H, W, ts = CASES[case]
    x, ctx, added = make_inputs(B, H, W, seed=7)
    t = 500.0 if ts is None else torch.tensor(ts, device="cuda")
    return model(x, t, ctx, added_cond_kwargs=added).sample


@pytest.mark.parametrize("case", list(CASES))
def test_sdxl_blocks_vs_oracle(sdxl, case, monkeypatch):
    model, Pd = sdxl
    B, H, W, ts = CASES[case]
    x, ctx, added = make_inputs(B, H, W, seed=7)
    cap = Capture(monkeypatch)
    t_model = 500.0 if ts is None else torch.tensor(ts, device="cuda")
    out = model(x, t_model, ctx, added_cond_kwargs=added).sample
    monkeypatch.undo()
    t = torch.tensor(500.0, device="cuda") if ts is None else torch.tensor(ts, device="cuda")
    G, eps, osf = CFG["norm_num_groups"], CFG["norm_eps"], CFG["resnet_out_scale_factor"]
    kinds = [c["kind"] for c in cap.calls]
    n_res = sum(d["layers"] for d in LAYOUT["down"]) + 2 + sum(u["layers"] for u in LAYOUT["up"])
    assert kinds.count("resnet") == n_res == len(model.resnets)
    assert kinds.count("transformer") == len(model.transformers)
    assert kinds.count("block") == sum(len(tr.blocks) for tr in model.transformers) == 70
    assert kinds.count("up") == len(UP_SITES)
    with torch.no_grad():
        emb = oracle_emb(Pd, t, added, B)
        temb_all = next(c for c in cap.calls if c["kind"] == "resnet")["temb_all"]
        s_emb = F.silu(emb)
        for r in model.resnets:
            off, size = r.temb_slice
            check(temb_all[:, off:off + size], O.linear(s_emb, Pd, r.name + ".time_emb_proj"), EMBED_ATOL_RMS,
                  EMBED_L2, f"{case} {r.name} time_emb_proj")
        for c in cap.calls:
            obj, h = c["obj"], c["h"]
            if c["kind"] == "resnet":
                xin = h if c["skip"] is None else torch.cat([h, c["skip"]], -1)
                ref = O.resnet_block(nchw(xin), emb, Pd, obj.name, G, eps, osf)
                check(c["out"], ref.permute(0, 2, 3, 1), BLOCK_ATOL_RMS, BLOCK_L2, f"{case} {obj.name}")
            elif c["kind"] == "transformer":
                heads = obj.blocks[0].attn1.heads
                ref = O.transformer_2d(nchw(h), ctx, Pd, obj.name, heads, len(obj.blocks), G, CFG["use_linear_projection"])
                check(c["out"], ref.permute(0, 2, 3, 1), STACK_ATOL_RMS, STACK_L2, f"{case} {obj.name}")
            elif c["kind"] == "block":
                ref = O.basic_transformer_block(h.float(), ctx, Pd, obj.name, obj.attn1.heads)
                check(c["out"], ref, BLOCK_ATOL_RMS, BLOCK_L2, f"{case} {obj.name}")
                assert c["stats"] is not None, f"{obj.name} ran without row statistics"
                buf, width = c["stats"]
                from paddlemix_b200.ops import RowStats
                check_stats(RowStats(buf, width), h, f"{case} {obj.name} entering")
            else:
                ref = F.conv2d(F.interpolate(nchw(h), scale_factor=2.0, mode="nearest"), Pd[obj.name + ".weight"],
                               Pd[obj.name + ".bias"], padding=1)
                check(c["out"], ref.permute(0, 2, 3, 1), BLOCK_ATOL_RMS, BLOCK_L2, f"{case} {obj.name}")
        cap.calls.clear()
        ref = O.unet_forward(CFG, Pd, x, t, ctx, added)
        _REF_CACHE[case] = ref.cpu()
    check(out, ref, FINAL_ATOL_RMS, FINAL_L2, f"{case} output")


@pytest.mark.parametrize("path", ["roundrobin", "streamk2_7clusters", "explicit_layernorm"])
def test_sdxl_other_paths_vs_oracle(sdxl, path, monkeypatch):
    """The same model with the round-robin schedule, with every GEMM of >= 8 k-blocks split on 7 clusters, and with the
    LayerNorms as explicit kernels instead of folded."""
    from paddlemix_b200.ppdiffusers import unet_2d_condition as U
    model, Pd = sdxl
    case = "bench_128x128_B2"
    ref = oracle_output(Pd, case)
    if path == "explicit_layernorm":
        monkeypatch.setattr(U._Transformer2D, "FOLD_LAYERNORM", False)
        out = run_model(model, case)
    else:
        with knobs(streamk=0) if path == "roundrobin" else knobs(streamk=2, clusters=7):
            out = run_model(model, case)
    check(out, ref, FINAL_ATOL_RMS, FINAL_L2, f"{case} output, {path}")


def test_sdxl_sample_independence_on_bucket(sdxl):
    """On 152 x 104 the conv boxes at the 1280 level span images: each sample run alone must match its row of the
    batch. The two runs split different GEMMs (the tile counts differ), so they differ by two whole-forward roundings
    and are held to the whole-forward bound; a sample mix-up moves the output by its full size."""
    model, _ = sdxl
    B, H, W, ts = CASES["bucket_152x104_B3"]
    x, ctx, added = make_inputs(B, H, W, seed=7)
    t = torch.tensor(ts, device="cuda")
    out = model(x, t, ctx, added_cond_kwargs=added).sample
    for b in range(B):
        one = model(x[b:b + 1], t[b:b + 1], ctx[b:b + 1],
                    added_cond_kwargs={k: v[b:b + 1] for k, v in added.items()}).sample
        check(one[0], out[b].float(), FINAL_ATOL_RMS, FINAL_L2, f"sample {b} alone vs in the batch")
    for b in range(1, B):
        assert (out[b].float() - out[0].float()).abs().max() > 0.1 * out.float().abs().max(), "samples collapsed"


# ---------------------------------------------------------------------------------------------------------------------
# Part 3: graph against eager at production geometry
# ---------------------------------------------------------------------------------------------------------------------
def test_sdxl_graphed_pipeline_matches_eager(sdxl):
    from paddlemix_b200.ppdiffusers.pipelines import StableDiffusionPipeline
    from paddlemix_b200.ppdiffusers.schedulers import EulerDiscreteScheduler
    XL = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", timestep_spacing="leading", steps_offset=1)
    model, _ = sdxl
    x, ctx, added = make_inputs(2, 128, 128, seed=21)
    neg = (0.1 * ctx).to(bf16).float()
    lat = {}
    for graph in (True, False):
        pipe = StableDiffusionPipeline(model, EulerDiscreteScheduler(**XL), use_cuda_graph=graph)
        lat[graph] = pipe(prompt_embeds=ctx, negative_prompt_embeds=neg, latents=x, num_inference_steps=2,
                          guidance_scale=5.0, added_cond_kwargs=added)
        del pipe
    assert bool(torch.isfinite(lat[False]).all())
    assert torch.equal(lat[True], lat[False]), (lat[True] - lat[False]).abs().max().item()
