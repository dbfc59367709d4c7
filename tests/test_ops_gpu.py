"""Kernel-level parity: every CUDA kernel, called through the C ABI, against a plain PyTorch fp32 evaluation of the
same operator on the same (bf16-rounded) inputs. Tolerances are stated per test."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16


@pytest.fixture(scope="module")
def ops():
    from paddlemix_b200 import ops as _ops
    _ops.init(0)
    return _ops


def rnd(*shape, seed=0, scale=1.0, dtype=bf16):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype).cuda()


def close(a, b, atol, rtol, what=""):
    a, b = a.float().cpu(), b.float().cpu()
    err = (a - b).abs()
    tol = atol + rtol * b.abs()
    bad = (err > tol).sum().item()
    assert bad == 0, f"{what}: {bad}/{a.numel()} mismatches, max err {err.max().item():.4g}, ref max {b.abs().max().item():.4g}"


# bf16 output of a K-long fp32-accumulated dot product: 2^-8 relative rounding on the output dominates.
GEMM_RTOL, GEMM_ATOL = 1.0e-2, 2e-2


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (256, 640, 320), (8, 1280, 320), (1000, 328, 200), (4096, 1920, 640),
                                   (77, 64, 2048), (300, 40, 1176)])
@pytest.mark.parametrize("bn", [0, 32, 64, 128, 160, 192, 224, 256])
@pytest.mark.parametrize("pair", [1, 0])  # 1: CTA pairs sharing the B tile through TMA multicast (default); 0: independent CTAs
def test_linear_plain(ops, M, N, K, bn, pair):
    from paddlemix_b200._lib import lib
    a, w = rnd(M, K, seed=1), rnd(N, K, seed=2, scale=K ** -0.5)
    bias = rnd(N, seed=3, dtype=torch.float32)
    lib.b200mix_debug_force_bn(bn)
    lib.b200mix_debug_gemm_pair(pair)
    try:
        out = ops.linear(a, w, bias)
    finally:
        lib.b200mix_debug_force_bn(0)
        lib.b200mix_debug_gemm_pair(1)
    ref = a.float() @ w.float().t() + bias
    close(out, ref, GEMM_ATOL, GEMM_RTOL, f"linear {M}x{N}x{K} bn={bn}")


def test_linear_persistent_many_tiles(ops):
    M, N, K = 8192, 2560, 1280  # 64 x 10+ tiles: several tiles per CTA and all ring phases
    a, w = rnd(M, K, seed=4), rnd(N, K, seed=5, scale=K ** -0.5)
    out = ops.linear(a, w)
    ref = a.float() @ w.float().t()
    close(out, ref, GEMM_ATOL, GEMM_RTOL, "big linear")


def _streamk(lib, on, max_clusters=0):
    import ctypes
    for f in (lib.b200mix_debug_streamk, lib.b200mix_debug_max_clusters):
        f.argtypes, f.restype = [ctypes.c_int], None
    lib.b200mix_debug_streamk(on)
    lib.b200mix_debug_max_clusters(max_clusters)


@pytest.mark.parametrize("M,N,K,clusters,bn", [
    (8192, 1280, 1280, 0, 0),     # SDXL out-projection: 160 tile pairs on 66 clusters -> 94 stream-K tiles + 1 round
    (8192, 1280, 5120, 0, 0),     # FF2
    (2048, 512, 1024, 3, 256),    # 16 tile pairs on 3 clusters: 4 stream-K tiles, every cluster has a tail and / or a head
    (1536, 768, 576, 5, 128),     # 36 tile pairs on 5 clusters, 9 k-blocks: 6 stream-K tiles; ragged last n-tile
    (1000, 328, 640, 3, 64),      # ragged M (phantom rows in the last pair) and ragged N
    (1280, 1024, 512, 7, 256),    # 20 on 7: 13 stream-K tiles (almost two rounds)
])
@pytest.mark.parametrize("epi", ["plain", "bias_res", "glu", "fp32"])
def test_linear_streamk(ops, M, N, K, clusters, bn, epi):
    """Stream-K head of the tile schedule (csrc/gemm.cu SegIter): tiles split between two clusters must give the same
    result as the round-robin schedule up to the fp32 summation order, for every epilogue path (coalesced, direct / GLU,
    fp32 output), and must be reproducible run to run."""
    from paddlemix_b200._lib import lib
    a, w = rnd(M, K, seed=31), rnd(N, K, seed=32, scale=K ** -0.5)
    bias = rnd(N, seed=33, dtype=torch.float32) if epi != "plain" else None
    res = rnd(M, N, seed=34) if epi == "bias_res" else None
    kw = dict(residual=res, glu=1 if epi == "glu" else 0, out_fp32=(epi == "fp32"))
    outs = {}
    try:
        for on in (1, 0):
            _streamk(lib, 2 * on, clusters)  # 2 = split shallow reductions too (the default keeps them round-robin)
            lib.b200mix_debug_force_bn(bn)
            outs[on] = ops.linear(a, w, bias, **kw)
            if on:
                again = ops.linear(a, w, bias, **kw)
    finally:
        _streamk(lib, 1, 0)
        lib.b200mix_debug_force_bn(0)
    assert torch.equal(outs[1], again), "stream-K result is not reproducible"
    z = a.float() @ w.float().t() + (bias if bias is not None else 0)
    if epi == "glu":
        ref = z[:, 0::2] * F.gelu(z[:, 1::2])
    else:
        ref = z + (res.float() if res is not None else 0)
    close(outs[1], ref, GEMM_ATOL, 1.5e-2 if epi == "glu" else GEMM_RTOL, f"stream-K {M}x{N}x{K} {epi}")
    close(outs[1], outs[0].float(), GEMM_ATOL, 1.5e-2 if epi == "glu" else GEMM_RTOL, f"stream-K vs round-robin {epi}")


@pytest.mark.parametrize("clusters", [0, 5])
def test_conv3x3_streamk(ops, clusters):
    from paddlemix_b200._lib import lib
    B, H, W, Cin, Cout = (8, 32, 32, 320, 1280) if clusters == 0 else (3, 32, 32, 128, 320)
    x = rnd(B, H, W, Cin, seed=35)
    w = rnd(Cout, 3, 3, Cin, seed=36, scale=(9 * Cin) ** -0.5)
    bias, temb, res = rnd(Cout, seed=37, dtype=torch.float32), rnd(B, Cout, seed=38, dtype=torch.float32), rnd(B, H, W, Cout, seed=39)
    try:
        _streamk(lib, 2, clusters)
        out = ops.conv3x3(x, w, bias, row_add=temb, residual=res)
    finally:
        _streamk(lib, 1, 0)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2), bias, padding=1)
    ref = (ref + temb[:, :, None, None]).permute(0, 2, 3, 1) + res.float()
    close(out, ref, GEMM_ATOL, GEMM_RTOL, f"conv3x3 stream-K clusters={clusters}")


def test_linear_streamk_many_launches_and_streams(ops):
    """Flags are lowered by the consumer: 50 back-to-back launches, then a second stream (its own workspace slot), then a
    CUDA graph captured on a third stream, all give the bits of the first launch."""
    M, N, K = 8192, 1280, 5120  # 80 k-blocks: stream-K by default
    a, w, res = rnd(M, K, seed=40), rnd(N, K, seed=41, scale=K ** -0.5), rnd(M, N, seed=42)
    first = ops.linear(a, w, residual=res)
    for _ in range(50):
        out = ops.linear(a, w, residual=res)
    assert torch.equal(out, first)
    s2 = torch.cuda.Stream()
    s2.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s2):
        out2 = ops.linear(a, w, residual=res)
    s2.synchronize()
    assert torch.equal(out2, first)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out3 = ops.linear(a, w, residual=res)
    for _ in range(3):
        out3.zero_()
        g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out3, first)


@pytest.mark.parametrize("M,C,N2,bn", [(8192, 1280, 3840, 0), (1000, 320, 640, 0), (300, 64, 96, 32), (4096, 640, 5120, 0),
                                        (2048, 1280, 1280, 160), (520, 96, 64, 64)])
@pytest.mark.parametrize("glu", [0, 1])
def test_linear_folded_layernorm(ops, M, C, N2, bn, glu):
    """BasicTransformerBlock (attention.py:352-489): h = to_out(o) + bias + residual; q = to_q(LayerNorm(h)).
    Producer epilogue statistics + consumer epilogue normalisation against F.layer_norm -> F.linear in fp32 on the same
    bf16 h. Tolerance: the usual bf16-output GEMM bound (the folded form rounds h once instead of twice)."""
    from paddlemix_b200._lib import lib
    K0 = 256
    a, w0 = rnd(M, K0, seed=60), rnd(C, K0, seed=61, scale=K0 ** -0.5)
    b0, res = rnd(C, seed=62, dtype=torch.float32), rnd(M, C, seed=63, scale=2.0)
    res = (res.float() + 1.5).to(bf16)  # a row mean well away from zero
    gamma = 1.0 + 0.3 * rnd(C, seed=64, dtype=torch.float32)
    beta = 0.2 * rnd(C, seed=65, dtype=torch.float32)
    w1 = rnd(N2, C, seed=66, dtype=torch.float32) * C ** -0.5
    b1 = rnd(N2, seed=67, dtype=torch.float32)
    lib.b200mix_debug_force_bn(bn)
    try:
        h, st = ops.linear(a, w0, b0, residual=res, stats=True)
        plain = ops.linear(a, w0, b0, residual=res)
        assert torch.equal(h, plain), "taking the statistics must not change the output"
        hf = h.float()
        tot = st.buf.double() / st.SCALE
        close(tot[:, 0], hf.double().sum(1), 2e-2, 1e-4, "row sums")
        close(tot[:, 1], (hf.double() * hf.double()).sum(1), 2e-2, 1e-4, "row sums of squares")
        h2, st2 = ops.linear(a, w0, b0, residual=res, stats=True)
        assert torch.equal(st2.buf, st.buf), "fixed-point row statistics must be reproducible bit for bit"
        mean, rstd = st.mean_rstd(1e-5)
        close(mean, hf.mean(1), 1e-4, 1e-4, "mean")
        close(rstd, torch.rsqrt(hf.var(1, unbiased=False) + 1e-5), 1e-4, 2e-3, "rstd")
        w1f, colsum, b1f = ops.fold_layernorm_into_linear(w1, gamma, beta, b1)
        out = ops.linear(h, w1f, b1f, ln=(st, colsum, 1e-5), glu=glu)
        again = ops.linear(h, w1f, b1f, ln=(st, colsum, 1e-5), glu=glu)
    finally:
        lib.b200mix_debug_force_bn(0)
    assert torch.equal(out, again)
    z = F.linear(F.layer_norm(hf, (C,), gamma, beta, 1e-5), w1, b1)
    ref = z[:, 0::2] * F.gelu(z[:, 1::2]) if glu else z
    close(out, ref, 3e-2, 1.5e-2, f"folded layernorm {M}x{C}->{N2} glu={glu}")
    # and against the two-kernel form it replaces
    n = ops.layernorm(h, gamma, beta, eps=1e-5)
    two = ops.linear(n, w1.to(bf16), b1, glu=glu)
    close(out, two.float(), 6e-2, 3e-2, "folded vs layernorm kernel + linear")


@pytest.mark.parametrize("act", [1, 2, 3, 4])
def test_linear_act(ops, act):
    M, N, K = 512, 256, 192
    a, w = rnd(M, K, seed=6), rnd(N, K, seed=7, scale=K ** -0.5)
    bias = rnd(N, seed=8, dtype=torch.float32)
    out = ops.linear(a, w, bias, act=act)
    z = a.float() @ w.float().t() + bias
    ref = {1: F.silu(z), 2: F.gelu(z), 3: F.gelu(z, approximate="tanh"), 4: z * torch.sigmoid(1.702 * z)}[act]
    close(out, ref, GEMM_ATOL, GEMM_RTOL, f"act {act}")


@pytest.mark.parametrize("glu", [1, 2])
def test_linear_glu(ops, glu):
    M, N2, K = 640, 384, 320
    a = rnd(M, K, seed=9)
    wv, wg = rnd(N2, K, seed=10, scale=K ** -0.5), rnd(N2, K, seed=11, scale=K ** -0.5)
    bv, bg = rnd(N2, seed=12, dtype=torch.float32), rnd(N2, seed=13, dtype=torch.float32)
    w = torch.stack([wv, wg], dim=1).reshape(2 * N2, K).contiguous()  # interleave rows: 2j = value, 2j+1 = gate
    b = torch.stack([bv, bg], dim=1).reshape(2 * N2).contiguous()
    out = ops.linear(a, w, b, glu=glu)
    val = a.float() @ wv.float().t() + bv
    gate = a.float() @ wg.float().t() + bg
    ref = val * (F.gelu(gate) if glu == 1 else F.silu(gate))
    assert out.shape == (M, N2)
    close(out, ref, GEMM_ATOL, 1.5e-2, f"glu {glu}")


def test_linear_gate_residual_rowadd_fp32(ops):
    B, S, N, K = 3, 200, 256, 128
    a, w = rnd(B * S, K, seed=14), rnd(N, K, seed=15, scale=K ** -0.5)
    bias = rnd(N, seed=16, dtype=torch.float32)
    gate, radd = rnd(B, N, seed=17, dtype=torch.float32), rnd(B, N, seed=18, dtype=torch.float32)
    res = rnd(B * S, N, seed=19)
    out = ops.linear(a, w, bias, residual=res, row_gate=gate, row_add=radd, rows_per_group=S, out_fp32=True)
    z = a.float() @ w.float().t() + bias + radd.repeat_interleave(S, 0)
    ref = z * gate.repeat_interleave(S, 0) + res.float()
    assert out.dtype == torch.float32
    close(out, ref, 1e-3, 1e-3, "gate/residual/rowadd fp32")


@pytest.mark.parametrize("B,H,W,Cin,Cout,stride", [(2, 16, 16, 64, 64, 1), (1, 8, 8, 128, 320, 1), (3, 32, 32, 320, 640, 1),
                                                   (2, 64, 64, 64, 128, 1), (2, 16, 16, 64, 64, 2), (3, 32, 32, 320, 320, 2),
                                                   (1, 128, 128, 64, 32, 1), (2, 32, 32, 320, 4, 1)])
def test_conv3x3(ops, B, H, W, Cin, Cout, stride):
    x = rnd(B, H, W, Cin, seed=20)
    w = rnd(Cout, 3, 3, Cin, seed=21, scale=(9 * Cin) ** -0.5)
    bias = rnd(Cout, seed=22, dtype=torch.float32)
    temb = rnd(B, Cout, seed=23, dtype=torch.float32)
    out = ops.conv3x3(x, w, bias, stride=stride, row_add=temb)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2), bias, stride=stride, padding=1)
    ref = (ref + temb[:, :, None, None]).permute(0, 2, 3, 1)
    assert out.shape == ref.shape
    close(out, ref, GEMM_ATOL, GEMM_RTOL, f"conv3x3 {B}x{H}x{W} {Cin}->{Cout} s{stride}")


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 16, 16, 64, 64), (1, 8, 8, 128, 320), (3, 32, 32, 320, 640),
                                            (1, 4, 4, 64, 32), (5, 8, 16, 64, 96), (2, 64, 64, 128, 128)])
@pytest.mark.parametrize("epi", ["bias", "full"])
def test_conv3x3_up2x(ops, B, H, W, Cin, Cout, epi):
    """Upsample2D (resnet.py:169-218): F.interpolate(scale_factor=2, mode='nearest') + conv3x3, fused as per-parity 2x2
    convs over the low-resolution input. Odd tile counts per parity (phantom tile), ragged N and every border are covered."""
    x = rnd(B, H, W, Cin, seed=50)
    w = rnd(Cout, 3, 3, Cin, seed=51, scale=(9 * Cin) ** -0.5)
    bias = rnd(Cout, seed=52, dtype=torch.float32)
    w4 = ops.fold_upsample_conv_weight(w)
    assert w4.shape == (Cout, 16, Cin)
    kw = {}
    if epi == "full":
        kw = dict(row_add=rnd(B, Cout, seed=53, dtype=torch.float32), residual=rnd(B, 2 * H, 2 * W, Cout, seed=54), out_scale=0.5)
    out = ops.conv3x3_up2x(x, w4, bias, **kw)
    up = F.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=2.0, mode="nearest")
    ref = F.conv2d(up, w.float().permute(0, 3, 1, 2), bias, padding=1)
    if epi == "full":
        ref = (ref + kw["row_add"][:, :, None, None] + kw["residual"].float().permute(0, 3, 1, 2)) * 0.5
    ref = ref.permute(0, 2, 3, 1)
    assert out.shape == ref.shape
    close(out, ref, GEMM_ATOL, GEMM_RTOL, f"conv3x3_up2x {B}x{H}x{W} {Cin}->{Cout} {epi}")
    # the unfused pair of launches it replaces
    two = ops.conv3x3(ops.upsample_nearest2x(x), w, bias, **kw)
    close(out, two.float(), GEMM_ATOL, GEMM_RTOL, "fused vs upsample + conv")


def test_conv3x3_residual(ops):
    B, H, W, C = 2, 32, 32, 128
    x, w = rnd(B, H, W, C, seed=24), rnd(C, 3, 3, C, seed=25, scale=(9 * C) ** -0.5)
    res = rnd(B, H, W, C, seed=26)
    out = ops.conv3x3(x, w, None, residual=res, out_scale=0.5)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2), None, padding=1).permute(0, 2, 3, 1)
    close(out, (ref + res.float()) * 0.5, GEMM_ATOL, GEMM_RTOL, "conv residual")


@pytest.mark.parametrize("B,H,W,Cin,Cout,fp32_in", [(2, 32, 32, 4, 320, True), (3, 17, 23, 4, 64, False),
                                                    (1, 8, 8, 8, 32, True), (2, 9, 5, 3, 16, False), (1, 64, 64, 4, 1152, True)])
def test_conv_small_cin(ops, B, H, W, Cin, Cout, fp32_in):
    # Cin == 4 (16-byte aligned input) takes the pixel-per-thread kernel, everything else the generic one
    x = rnd(B, H, W, Cin, seed=27, dtype=torch.float32)
    if not fp32_in:
        x = x.to(bf16)
    w, bias = rnd(Cout, 3, 3, Cin, seed=28, scale=0.2), rnd(Cout, seed=29, dtype=torch.float32)
    out = ops.conv3x3_small_cin(x, w, bias)
    xr = x.to(bf16).float()
    ref = F.conv2d(xr.permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2), bias, padding=1).permute(0, 2, 3, 1)
    close(out, ref, 1e-2, 1e-2, f"conv_in {B}x{H}x{W} {Cin}->{Cout}")
    out_nb = ops.conv3x3_small_cin(x, w, None)
    close(out_nb, ref - bias, 1e-2, 1e-2, "conv_in without bias")


def ref_sdpa(q, k, v, scale, causal=False, cu=None):
    # q [B,Sq,Hq,D], k/v [B,Sk,Hkv,D] -> [B,Sq,Hq,D]; fp32 math softmax(q k^T * scale + mask) v
    B, Sq, Hq, D = q.shape
    Sk, Hkv = k.shape[1], k.shape[2]
    qf, kf, vf = q.float().permute(0, 2, 1, 3), k.float().permute(0, 2, 1, 3), v.float().permute(0, 2, 1, 3)
    kf, vf = kf.repeat_interleave(Hq // Hkv, 1), vf.repeat_interleave(Hq // Hkv, 1)
    s = qf @ kf.transpose(-1, -2) * scale
    mask = torch.zeros(Sq, Sk, device=q.device)
    if causal:
        i = torch.arange(Sq, device=q.device)[:, None] + (Sk - Sq)
        mask = mask.masked_fill(torch.arange(Sk, device=q.device)[None, :] > i, float("-inf"))
    if cu is not None:
        seg = torch.zeros(Sq, dtype=torch.long, device=q.device)
        for i in range(len(cu) - 1):
            seg[cu[i]:cu[i + 1]] = i
        mask = mask.masked_fill(seg[:, None] != seg[None, :], float("-inf"))
    p = torch.softmax(s + mask, -1)
    return (p @ vf).permute(0, 2, 1, 3)


# P is rounded to bf16 before the PV product and the output is bf16: 2^-8 relative on O(1) values.
ATT_ATOL, ATT_RTOL = 1.5e-2, 2e-2


@pytest.mark.parametrize("B,Sq,Sk,Hq,Hkv,D,causal", [
    (2, 128, 128, 2, 2, 64, False), (1, 256, 384, 3, 3, 64, False), (2, 1024, 1024, 4, 4, 64, False),
    (2, 200, 77, 5, 5, 64, False), (1, 4250, 4250, 2, 2, 64, False), (2, 128, 128, 2, 2, 128, False),
    (1, 768, 768, 4, 2, 128, True), (2, 300, 300, 2, 1, 128, True), (1, 64, 64, 8, 8, 64, False),
    (2, 256, 256, 8, 8, 192, False), (1, 64, 77, 2, 2, 192, False), (1, 400, 400, 2, 2, 192, True),
])
def test_sdpa(ops, B, Sq, Sk, Hq, Hkv, D, causal):
    q, k, v = rnd(B, Sq, Hq, D, seed=30), rnd(B, Sk, Hkv, D, seed=31), rnd(B, Sk, Hkv, D, seed=32)
    scale = D ** -0.5
    out = ops.sdpa(q, k, v, scale=scale, causal=causal)
    ref = ref_sdpa(q, k, v, scale, causal)
    close(out, ref, ATT_ATOL, ATT_RTOL, f"sdpa B{B} Sq{Sq} Sk{Sk} H{Hq}/{Hkv} D{D} causal={causal}")


@pytest.mark.parametrize("B,Sq,Sk,Hq,Hkv", [(8, 1024, 77, 20, 20), (2, 4096, 77, 10, 10), (3, 1000, 1, 2, 2),
                                            (1, 130, 17, 3, 3), (5, 384, 96, 6, 2), (2, 256, 128, 4, 4),
                                            (1, 128, 33, 1, 1), (37, 200, 64, 9, 3)])
def test_sdpa_short_kv_persistent(ops, B, Sq, Sk, Hq, Hkv):
    """Sk <= 128, D = 64, non-causal (cross-attention against a short context): the default 128-key blocks (one block
    covers every key) must agree with the 64-key-block configuration and with the fp32 reference."""
    from paddlemix_b200._lib import lib
    D = 64
    q, k, v = rnd(B, Sq, Hq, D, seed=90), rnd(B, Sk, Hkv, D, seed=91), rnd(B, Sk, Hkv, D, seed=92)
    lens = torch.tensor([max(1, Sk - 3 * b) for b in range(B)], dtype=torch.int32, device="cuda")
    for kv_lens in (None, lens):
        out = ops.sdpa(q, k, v, kv_lens=kv_lens)
        lib.b200mix_debug_attn_bn64(1)
        try:
            gen = ops.sdpa(q, k, v, kv_lens=kv_lens)
        finally:
            lib.b200mix_debug_attn_bn64(0)
        close(out, gen.float(), ATT_ATOL, ATT_RTOL, f"short-kv 128- vs 64-key blocks B{B} Sq{Sq} Sk{Sk}")
        for b in ([0, B - 1] if kv_lens is not None else [0]):
            n = int(lens[b]) if kv_lens is not None else Sk
            ref = ref_sdpa(q[b:b + 1], k[b:b + 1, :n], v[b:b + 1, :n], D ** -0.5)
            close(out[b:b + 1], ref, ATT_ATOL, ATT_RTOL, f"short-kv B{B} Sq{Sq} Sk{Sk} H{Hq}/{Hkv} b{b} n{n}")


@pytest.mark.parametrize("B,Sq,Sk,H,causal", [(2, 1024, 1024, 4, False), (1, 300, 450, 3, False), (1, 333, 333, 2, True)])
def test_sdpa_d64_64_key_blocks(ops, B, Sq, Sk, H, causal):
    """The D = 64 kernel with 64-key blocks (not the default, kept for A/B runs) against the fp32 reference."""
    from paddlemix_b200._lib import lib
    q, k, v = rnd(B, Sq, H, 64, seed=93), rnd(B, Sk, H, 64, seed=94), rnd(B, Sk, H, 64, seed=95)
    lib.b200mix_debug_attn_bn64(1)
    try:
        out = ops.sdpa(q, k, v, causal=causal)
    finally:
        lib.b200mix_debug_attn_bn64(0)
    close(out, ref_sdpa(q, k, v, 64 ** -0.5, causal), ATT_ATOL, ATT_RTOL, f"sdpa bn64 B{B} Sq{Sq} Sk{Sk} causal={causal}")


@pytest.mark.parametrize("B,Sq,Sk,H,causal,scale", [(2, 1024, 1024, 4, False, 1.0), (1, 300, 450, 3, False, 1.0),
                                                      (1, 333, 333, 2, True, 1.0), (1, 512, 512, 2, False, 4.0)])
def test_sdpa_d64_64_key_blocks_lazy_rescale(ops, B, Sq, Sk, H, causal, scale):
    """The D = 64 kernel with 64-key blocks against the fp32 reference, incl. masked tiles and the lazy-rescale path
    (large logits: the running max grows by more than 2^8 between blocks)."""
    from paddlemix_b200._lib import lib
    q, k, v = rnd(B, Sq, H, 64, seed=96, scale=scale), rnd(B, Sk, H, 64, seed=97, scale=scale), rnd(B, Sk, H, 64, seed=98)
    lib.b200mix_debug_attn_bn64(1)
    try:
        out = ops.sdpa(q, k, v, causal=causal)
    finally:
        lib.b200mix_debug_attn_bn64(0)
    close(out, ref_sdpa(q, k, v, 64 ** -0.5, causal), ATT_ATOL, ATT_RTOL, f"sdpa 64-key blocks B{B} Sq{Sq} Sk{Sk} causal={causal}")


def test_sdpa_large_logits(ops):
    # large |q.k| exercises the lazy-rescale path (running max grows by more than 2^8 between tiles)
    B, S, H, D = 1, 512, 2, 64
    q, k, v = rnd(B, S, H, D, seed=33, scale=4.0), rnd(B, S, H, D, seed=34, scale=4.0), rnd(B, S, H, D, seed=35)
    out = ops.sdpa(q, k, v, scale=D ** -0.5)
    close(out, ref_sdpa(q, k, v, D ** -0.5), ATT_ATOL, ATT_RTOL, "sdpa large logits")


def test_sdpa_fused_qkv_strides(ops):
    # q/k/v as strided views into one fused projection buffer [B, S, 3*H*D] (how the UNet calls it)
    B, S, H, D = 2, 256, 5, 64
    qkv = rnd(B, S, 3 * H * D, seed=36)
    q, k, v = (qkv[:, :, i * H * D:(i + 1) * H * D].unflatten(-1, (H, D)) for i in range(3))
    out = ops.sdpa(q, k, v)
    close(out, ref_sdpa(q, k, v, D ** -0.5), ATT_ATOL, ATT_RTOL, "sdpa strided")


def test_sdpa_varlen(ops):
    H, D = 4, 128
    lens = [1024, 200, 77, 384]
    cu = [0]
    for n in lens:
        cu.append(cu[-1] + n)
    T = cu[-1]
    q, k, v = rnd(1, T, H, D, seed=37), rnd(1, T, H, D, seed=38), rnd(1, T, H, D, seed=39)
    cu_t = torch.tensor(cu, dtype=torch.int32, device="cuda")
    out = ops.sdpa(q, k, v, cu_seqlens=cu_t)
    ref = ref_sdpa(q, k, v, D ** -0.5, cu=cu)
    close(out, ref, ATT_ATOL, ATT_RTOL, "sdpa varlen")


@pytest.mark.parametrize("B,HW,C1,C2,silu", [(2, 64, 320, 0, True), (3, 1024, 640, 0, False), (2, 256, 1280, 640, True),
                                             (1, 4096, 320, 320, True), (2, 100, 32, 0, True), (2, 64, 1280, 1280, True)])
def test_groupnorm(ops, B, HW, C1, C2, silu):
    x1 = rnd(B, HW, C1, seed=40) * 2 + 0.5
    x2 = None if C2 == 0 else rnd(B, HW, C2, seed=41)
    C = C1 + C2
    gamma, beta = rnd(C, seed=42, dtype=torch.float32), rnd(C, seed=43, dtype=torch.float32)
    x1 = x1.to(bf16)
    out = ops.groupnorm_nhwc(x1, gamma, beta, x2=x2, groups=32, eps=1e-5, silu=silu)
    xc = x1 if x2 is None else torch.cat([x1, x2], -1)
    ref = F.group_norm(xc.float().permute(0, 2, 1), 32, gamma, beta, 1e-5).permute(0, 2, 1)
    if silu:
        ref = F.silu(ref)
    close(out, ref, 2e-2, 1e-2, f"groupnorm {B}x{HW}x{C1}+{C2}")


@pytest.mark.parametrize("M,N", [(77, 320), (4096, 640), (1000, 1280), (616, 1536), (33, 3584), (5, 8192), (64, 64)])
def test_layernorm_affine(ops, M, N):
    x = rnd(M, N, seed=44) + 0.3
    x = x.to(bf16)
    w, b = rnd(N, seed=45, dtype=torch.float32), rnd(N, seed=46, dtype=torch.float32)
    out = ops.layernorm(x, w, b, eps=1e-5)
    close(out, F.layer_norm(x.float(), (N,), w, b, 1e-5), 2e-2, 1e-2, f"layernorm {M}x{N}")


def test_layernorm_adaln_fused(ops):
    # the reference Triton op fused_adaLN_scale_residual (triton_ops.py:790-798): resi = x + gate*mha; y = LN(resi)*(1+scale)+shift
    B, S, N = 3, 154, 1536
    x, mha = rnd(B, S, N, seed=47), rnd(B, S, N, seed=48)
    gate, scale, shift = (rnd(B, N, seed=s, dtype=torch.float32) for s in (49, 50, 51))
    resid, y = ops.layernorm(x, None, None, eps=1e-6, delta=mha, gate=gate, scale=scale, shift=shift, rows_per_group=S,
                             want_resid=True)
    r_ref = x.float() + gate[:, None] * mha.float()
    close(resid, r_ref, 2e-2, 1e-2, "adaln resid")
    r_b = r_ref.to(bf16).float()
    y_ref = F.layer_norm(r_b, (N,), None, None, 1e-6) * (1 + scale[:, None]) + shift[:, None]
    close(y, y_ref, 3e-2, 1.5e-2, "adaln y")


@pytest.mark.parametrize("M,N,mode", [(8192, 1280, "affine"), (4099, 640, "affine"), (3 * 1367, 1536, "adaln"),
                                      (2 * 2048, 1152, "adaln_noresid"), (3000, 3584, "rms"), (20001, 128, "affine")])
def test_layernorm_block_kernel_matches_register_kernel(ops, M, N, mode):
    """Inputs >= 4 MB take the shared-memory block kernel (bulk-copy row blocks); it must agree BIT FOR BIT with the
    register-resident kernel (same accumulation order) and with the fp32 torch reference within bf16 tolerance."""
    from paddlemix_b200._lib import lib
    x = (rnd(M, N, seed=61) + 0.25).to(bf16)
    kw = dict(eps=1e-6)
    args = (None, None)
    if mode == "affine":
        args = (rnd(N, seed=62, dtype=torch.float32), rnd(N, seed=63, dtype=torch.float32))
    elif mode == "rms":
        args = (rnd(N, seed=62, dtype=torch.float32), None)
        kw["rms"] = True
    else:
        G = 3 if mode == "adaln" else 2
        S = M // G
        kw.update(delta=rnd(M, N, seed=64), gate=rnd(G, N, seed=65, dtype=torch.float32),
                  scale=rnd(G, N, seed=66, dtype=torch.float32), shift=rnd(G, N, seed=67, dtype=torch.float32),
                  rows_per_group=S, want_resid=(mode == "adaln"))

    def run():
        o = ops.layernorm(x, *args, **kw)
        return o if isinstance(o, tuple) else (o,)

    blk = run()
    lib.b200mix_debug_ln_register_only(1)
    try:
        reg = run()
    finally:
        lib.b200mix_debug_ln_register_only(0)
    for a, b in zip(blk, reg):
        assert torch.equal(a, b), f"block vs register layernorm differ ({mode} {M}x{N})"
    xf = x.float()
    if mode == "affine":
        close(blk[0], F.layer_norm(xf, (N,), args[0], args[1], 1e-6), 2e-2, 1e-2, "block layernorm")
    elif mode == "rms":
        ref = (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-6)).to(bf16).float() * args[0]
        close(blk[0], ref, 2e-2, 1e-2, "block rmsnorm")
    else:
        G, S = kw["gate"].shape[0], kw["rows_per_group"]
        r = (xf.view(G, S, N) + kw["gate"][:, None] * kw["delta"].float().view(G, S, N)).to(bf16).float()
        y_ref = F.layer_norm(r, (N,), None, None, 1e-6) * (1 + kw["scale"][:, None]) + kw["shift"][:, None]
        close(blk[-1].view(G, S, N), y_ref, 3e-2, 1.5e-2, "block adaln y")
        if mode == "adaln":
            close(blk[0].view(G, S, N), r, 2e-2, 1e-2, "block adaln resid")


def test_rmsnorm(ops):
    M, N = 300, 3584
    x, w = rnd(M, N, seed=52), rnd(N, seed=53, dtype=torch.float32)
    out = ops.layernorm(x, w, None, eps=1e-6, rms=True)
    xf = x.float()
    ref = (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-6)).to(bf16).float() * w
    close(out, ref, 2e-2, 1e-2, "rmsnorm")


def test_timestep_embedding(ops):
    t = torch.tensor([981.0, 1.0, 481.0, 0.0], device="cuda")
    for dim, flip, shift in [(320, True, 0.0), (256, True, 0.0), (256, False, 1.0)]:
        out = ops.timestep_embedding(t, dim, flip_sin_to_cos=flip, downscale_freq_shift=shift, out_dtype=torch.float32)
        half = dim // 2
        exponent = -math.log(10000) * torch.arange(half, dtype=torch.float32, device="cuda") / (half - shift)
        emb = t[:, None] * torch.exp(exponent)[None]
        ref = torch.cat([torch.sin(emb), torch.cos(emb)], -1)
        if flip:
            ref = torch.cat([ref[:, half:], ref[:, :half]], -1)
        close(out, ref, 2e-4, 0, f"timestep embedding {dim}")


def test_elementwise_misc(ops):
    x = rnd(2, 8, 8, 64, seed=54)
    up = ops.upsample_nearest2x(x)
    ref = F.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=2.0, mode="nearest").permute(0, 2, 3, 1)
    assert torch.equal(up.float(), ref)
    y = rnd(2, 8, 8, 32, seed=55)
    assert torch.equal(ops.concat_channels(x, y), torch.cat([x, y], -1))
    lat = rnd(2, 4, 16, 16, seed=56, dtype=torch.float32)
    nhwc = ops.nchw_to_nhwc(lat)
    assert torch.equal(nhwc, lat.permute(0, 2, 3, 1).to(bf16))
    back = ops.nhwc_to_nchw(nhwc)
    assert torch.equal(back, lat.to(bf16).float())
    for act, fn in [(1, F.silu), (2, F.gelu)]:
        a = rnd(1000, seed=57, dtype=torch.float32)
        close(ops.activation(a, act), fn(a), 1e-5, 1e-5, "activation")
    assert torch.equal(ops.cast(lat, bf16), lat.to(bf16))


def test_ddim_step_bit_exact(ops):
    # fp32 inputs, same expression order as scheduling_ddim.py:420-457 -> bit-identical to the CPU evaluation
    g = torch.Generator().manual_seed(58)
    x, eu, ec = (torch.randn(2, 4, 32, 32, generator=g) for _ in range(3))
    sa_t, sb_t, sa_p, sb_p = (torch.tensor(v, dtype=torch.float32) for v in (0.0413, 0.99915, 0.2213, 0.9752))
    gs = 5.0
    eps = eu + gs * (ec - eu)
    x0 = (x - sb_t * eps) / sa_t
    ref = sa_p * x0 + sb_p * eps
    out = ops.ddim_step(eu.cuda(), ec.cuda(), gs, x.cuda(), sa_t.item(), sb_t.item(), sa_p.item(), sb_p.item())
    assert torch.equal(out.cpu(), ref)
    ref2 = sa_p * ((x - sb_t * eu) / sa_t) + sb_p * eu
    out2 = ops.ddim_step(eu.cuda(), None, 0.0, x.cuda(), sa_t.item(), sb_t.item(), sa_p.item(), sb_p.item())
    assert torch.equal(out2.cpu(), ref2)
    sigma, sigma_next = torch.tensor(0.8731, dtype=torch.float32), torch.tensor(0.8360, dtype=torch.float32)
    dt = sigma_next - sigma
    out3 = ops.euler_step(eu.cuda(), None, 0.0, x.cuda(), sigma.item(), dt.item())
    den = x - eu * sigma
    assert torch.equal(out3.cpu(), x + (x - den) / sigma * dt)


def test_rope(ops):
    T, H, D = 50, 4, 80
    x = rnd(T, H, 128, seed=59)
    ang = torch.rand(T, D // 2, generator=torch.Generator().manual_seed(60)).cuda() * 6
    cos, sin = torch.cat([ang.cos(), ang.cos()], -1).contiguous(), torch.cat([ang.sin(), ang.sin()], -1).contiguous()
    xr = x.clone()
    ops.rope_inplace(xr, cos, sin, rot_dim=D)
    xf = x.float()[..., :D]
    rot = torch.cat([-xf[..., D // 2:], xf[..., :D // 2]], -1)
    ref = xf * cos[:, None] + rot * sin[:, None]
    close(xr[..., :D], ref, 2e-2, 1e-2, "rope")
    assert torch.equal(xr[..., D:], x[..., D:])


def test_linear_batched_strided(ops):
    # image / text token ranges of a joint [B, n+L, *] buffer, produced and consumed in place
    B, n, L, K, N = 3, 300, 154, 192, 256
    S = n + L
    xi, xt = rnd(B, n, K, seed=61), rnd(B, L, K, seed=62)
    w, bias = rnd(N, K, seed=63, scale=K ** -0.5), rnd(N, seed=64, dtype=torch.float32)
    joint = torch.zeros(B, S, N, device="cuda", dtype=bf16)
    ops.linear_batched(xi, w, bias, out=joint[:, :n])
    ops.linear_batched(xt, w, bias, out=joint[:, n:])
    ref = torch.cat([xi.float() @ w.float().t() + bias, xt.float() @ w.float().t() + bias], 1)
    close(joint, ref, GEMM_ATOL, GEMM_RTOL, "batched write")
    gate, res = rnd(B, K, seed=65, dtype=torch.float32), rnd(B, L, K, seed=66)
    w2 = rnd(K, N, seed=67, scale=N ** -0.5)
    out = torch.empty(B, L, K, device="cuda", dtype=bf16)
    ops.linear_batched(joint[:, n:], w2, None, out=out, row_gate=gate, residual=res)
    ref2 = (joint[:, n:].float() @ w2.float().t()) * gate[:, None] + res.float()
    close(out, ref2, GEMM_ATOL, GEMM_RTOL, "batched read + gate + residual")


def test_patchify_roundtrip_and_posembed(ops):
    B, C, H, W, p, D = 2, 16, 32, 32, 2, 128
    x = rnd(B, C, H, W, seed=68, dtype=torch.float32)
    rows = ops.patchify(x, p)
    ref = torch.nn.functional.unfold(x.to(bf16).float(), p, stride=p).transpose(1, 2)  # [B, n, C*p*p] in (c, ph, pw) order
    assert torch.equal(rows.float(), ref)
    w, bias, pos = rnd(D, C * p * p, seed=69, scale=0.1), rnd(D, seed=70, dtype=torch.float32), rnd(256, D, seed=71)
    y = ops.linear(rows, w, bias, residual=pos, residual_row_mod=256)
    close(y, ref @ w.float().t() + bias + pos.float()[None], GEMM_ATOL, GEMM_RTOL, "patch embed + pos")
    t = rnd(B, 256, p * p * C, seed=72)
    img = ops.unpatchify(t, C, H // p, W // p, p, out_dtype=torch.float32)
    ref_img = t.float().reshape(B, H // p, W // p, p, p, C).permute(0, 5, 1, 3, 2, 4).reshape(B, C, H, W)
    assert torch.equal(img, ref_img)


def test_sdpa_kv_lens(ops):
    B, Sq, Sk, H, D = 3, 256, 120, 2, 128
    q, k, v = rnd(B, Sq, H, D, seed=73), rnd(B, Sk, H, D, seed=74), rnd(B, Sk, H, D, seed=75)
    lens = [120, 77, 9]
    out = ops.sdpa(q, k, v, kv_lens=torch.tensor(lens, dtype=torch.int32, device="cuda"))
    for b, n in enumerate(lens):
        ref = ref_sdpa(q[b:b + 1], k[b:b + 1, :n], v[b:b + 1, :n], D ** -0.5)
        close(out[b:b + 1], ref, ATT_ATOL, ATT_RTOL, f"kv_lens b{b}")


def test_small_attention_rope_qknorm(ops):
    B, T, S, H, d = 2, 16, 24, 3, 72
    qkv = rnd(B * T * S, 3 * H * d, seed=76)
    qw, kw = 1 + 0.1 * rnd(d, seed=77, dtype=torch.float32), 1 + 0.1 * rnd(d, seed=78, dtype=torch.float32)
    freqs = 1.0 / 10000 ** (torch.arange(0, d, 2).float() / d)
    ang = torch.outer(torch.arange(T).float(), freqs).cuda()  # [T, d/2]
    out = ops.small_attention(qkv, B, T, S, H, d, scale=d ** -0.5, rope_cos=ang.cos().contiguous(), rope_sin=ang.sin().contiguous(),
                              q_norm_w=qw, k_norm_w=kw)
    x = qkv.float().reshape(B, T, S, 3, H, d).permute(3, 0, 2, 4, 1, 5)  # [3, B, S, H, T, d]
    q, k, v = x[0], x[1], x[2]

    def rope(t):
        t2 = t.reshape(*t.shape[:-1], -1, 2)
        rot = torch.stack((-t2[..., 1], t2[..., 0]), -1).flatten(-2)
        f = ang.repeat_interleave(2, -1)
        return t * f.cos() + rot * f.sin()

    def rms(t, w):
        return w * (t * torch.rsqrt(t.pow(2).mean(-1, keepdim=True) + 1e-6))
    q, k = rms(rope(q), qw), rms(rope(k), kw)
    a = torch.softmax(q @ k.transpose(-1, -2) * d ** -0.5, -1) @ v  # [B, S, H, T, d]
    ref = a.permute(0, 3, 1, 2, 4).reshape(B * T * S, H * d)
    close(out, ref, 2e-2, 2e-2, "small attention")


def test_stdit_helpers(ops):
    x, table = rnd(3, 40, seed=79, dtype=torch.float32), rnd(5, 40, seed=80, dtype=torch.float32)
    assert torch.equal(ops.broadcast_add(x, table), x[:, None] + table[None])
    h = rnd(50, 4, 128, seed=81)
    w = 1 + 0.1 * rnd(72, seed=82, dtype=torch.float32)
    ref = h.float().clone()
    r = ref[..., :72]
    ref[..., :72] = (r * torch.rsqrt(r.pow(2).mean(-1, keepdim=True) + 1e-6)).to(bf16).float() * w
    got = ops.head_rmsnorm_inplace(h.clone(), w, 72)
    close(got, ref, 2e-2, 1e-2, "head rmsnorm")
    vid = rnd(2, 4, 3, 8, 8, seed=83, dtype=torch.float32)
    rows = ops.patchify3d(vid, 2)
    ref_rows = torch.nn.functional.unfold(vid.to(bf16).float().permute(0, 2, 1, 3, 4).reshape(6, 4, 8, 8), 2, stride=2).transpose(1, 2).reshape(2, 3 * 16, 16)
    assert torch.equal(rows.float(), ref_rows)
    t = rnd(2, 3 * 16, 2 * 2 * 8, seed=84)
    vol = ops.unpatchify3d(t, 8, 3, 4, 4, 2)
    ref_vol = t.float().reshape(2, 3, 4, 4, 2, 2, 8).permute(0, 6, 1, 2, 4, 3, 5).reshape(2, 8, 3, 8, 8)
    assert torch.equal(vol, ref_vol)


def test_llama_decoder_layer_from_ops(ops):
    """LLaVA's language backbone (PaddleNLP LlamaDecoderLayer: RMSNorm -> q/k/v without bias -> 1-D RoPE -> causal
    attention -> o_proj -> RMSNorm -> SwiGLU MLP; PaddleNLP/paddlenlp/transformers/llama/modeling.py:386-420,534-555,
    618-…) is the same block shape as Qwen2-VL's decoder minus bias / M-RoPE / GQA: composed here from the same
    kernels and checked against a plain fp32 evaluation."""
    from paddlemix_b200._lib import GLU_SWIGLU
    B, S, H, hd, I = 2, 200, 4, 128, 1024
    D = H * hd
    x = rnd(B * S, D, seed=90)
    wq, wk, wv, wo = (rnd(D, D, seed=91 + i, scale=D ** -0.5) for i in range(4))
    wg, wu, wd = rnd(I, D, seed=95, scale=D ** -0.5), rnd(I, D, seed=96, scale=D ** -0.5), rnd(D, I, seed=97, scale=I ** -0.5)
    n1, n2 = 1 + 0.1 * rnd(D, seed=98, dtype=torch.float32), 1 + 0.1 * rnd(D, seed=99, dtype=torch.float32)
    inv = 1.0 / 10000 ** (torch.arange(0, hd, 2).float() / hd)
    ang = torch.outer(torch.arange(S).float(), inv)
    cos = torch.cat([ang.cos(), ang.cos()], -1).repeat(B, 1).contiguous().cuda()
    sin = torch.cat([ang.sin(), ang.sin()], -1).repeat(B, 1).contiguous().cuda()
    # --- kernels ---
    h1 = ops.layernorm(x, n1, None, eps=1e-6, rms=True)
    qkv = ops.linear(h1, torch.cat([wq, wk, wv], 0).contiguous())
    q, k, v = (qkv[:, i * D:(i + 1) * D].unflatten(-1, (H, hd)) for i in range(3))
    ops.rope_inplace(q, cos, sin), ops.rope_inplace(k, cos, sin)
    a = ops.sdpa(q.unflatten(0, (B, S)), k.unflatten(0, (B, S)), v.unflatten(0, (B, S)), causal=True)
    y = ops.linear(a.reshape(B * S, D), wo, residual=x)
    h2 = ops.layernorm(y, n2, None, eps=1e-6, rms=True)
    gu = torch.stack([wu, wg], 1).reshape(2 * I, D).contiguous()
    out = ops.linear(ops.linear(h2, gu, glu=GLU_SWIGLU), wd, residual=y)
    # --- fp32 reference ---
    xf = x.float()

    def rms(t, w):
        return t * torch.rsqrt(t.pow(2).mean(-1, keepdim=True) + 1e-6) * w

    def rope(t):  # [B*S, H, hd]
        rot = torch.cat([-t[..., hd // 2:], t[..., :hd // 2]], -1)
        return t * cos[:, None] + rot * sin[:, None]
    r1 = rms(xf, n1)
    qf, kf, vf = (r1 @ w.float().t() for w in (wq, wk, wv))
    qf, kf = rope(qf.unflatten(-1, (H, hd))), rope(kf.unflatten(-1, (H, hd)))
    sp = lambda t: t.reshape(B, S, H, hd).transpose(1, 2)
    att = torch.nn.functional.scaled_dot_product_attention(sp(qf), sp(kf), sp(vf.unflatten(-1, (H, hd))), is_causal=True)
    yf = xf + att.transpose(1, 2).reshape(B * S, D) @ wo.float().t()
    r2 = rms(yf, n2)
    ref = yf + (torch.nn.functional.silu(r2 @ wg.float().t()) * (r2 @ wu.float().t())) @ wd.float().t()
    close(out, ref, 6e-2, 3e-2, "llama decoder layer")


@pytest.mark.parametrize("M", [1, 2, 3, 4, 5, 8])
@pytest.mark.parametrize("N,K", [(37, 64), (4608, 3584), (10, 18944), (1280, 2816)])
@pytest.mark.parametrize("epi", ["plain", "bias+silu", "bias+res", "f32", "swiglu", "geglu"])
def test_linear_skinny_m(ops, M, N, K, epi):
    """M <= 8 rows take the weight-streaming kernel (decode steps, embedding MLPs); it must agree with the fp32
    reference and with the tensor-core kernel on every epilogue it accepts."""
    from paddlemix_b200._lib import lib
    lib.b200mix_debug_skinny.argtypes, lib.b200mix_debug_skinny.restype = [__import__("ctypes").c_int], None
    if epi in ("swiglu", "geglu") and N % 2:
        N += 1
    a, w = rnd(M, K, seed=110), rnd(N, K, seed=111, scale=K ** -0.5)
    bias = rnd(N, seed=112, dtype=torch.float32)
    acc = a.float() @ w.float().t()
    kw = {}
    if epi == "plain":
        ref, b = acc, None
    elif epi == "bias+silu":
        ref, b, kw = F.silu(acc + bias), bias, dict(act=1)
    elif epi == "bias+res":
        res = rnd(M, N, seed=113)
        ref, b, kw = acc + bias + res.float(), bias, dict(residual=res)
    elif epi == "f32":
        ref, b, kw = acc + bias, bias, dict(out_fp32=True)
    else:
        z = acc + bias
        ref, b = z[:, 0::2] * (F.silu(z[:, 1::2]) if epi == "swiglu" else F.gelu(z[:, 1::2])), bias
        kw = dict(glu=2 if epi == "swiglu" else 1)
    out = ops.linear(a, w, b, **kw)
    close(out, ref, GEMM_ATOL, GEMM_RTOL, f"skinny M{M} {N}x{K} {epi}")
    lib.b200mix_debug_skinny(0)
    try:
        tc = ops.linear(a, w, b, **kw)
    finally:
        lib.b200mix_debug_skinny(1)
    close(out, tc.float(), GEMM_ATOL, GEMM_RTOL, f"skinny vs tensor-core M{M} {N}x{K} {epi}")


@pytest.mark.parametrize("splits", [1, 2, 3, 5, 8])
@pytest.mark.parametrize("M,N,K", [(4, 3584, 18944), (4, 38, 3584), (8, 130, 1096), (1, 1000, 4096), (7, 66, 520)])
def test_linear_skinny_cluster_split_k(ops, M, N, K, splits):
    """The K split of the skinny kernel (partials travel through distributed shared memory to the cluster's first CTA and
    are added in rank order): every forced split factor gives the fp32 reference and is bit-identical run to run."""
    import ctypes
    from paddlemix_b200._lib import lib
    lib.b200mix_debug_skinny_splits.argtypes, lib.b200mix_debug_skinny_splits.restype = [ctypes.c_int], None
    a, w = rnd(M, K, seed=120), rnd(N, K, seed=121, scale=K ** -0.5)
    bias, res = rnd(N, seed=122, dtype=torch.float32), rnd(M, N, seed=123)
    ref = a.float() @ w.float().t() + bias + res.float()
    lib.b200mix_debug_skinny_splits(splits)
    try:
        out = ops.linear(a, w, bias, residual=res)
        again = ops.linear(a, w, bias, residual=res)
    finally:
        lib.b200mix_debug_skinny_splits(0)
    close(out, ref, GEMM_ATOL, GEMM_RTOL, f"skinny split{splits} M{M} {N}x{K}")
    assert torch.equal(out, again)
