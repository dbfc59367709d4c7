"""Which thread of the implicit-GEMM epilogue owns which output element depends on the tile width, and ragged edges
are where an ownership mistake shows. Every tile width x every epilogue flavour x shapes with M % 128 != 0,
N % 32 != 0, N % 8 != 0 (rows not 16-byte aligned: element-wise stores) and an odd number of m-tiles, against a PyTorch
fp32 evaluation on the same bf16-rounded inputs."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16
ATOL, RTOL = 2e-2, 1.0e-2  # bf16 output of an fp32-accumulated dot product: 2^-8 relative rounding dominates
BNS = [32, 64, 128, 160, 192, 224, 256]
# (M, N, K): ragged M + N % 32 != 0 | 5 m-tiles | N % 8 != 0 | ragged M + N % 64 == 32
SHAPES = [(1000, 328, 200), (640, 672, 128), (300, 100, 136), (1000, 352, 200)]
FLAVOURS = ["plain", "stats", "ln", "residual", "geglu", "rowadd_silu", "fp32"]


@pytest.fixture(scope="module")
def gemm():
    from paddlemix_b200 import ops
    from paddlemix_b200._lib import lib
    ops.init(0)
    yield ops, lib
    lib.b200mix_debug_force_bn(0)


def rnd(*shape, seed, scale=1.0, dtype=bf16):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype).cuda()


def close(a, b, atol=ATOL, rtol=RTOL, what=""):
    a, b = a.float().cpu(), b.float().cpu()
    err = (a - b).abs()
    bad = (err > atol + rtol * b.abs()).sum().item()
    assert bad == 0, f"{what}: {bad}/{a.numel()} mismatches, max err {err.max().item():.4g}"


@pytest.mark.parametrize("M,N,K", SHAPES)
@pytest.mark.parametrize("flavour", FLAVOURS)
@pytest.mark.parametrize("bn", BNS)
def test_linear_epilogue_sweep(gemm, bn, flavour, M, N, K):
    ops, lib = gemm
    if flavour == "stats" and N % 32:
        pytest.skip("row statistics need N % 32 == 0")
    a, w = rnd(M, K, seed=1), rnd(N, K, seed=2, scale=K ** -0.5)
    bias = rnd(N, seed=3, dtype=torch.float32)
    res = rnd(M, N, seed=4)
    z = a.float() @ w.float().t() + bias
    lib.b200mix_debug_force_bn(bn)
    try:
        if flavour == "plain":
            out, ref = ops.linear(a, w, bias), z
        elif flavour == "residual":
            out, ref = ops.linear(a, w, bias, residual=res), z + res.float()
        elif flavour == "geglu":
            out, ref = ops.linear(a, w, bias, glu=ops.GLU_GEGLU), z[:, 0::2] * F.gelu(z[:, 1::2])
        elif flavour == "fp32":
            out, ref = ops.linear(a, w, bias, out_fp32=True), z
            assert out.dtype == torch.float32
        elif flavour == "rowadd_silu":
            rpg = 100
            radd = rnd((M + rpg - 1) // rpg, N, seed=5, dtype=torch.float32)
            out = ops.linear(a, w, bias, row_add=radd, rows_per_group=rpg, act=ops.ACT_SILU)
            ref = F.silu(z + radd[torch.arange(M, device="cuda") // rpg])
        elif flavour == "stats":
            out, st = ops.linear(a, w, bias, residual=res, stats=True)
            ref = z + res.float()
            assert torch.equal(out, ops.linear(a, w, bias, residual=res)), "taking the statistics must not change the output"
            tot, of = st.buf.double() / st.SCALE, out.double()
            close(tot[:, 0], of.sum(1), 2e-2, 1e-4, "row sums")
            close(tot[:, 1], (of * of).sum(1), 2e-2, 1e-4, "row sums of squares")
            _, st2 = ops.linear(a, w, bias, residual=res, stats=True)
            assert torch.equal(st2.buf, st.buf), "fixed-point row statistics must be reproducible bit for bit"
        else:  # ln: the consumer side, with the statistics of `a`'s rows computed exactly on the host side
            af = (a.float() + 1.5).to(bf16)  # a row mean well away from zero
            d = af.double()
            buf = torch.stack([d.sum(1), (d * d).sum(1)], 1).mul(ops.RowStats.SCALE).round().to(torch.int64).contiguous()
            gamma = 1.0 + 0.3 * rnd(K, seed=6, dtype=torch.float32)
            beta = 0.2 * rnd(K, seed=7, dtype=torch.float32)
            w1 = rnd(N, K, seed=8, dtype=torch.float32) * K ** -0.5
            w1f, colsum, b1f = ops.fold_layernorm_into_linear(w1, gamma, beta, bias)
            out = ops.linear(af, w1f, b1f, ln=(ops.RowStats(buf, K), colsum, 1e-5))
            ref = F.linear(F.layer_norm(af.float(), (K,), gamma, beta, 1e-5), w1, bias)
            close(out, ref, 3e-2, 1.5e-2, f"ln {M}x{N}x{K} bn={bn}")
            return
    finally:
        lib.b200mix_debug_force_bn(0)
    close(out, ref, what=f"{flavour} {M}x{N}x{K} bn={bn}")


@pytest.mark.parametrize("flavour", ["plain", "residual", "rowadd_silu"])
@pytest.mark.parametrize("bn", BNS)
def test_conv3x3_epilogue_sweep(gemm, bn, flavour):
    """3 x 12 x 20 pixels: 4 x 4 x 8 tile boxes, 15 m-tiles (odd), boxes that run past the batch; Cout % 32 != 0."""
    ops, lib = gemm
    B, H, W, Cin, Cout = 3, 12, 20, 64, 72
    x = rnd(B, H, W, Cin, seed=11)
    w = rnd(Cout, 3, 3, Cin, seed=12, scale=(9 * Cin) ** -0.5)
    bias = rnd(Cout, seed=13, dtype=torch.float32)
    res = rnd(B, H, W, Cout, seed=14)
    radd = rnd(B, Cout, seed=15, dtype=torch.float32)
    z = F.conv2d(x.float().permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2), bias, padding=1).permute(0, 2, 3, 1)
    lib.b200mix_debug_force_bn(bn)
    try:
        if flavour == "plain":
            out, ref = ops.conv3x3(x, w, bias), z
        elif flavour == "residual":
            out, ref = ops.conv3x3(x, w, bias, residual=res), z + res.float()
        else:
            out, ref = ops.conv3x3(x, w, bias, row_add=radd, act=ops.ACT_SILU), F.silu(z + radd[:, None, None, :])
    finally:
        lib.b200mix_debug_force_bn(0)
    close(out, ref, what=f"conv3x3 {flavour} bn={bn}")
