"""The implicit GEMM's shared-memory ring under load: persistent CTAs that run many tiles, so every stage is refilled many
times, with the stages of the clustered kernel released across the two CTAs of a cluster (gemm_pair 1) and without
clusters (gemm_pair 0). Both schedules run the same tiles with the same k order, so their outputs must agree bit for bit,
and two runs of either must too. A stage handed back to TMA before every wgmma that reads it has finished would show up
here as a mismatch. Covered: every tile width, the plain / residual / GEGLU epilogues, odd tile counts per cluster
(capped grids) and stream-K heads (shallow reductions split as well)."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16
BNS = [32, 64, 128, 160, 192, 224, 256]


@pytest.fixture(scope="module")
def gemm():
    from paddlemix_b200 import ops
    from paddlemix_b200._lib import lib
    ops.init(0)
    for f in (lib.b200mix_debug_streamk, lib.b200mix_debug_max_clusters):
        f.argtypes, f.restype = [ctypes.c_int], None
    yield ops, lib
    lib.b200mix_debug_force_bn(0)
    lib.b200mix_debug_gemm_pair(1)
    lib.b200mix_debug_streamk(1)
    lib.b200mix_debug_max_clusters(0)


def rnd(*shape, seed, scale=1.0, dtype=bf16):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype).cuda()


def run(ops, lib, flavour, a, w, bias, res, bn, pair, streamk, clusters):
    lib.b200mix_debug_force_bn(bn)
    lib.b200mix_debug_gemm_pair(pair)
    lib.b200mix_debug_streamk(streamk)
    lib.b200mix_debug_max_clusters(clusters)
    try:
        if flavour == "plain":
            out = ops.linear(a, w, bias)
        elif flavour == "residual":
            out = ops.linear(a, w, bias, residual=res)
        else:
            out = ops.linear(a, w, bias, glu=ops.GLU_GEGLU)
        torch.cuda.synchronize()
        return out
    finally:
        lib.b200mix_debug_force_bn(0)
        lib.b200mix_debug_gemm_pair(1)
        lib.b200mix_debug_streamk(1)
        lib.b200mix_debug_max_clusters(0)


# (streamk, max clusters): round-robin on the whole machine | 7 clusters (odd tile counts per cluster) with a stream-K
# head over a shallow reduction | 66 clusters with the stream-K head
SCHEDULES = [(0, 0), (2, 7), (2, 0)]


@pytest.mark.parametrize("streamk,clusters", SCHEDULES)
@pytest.mark.parametrize("flavour", ["plain", "residual", "geglu"])
@pytest.mark.parametrize("bn", BNS)
def test_ring_pair_and_single_agree(gemm, bn, flavour, streamk, clusters):
    ops, lib = gemm
    M, N, K = 3000, 1280, 1280 if clusters else 640  # 24 m-tiles (12 pairs), 20 / 10 k-blocks per tile
    a, w = rnd(M, K, seed=1), rnd(N, K, seed=2, scale=K ** -0.5)
    bias = rnd(N, seed=3, dtype=torch.float32)
    res = rnd(M, N, seed=4)
    args = (ops, lib, flavour, a, w, bias, res, bn)
    p1 = run(*args, 1, streamk, clusters)
    p0 = run(*args, 0, streamk, clusters)
    assert torch.equal(p1, p0), f"gemm_pair 1 and 0 differ: {flavour} bn={bn} streamk={streamk} clusters={clusters}"
    assert torch.equal(p1, run(*args, 1, streamk, clusters)), "two runs of the clustered kernel differ"
    z = a.float() @ w.float().t() + bias
    ref = z + res.float() if flavour == "residual" else (
        z[:, 0::2] * torch.nn.functional.gelu(z[:, 1::2]) if flavour == "geglu" else z)
    err = (p1.float() - ref).abs()
    assert (err <= 2e-2 + 1e-2 * ref.abs()).all(), f"max err {err.max().item():.4g}"
