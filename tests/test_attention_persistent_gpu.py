"""The persistent attention schedule (attn_kernel, csrc/attention.cu): each CTA walks (query tile, head, batch) work
tiles, so the shapes that matter are the ones that end the walk differently - fewer work tiles than SMs, a tile count
that is not a multiple of the grid, many short varlen sequences (work tiles without rows), causal attention with
Sq < Sk next to batch elements without keys - plus the SDXL 32x32-level shape and run-to-run bit identity.
Reference = fp32 torch softmax(q k^T * scale [+ causal]) v on the same bf16 inputs, tolerance as in
test_attention_gpu.py."""
import pytest
import torch

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16
ATOL, RTOL = 1.5e-2, 2e-2


@pytest.fixture(scope="module")
def ops():
    from paddlemix_b200 import ops as _ops
    _ops.init(0)
    return _ops


def rnd(*shape, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g).to(bf16).cuda()


def close(a, b, what=""):
    a, b = a.float().cpu(), b.float().cpu()
    err = (a - b).abs()
    bad = (err > ATOL + RTOL * b.abs()).sum().item()
    assert bad == 0 and torch.isfinite(a).all(), f"{what}: {bad}/{a.numel()} mismatches, max err {err.max().item():.4g}"


def ref_sdpa(q, k, v, causal=False, kv_lens=None):
    """q [B,Sq,H,D], k/v [B,Sk,Hkv,D] -> fp32 [B,Sq,H,D]; causal is bottom-right aligned (query i sees keys
    <= i + Sk - Sq); rows without a visible key give zeros."""
    qf, kf, vf = (t.float().permute(0, 2, 1, 3) for t in (q, k, v))
    rep = qf.shape[1] // kf.shape[1]
    kf, vf = kf.repeat_interleave(rep, 1), vf.repeat_interleave(rep, 1)
    s = qf @ kf.transpose(-1, -2) * q.shape[-1] ** -0.5
    Sq, Sk = s.shape[-2:]
    if causal:
        vis = torch.arange(Sk)[None, :] <= torch.arange(Sq)[:, None] + (Sk - Sq)
        s = s.masked_fill(~vis.to(s.device), float("-inf"))
    if kv_lens is not None:
        for b, n in enumerate(kv_lens):
            s[b, :, :, n:] = float("-inf")
    p = torch.nan_to_num(torch.softmax(s, -1), nan=0.0)
    return (p @ vf).permute(0, 2, 1, 3)


def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("D", [64, 128, 192])
def test_fewer_work_tiles_than_sms(ops, D):
    B, S, H = 1, 300, 2  # 3 query tiles x 2 heads
    assert B * H * 3 < num_sms()
    q, k, v = rnd(B, S, H, D, seed=1), rnd(B, S, H, D, seed=2), rnd(B, S, H, D, seed=3)
    close(ops.sdpa(q, k, v), ref_sdpa(q, k, v), f"6 work tiles D{D}")


@pytest.mark.parametrize("causal", [False, True])
def test_work_tiles_not_a_multiple_of_the_grid(ops, causal):
    B, S, H = 1, 2048, 9  # 16 query tiles x 9 heads = 144 work tiles
    tiles = B * H * (S // 128)
    assert tiles > num_sms() and tiles % num_sms()
    q, k, v = rnd(B, S, H, 64, seed=4), rnd(B, S, H, 64, seed=5), rnd(B, S, H, 64, seed=6)
    close(ops.sdpa(q, k, v, causal=causal), ref_sdpa(q, k, v, causal=causal), f"144 work tiles causal={causal}")


def test_sdxl_level3_shape_and_run_to_run_bits(ops):
    B, S, H = 8, 1024, 20  # SDXL 32x32 level: 8 x 20 x 8 = 1280 work tiles
    q, k, v = rnd(B, S, H, 64, seed=7), rnd(B, S, H, 64, seed=8), rnd(B, S, H, 64, seed=9)
    out = ops.sdpa(q, k, v)
    for b in (0, 3, 7):
        close(out[b:b + 1], ref_sdpa(q[b:b + 1], k[b:b + 1], v[b:b + 1]), f"SDXL level 3 b{b}")
    assert torch.equal(out, ops.sdpa(q, k, v)), "two runs must agree bit for bit"
    ctx_k, ctx_v = rnd(B, 77, H, 64, seed=10), rnd(B, 77, H, 64, seed=11)  # cross-attention over 77 keys
    cross = ops.sdpa(q, ctx_k, ctx_v)
    close(cross[:2], ref_sdpa(q[:2], ctx_k[:2], ctx_v[:2]), "SDXL level 3 cross-attention")
    assert torch.equal(cross, ops.sdpa(q, ctx_k, ctx_v)), "two runs must agree bit for bit"


@pytest.mark.parametrize("D,causal", [(64, False), (64, True), (128, True), (192, False)])
def test_varlen_many_short_sequences(ops, D, causal):
    g = torch.Generator().manual_seed(12)
    lens = torch.randint(1, 200, (40,), generator=g).tolist() + [1, 129, 300]
    cu = [0]
    for n in lens:
        cu.append(cu[-1] + n)
    T, H = cu[-1], 3
    q, k, v = rnd(1, T, H, D, seed=13), rnd(1, T, H, D, seed=14), rnd(1, T, H, D, seed=15)
    out = ops.sdpa(q, k, v, causal=causal, cu_seqlens=torch.tensor(cu, dtype=torch.int32, device="cuda"))
    ref = torch.cat([ref_sdpa(q[:, a:b], k[:, a:b], v[:, a:b], causal=causal) for a, b in zip(cu[:-1], cu[1:])], 1)
    close(out, ref, f"varlen {len(lens)} sequences D{D} causal={causal}")


@pytest.mark.parametrize("D", [64, 128])
def test_causal_short_queries_with_empty_batch_elements(ops, D):
    B, Sq, Sk, H = 3, 200, 500, 2
    lens = [500, 0, 260]
    q, k, v = rnd(B, Sq, H, D, seed=16), rnd(B, Sk, H, D, seed=17), rnd(B, Sk, H, D, seed=18)
    out = ops.sdpa(q, k, v, causal=True, kv_lens=torch.tensor(lens, dtype=torch.int32, device="cuda"))
    assert (out[1] == 0).all()
    close(out, ref_sdpa(q, k, v, causal=True, kv_lens=lens), f"causal Sq<Sk with kv_lens D{D}")
