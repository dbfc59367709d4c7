"""Attention kernels (round 2): the persistent ping-pong kernel (D = 64 self-attention), additive attention masks on
every kernel (the reference's `attn_mask`, paddle_patch.py:418,454-455), batch elements without visible keys, and the
argument checks of b200mix_sdpa. Reference = fp32 torch softmax(q k^T * scale + mask) v on the same bf16 inputs.
Tolerance: P is rounded to bf16 before PV and the output is bf16 -> 1.5e-2 abs + 2e-2 rel."""
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


def rnd(*shape, seed=0, scale=1.0, dtype=bf16):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype).cuda()


def close(a, b, what=""):
    a, b = a.float().cpu(), b.float().cpu()
    err = (a - b).abs()
    bad = (err > ATOL + RTOL * b.abs()).sum().item()
    assert bad == 0 and torch.isfinite(a).all(), f"{what}: {bad}/{a.numel()} mismatches, max err {err.max().item():.4g}"


def ref_sdpa(q, k, v, scale, mask=None, kv_lens=None):
    """q [B,Sq,H,D], k/v [B,Sk,Hkv,D], mask broadcastable to [B,H,Sq,Sk] (additive), kv_lens list -> [B,Sq,H,D] fp32."""
    qf, kf, vf = (t.float().permute(0, 2, 1, 3) for t in (q, k, v))
    rep = qf.shape[1] // kf.shape[1]
    kf, vf = kf.repeat_interleave(rep, 1), vf.repeat_interleave(rep, 1)
    s = qf @ kf.transpose(-1, -2) * scale
    if mask is not None:
        s = s + mask.float()
    if kv_lens is not None:
        for b, n in enumerate(kv_lens):
            s[b, :, :, n:] = float("-inf")
    p = torch.softmax(s, -1)
    p = torch.nan_to_num(p, nan=0.0)  # rows without any visible key: zeros (the kernels' convention)
    return (p @ vf).permute(0, 2, 1, 3)


# ---- persistent ping-pong kernel ----------------------------------------------------------------------------------
@pytest.mark.parametrize("B,Sq,Sk,Hq,Hkv", [
    (1, 256, 256, 1, 1),      # one item, two blocks
    (2, 1024, 1024, 4, 4),    # several items per CTA range boundary
    (3, 300, 450, 3, 3),      # odd number of query tiles (phantom second tile), ragged last key block
    (1, 64, 200, 8, 8),       # fewer query rows than one tile
    (1, 4250, 4250, 2, 2),    # SD3: 4096 image + 154 text tokens
    (2, 640, 1300, 6, 2),     # GQA, Sq != Sk
    (2, 4096, 4096, 10, 10),  # SDXL top level
    (8, 1024, 1024, 20, 20),  # SDXL 32x32 level (the benched shape)
])
def test_pingpong_matches_reference(ops, B, Sq, Sk, Hq, Hkv):
    q, k, v = rnd(B, Sq, Hq, 64, seed=1), rnd(B, Sk, Hkv, 64, seed=2), rnd(B, Sk, Hkv, 64, seed=3)
    out = ops.sdpa(q, k, v)
    for b in sorted({0, B - 1}):  # the fp32 reference of one batch element at a time keeps the score matrix small
        close(out[b:b + 1], ref_sdpa(q[b:b + 1], k[b:b + 1], v[b:b + 1], 0.125), f"pingpong B{B} Sq{Sq} Sk{Sk} b{b}")


@pytest.mark.parametrize("B,Sq,Sk,H", [(2, 1024, 1024, 4), (3, 300, 450, 3), (4, 2048, 2048, 10)])
def test_pingpong_agrees_with_one_tile_kernel(ops, B, Sq, Sk, H):
    from paddlemix_b200._lib import lib
    q, k, v = rnd(B, Sq, H, 64, seed=4), rnd(B, Sk, H, 64, seed=5), rnd(B, Sk, H, 64, seed=6)
    out = ops.sdpa(q, k, v)
    lib.b200mix_debug_attn_bn64(1)
    try:
        old = ops.sdpa(q, k, v)
    finally:
        lib.b200mix_debug_attn_bn64(0)
    close(out, old, "128-key vs 64-key blocks")
    assert torch.equal(out, ops.sdpa(q, k, v)), "the kernel must be deterministic"


def test_pingpong_kv_lens_and_large_logits(ops):
    B, Sq, Sk, H = 4, 512, 700, 3
    q, k, v = rnd(B, Sq, H, 64, seed=7, scale=4.0), rnd(B, Sk, H, 64, seed=8, scale=4.0), rnd(B, Sk, H, 64, seed=9)
    lens = [700, 129, 1, 0]  # full, just over one block, one key, no key at all (-> zeros)
    out = ops.sdpa(q, k, v, kv_lens=torch.tensor(lens, dtype=torch.int32, device="cuda"))
    close(out, ref_sdpa(q, k, v, 0.125, kv_lens=lens), "pingpong kv_lens + lazy rescale")
    assert (out[3] == 0).all()


def test_pingpong_fused_qkv_strides(ops):
    B, S, H = 2, 768, 5
    qkv = rnd(B, S, 3 * H * 64, seed=10)
    q, k, v = (qkv[:, :, i * H * 64:(i + 1) * H * 64].unflatten(-1, (H, 64)) for i in range(3))
    close(ops.sdpa(q, k, v), ref_sdpa(q, k, v, 0.125), "pingpong strided views")


# ---- additive masks ------------------------------------------------------------------------------------------------
def _mask(kind, B, H, Sq, Sk, dtype, seed=11):
    g = torch.Generator().manual_seed(seed)
    if kind == "keypad":  # (1 - m) * -10000, [B,1,1,Sk] (unet_2d_condition.py:916-927)
        keep = (torch.rand(B, Sk, generator=g) > 0.3).float()
        keep[:, 0] = 1.0
        return ((1 - keep) * -10000.0)[:, None, None, :].to(dtype).cuda()
    if kind == "full":  # arbitrary bias per (b, h, q, k)
        return (torch.randn(B, H, Sq, Sk, generator=g) * 2.0).to(dtype).cuda()
    if kind == "shared":  # one [Sq, Sk] bias for every batch element and head, with -inf holes
        m = torch.randn(1, 1, Sq, Sk, generator=g)
        m[..., ::7] = float("-inf")
        m[..., 0] = 0.0
        return m.to(dtype).cuda()
    raise ValueError(kind)


@pytest.mark.parametrize("kind", ["keypad", "full", "shared"])
@pytest.mark.parametrize("dtype", [torch.float32, bf16])
@pytest.mark.parametrize("B,Sq,Sk,H,D,path", [
    (2, 384, 300, 3, 64, "pingpong"), (2, 384, 300, 3, 64, "one_tile"), (3, 200, 77, 4, 64, "shortkv"),
    (3, 200, 77, 4, 64, "general_short"), (2, 256, 333, 2, 128, "d128"), (1, 130, 140, 2, 192, "d192"),
])
def test_attn_mask(ops, kind, dtype, B, Sq, Sk, H, D, path):
    from paddlemix_b200._lib import lib
    q, k, v = rnd(B, Sq, H, D, seed=12), rnd(B, Sk, H, D, seed=13), rnd(B, Sk, H, D, seed=14)
    mask = _mask(kind, B, H, Sq, Sk, dtype)
    # one_tile / general_short: the 64-key-block configuration of the D = 64 kernel
    hooks = {"one_tile": (lib.b200mix_debug_attn_bn64, 1, 0), "general_short": (lib.b200mix_debug_attn_bn64, 1, 0)}
    fn, on, off = hooks.get(path, (None, None, None))
    if fn:
        fn(on)
    try:
        out = ops.sdpa(q, k, v, attn_mask=mask)
    finally:
        if fn:
            fn(off)
    close(out, ref_sdpa(q, k, v, D ** -0.5, mask=mask), f"attn_mask {kind} {dtype} {path}")


@pytest.mark.parametrize("Sk,D", [(77, 64), (300, 64), (140, 128)])
def test_mask_last_token_equals_truncation(ops, Sk, D):
    """The property the reference tests (test_models_unet_2d_condition.py:486-519): masking the last context token with
    the (1 - m) * -10000 bias == dropping that token; a keep-all mask == no mask."""
    B, Sq, H = 2, 256, 4
    q, k, v = rnd(B, Sq, H, D, seed=15), rnd(B, Sk, H, D, seed=16), rnd(B, Sk, H, D, seed=17)
    keep_all = torch.zeros(B, 1, 1, Sk, device="cuda")
    assert torch.equal(ops.sdpa(q, k, v, attn_mask=keep_all), ops.sdpa(q, k, v))
    last = torch.zeros(B, 1, 1, Sk, device="cuda")
    last[..., -1] = -10000.0
    masked = ops.sdpa(q, k, v, attn_mask=last)
    trunc = ops.sdpa(q, k[:, :-1], v[:, :-1])
    close(masked, trunc, "mask-last vs truncated")
    assert not torch.allclose(masked.float(), ops.sdpa(q, k, v).float(), atol=1e-3)


# ---- batch elements without visible keys, argument checks ----------------------------------------------------------
@pytest.mark.parametrize("D,Sk,general", [(64, 96, False), (64, 96, True), (128, 120, True), (128, 300, True), (64, 300, True)])
def test_kv_lens_zero_gives_zeros_and_does_not_hang(ops, D, Sk, general):
    from paddlemix_b200._lib import lib
    B, Sq, H = 3, 200, 2
    q, k, v = rnd(B, Sq, H, D, seed=18), rnd(B, Sk, H, D, seed=19), rnd(B, Sk, H, D, seed=20)
    lens = [Sk, 0, 5]
    lib.b200mix_debug_attn_bn64(1 if general else 0)  # general: 64-key blocks
    try:
        out = ops.sdpa(q, k, v, kv_lens=torch.tensor(lens, dtype=torch.int32, device="cuda"))
        torch.cuda.synchronize()
    finally:
        lib.b200mix_debug_attn_bn64(0)
    assert (out[1] == 0).all()
    close(out, ref_sdpa(q, k, v, D ** -0.5, kv_lens=lens), f"kv_lens with an empty batch element D{D} Sk{Sk}")


def test_sdpa_argument_checks(ops):
    from paddlemix_b200._lib import B200MixError
    q, k, v = rnd(1, 256, 2, 128, seed=21), rnd(1, 128, 2, 128, seed=22), rnd(1, 128, 2, 128, seed=23)
    with pytest.raises(B200MixError, match="Sq <= Sk"):
        ops.sdpa(q, k, v, causal=True)  # bottom-right causal with Sq > Sk: first rows see no key
    with pytest.raises(B200MixError, match="attn_mask cannot be combined"):
        ops.sdpa(k, k, v, causal=True, attn_mask=torch.zeros(1, 1, 128, 128, device="cuda"))
    with pytest.raises(ValueError, match="does not broadcast"):
        ops.sdpa(q, k, v, attn_mask=torch.zeros(1, 1, 256, 64, device="cuda"))
    with pytest.raises(TypeError):
        ops.sdpa(q, k, v, attn_mask=torch.zeros(1, 1, 256, 128, device="cuda", dtype=torch.bool))
