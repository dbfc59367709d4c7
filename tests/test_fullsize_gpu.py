"""Parity at BASELINE.json's FULL sizes (configs[1]: SDXL-base UNet, batch 8, 1024^2 -> latent 128x128, bf16).

The CPU oracle needs ~20 s per image at this size, so (a) every dominant GEMM / conv / attention problem of that
forward is checked at its real shape against a plain fp32 torch evaluation ON THE GPU (TF32 off) of the same operator,
and (b) the whole model is checked through size-independent properties: determinism, batch independence (a sample's
output does not depend on its batch neighbours), finiteness, and the fused DDIM update against the CPU oracle's fp32
step on the full [8,4,128,128] state (bit-exact)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16


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
    err = (a.float() - b.float()).abs()
    bad = (err > atol + rtol * b.float().abs()).sum().item()
    assert bad == 0, f"{what}: {bad}/{a.numel()} mismatches, max err {err.max().item():.4g}"


def gelu_erf(x):
    return 0.5 * x * (1 + torch.erf(x * 0.7071067811865476))


# (name, M, N, K, epilogue) of the SDXL forward's dominant Linear problems 
LINEARS = [("ff1 GEGLU 1280", 8192, 10240, 1280, "geglu"), ("ff2 1280", 8192, 1280, 5120, "bias+res"),
           ("qkv 1280", 8192, 3840, 1280, "plain"), ("out 1280", 8192, 1280, 1280, "bias+res"),
           ("ff1 GEGLU 640", 32768, 5120, 640, "geglu"), ("ff2 640", 32768, 640, 2560, "bias+res"),
           ("out 640", 32768, 640, 640, "bias+res"), ("proj 320", 131072, 320, 320, "bias")]


@pytest.mark.parametrize("name,M,N,K,epi", LINEARS)
def test_sdxl_linear_shapes_vs_fp32(ops, name, M, N, K, epi):
    from paddlemix_b200._lib import GLU_GEGLU
    a, w = rnd(M, K, seed=1), rnd(N, K, seed=2, scale=K ** -0.5)
    bias = rnd(N, seed=3, dtype=torch.float32) if epi != "plain" else None
    acc = a.float() @ w.float().t()
    if bias is not None:
        acc = acc + bias
    if epi == "geglu":
        # the product interleaves (value_j, gate_j) rows of the reference's [value | gate] projection at load time
        out = ops.linear(a, w, bias, glu=GLU_GEGLU)
        ref = acc[:, 0::2] * gelu_erf(acc[:, 1::2])
    elif epi == "bias+res":
        res = rnd(M, N, seed=4)
        out = ops.linear(a, w, bias, residual=res)
        ref = acc + res.float()
    else:
        out = ops.linear(a, w, bias)
        ref = acc
    close(out, ref, 2e-2, 1e-2, f"{name} {M}x{N}x{K} {epi}")


@pytest.mark.parametrize("B,H,Cin,Cout,stride", [(8, 32, 1280, 1280, 1), (8, 64, 640, 640, 1), (8, 128, 320, 320, 1),
                                                 (8, 32, 2560, 1280, 1), (8, 128, 320, 320, 2), (8, 128, 960, 320, 1)])
def test_sdxl_conv_shapes_vs_fp32(ops, B, H, Cin, Cout, stride):
    x, w = rnd(B, H, H, Cin, seed=5), rnd(Cout, 3, 3, Cin, seed=6, scale=(9 * Cin) ** -0.5)
    bias = rnd(Cout, seed=7, dtype=torch.float32)
    out = ops.conv3x3(x, w, bias, stride=stride)
    for b in (0, B - 1):  # two images keep the fp32 reference's memory modest; every image runs the same code path
        ref = F.conv2d(x[b:b + 1].float().permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2), bias, stride=stride, padding=1)
        close(out[b:b + 1], ref.permute(0, 2, 3, 1), 2e-2, 1e-2, f"conv {Cin}->{Cout}@{H} s{stride} image {b}")


@pytest.mark.parametrize("B,Sq,Sk,H", [(8, 4096, 4096, 10), (8, 1024, 1024, 20), (8, 1024, 77, 20), (8, 4096, 77, 10)])
def test_sdxl_attention_shapes_vs_fp32(ops, B, Sq, Sk, H):
    D = 64
    q, k, v = rnd(B, Sq, H, D, seed=8), rnd(B, Sk, H, D, seed=9), rnd(B, Sk, H, D, seed=10)
    out = ops.sdpa(q, k, v)
    for b, h in ((0, 0), (B - 1, H - 1), (B // 2, H // 2)):
        s = (q[b, :, h].float() @ k[b, :, h].float().t()) * D ** -0.5
        ref = torch.softmax(s, -1) @ v[b, :, h].float()
        close(out[b, :, h], ref, 1.5e-2, 2e-2, f"attention B{B} Sq{Sq} Sk{Sk} H{H} slice ({b},{h})")


def test_sdxl_norm_shapes_vs_fp32(ops):
    x = (rnd(8192, 1280, seed=11) + 0.3).to(bf16)
    w, b = rnd(1280, seed=12, dtype=torch.float32), rnd(1280, seed=13, dtype=torch.float32)
    close(ops.layernorm(x, w, b, eps=1e-5), F.layer_norm(x.float(), (1280,), w, b, 1e-5), 2e-2, 1e-2, "layernorm 8192x1280")
    for B, HW, C in ((8, 16384, 320), (8, 1024, 1280)):
        xg = (rnd(B, HW, C, seed=14) * 1.5 + 0.2).to(bf16)
        g, be = rnd(C, seed=15, dtype=torch.float32), rnd(C, seed=16, dtype=torch.float32)
        ref = F.silu(F.group_norm(xg.float().permute(0, 2, 1), 32, g, be, 1e-5)).permute(0, 2, 1)
        close(ops.groupnorm_nhwc(xg, g, be, groups=32, eps=1e-5, silu=True), ref, 2e-2, 1e-2, f"groupnorm {B}x{HW}x{C}")


def test_sdxl_full_size_model_properties(ops):
    """SDXL-base UNet at 1024^2 (latent 128x128): determinism, batch independence, finiteness; DDIM update of the full
    [8,4,128,128] state bit-exact against the oracle's fp32 step."""
    from bench import SDXL
    from oracle.schedulers import DDIMScheduler as ODDIM
    from paddlemix_b200.ppdiffusers.schedulers import DDIMScheduler
    from paddlemix_b200.ppdiffusers.unet_2d_condition import UNet2DConditionModel
    unet = UNet2DConditionModel(**SDXL).init_synthetic_weights(seed=1, device=0)
    g = torch.Generator().manual_seed(2)
    B = 2
    x = torch.randn(B, 4, 128, 128, generator=g).cuda()
    ctx = torch.randn(B, 77, 2048, generator=g).to(bf16).cuda()
    added = {"text_embeds": torch.randn(B, 1280, generator=g).to(bf16).cuda(),
             "time_ids": torch.tensor([[1024., 1024., 0, 0, 1024., 1024.]] * B).cuda()}
    a = unet(x, 981, ctx, added_cond_kwargs=added).sample
    b = unet(x, 981, ctx, added_cond_kwargs=added).sample
    assert a.shape == (B, 4, 128, 128) and torch.isfinite(a.float()).all()
    assert torch.equal(a, b), "full-size forward is not deterministic"
    one = unet(x[1:2], 981, ctx[1:2], added_cond_kwargs={k: v[1:2] for k, v in added.items()}).sample
    scale = a.float().abs().max().item()
    assert (one.float() - a[1:2].float()).abs().max().item() <= 2e-2 * scale, "sample 1 depends on its batch neighbour"
    assert (a[0].float() - a[1].float()).abs().max().item() > 1e-3 * scale  # different inputs -> different outputs
    del unet
    torch.cuda.empty_cache()
    SD = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False, set_alpha_to_one=False,
              steps_offset=1)
    o, s = ODDIM(**SD), DDIMScheduler(**SD)
    o.set_timesteps(50), s.set_timesteps(50)
    lat, eps = torch.randn(8, 4, 128, 128, generator=g), torch.randn(8, 4, 128, 128, generator=g)
    for t in s.timesteps[:2]:
        nxt = s.step(eps.cuda(), int(t), lat.cuda())
        lat = o.step(eps, t, lat)
        assert torch.equal(nxt.cpu(), lat), f"DDIM step at t={int(t)} is not bit-exact on the full-size state"


# configs[2] SD3-medium (4 images per GPU: 4096 image + 154 text tokens, D = 1536, 24 x 64 heads) and configs[3] Qwen2-VL-7B
# prefill (3072 tokens, hidden 3584, 28 / 4 heads x 128, intermediate 18944): the dominant problems at their real shapes
@pytest.mark.parametrize("name,M,N,K,epi", [("sd3 qkv", 16384, 4608, 1536, "bias"), ("sd3 ff1 gelu_tanh", 16384, 6144, 1536, "gelu_tanh"),
                                            ("sd3 ff2 gate+res", 16384, 1536, 6144, "gate+res"),
                                            ("qwen gate_up SwiGLU", 3072, 37888, 3584, "swiglu"), ("qwen down", 3072, 3584, 18944, "res"),
                                            ("qwen lm_head fp32", 3072, 152064, 3584, "f32")])
def test_sd3_qwen_linear_shapes_vs_fp32(ops, name, M, N, K, epi):
    from paddlemix_b200._lib import ACT_GELU_TANH, GLU_SWIGLU
    a, w = rnd(M, K, seed=21), rnd(N, K, seed=22, scale=K ** -0.5)
    acc = a.float() @ w.float().t()
    if epi == "bias":
        bias = rnd(N, seed=23, dtype=torch.float32)
        out, ref = ops.linear(a, w, bias), acc + bias
    elif epi == "gelu_tanh":
        bias = rnd(N, seed=23, dtype=torch.float32)
        out, ref = ops.linear(a, w, bias, act=ACT_GELU_TANH), F.gelu(acc + bias, approximate="tanh")
    elif epi == "gate+res":  # h + gate_mlp * ff(...)  (attention.py:196-214): per-sample gate vector, 4 samples
        bias, gate, res = rnd(N, seed=23, dtype=torch.float32), rnd(4, N, seed=24, dtype=torch.float32), rnd(M, N, seed=25)
        out = ops.linear(a, w, bias, row_gate=gate, rows_per_group=M // 4, residual=res)
        ref = (acc + bias) * gate.repeat_interleave(M // 4, 0) + res.float()
    elif epi == "swiglu":  # interleaved (up_j, gate_j) rows: silu(gate) * up
        out, ref = ops.linear(a, w, glu=GLU_SWIGLU), acc[:, 0::2] * F.silu(acc[:, 1::2])
    elif epi == "res":
        res = rnd(M, N, seed=25)
        out, ref = ops.linear(a, w, residual=res), acc + res.float()
    else:
        out, ref = ops.linear(a, w, out_fp32=True), acc
        assert out.dtype == torch.float32
    close(out, ref, 2e-2, 1e-2, f"{name} {M}x{N}x{K}")


@pytest.mark.parametrize("B,S,Hq,Hkv,D,causal", [(4, 4250, 24, 24, 64, False), (4, 768, 28, 4, 128, True)])
def test_sd3_qwen_attention_shapes_vs_fp32(ops, B, S, Hq, Hkv, D, causal):
    q, k, v = rnd(B, S, Hq, D, seed=26), rnd(B, S, Hkv, D, seed=27), rnd(B, S, Hkv, D, seed=28)
    out = ops.sdpa(q, k, v, causal=causal)
    for b, h in ((0, 0), (B - 1, Hq - 1)):
        hk = h // (Hq // Hkv)
        s = (q[b, :, h].float() @ k[b, :, hk].float().t()) * D ** -0.5
        if causal:
            s = s.masked_fill(torch.ones(S, S, device="cuda", dtype=torch.bool).triu(1), float("-inf"))
        close(out[b, :, h], torch.softmax(s, -1) @ v[b, :, hk].float(), 1.5e-2, 2e-2, f"attention S{S} H{Hq}/{Hkv} D{D} ({b},{h})")
