"""Open-Sora text-to-video sampling on the GPU against oracle/iddpm.py: the fused IDDPM step kernel (bit-exact given
the noise, and its Philox normals), the pipeline's loop plumbing with a stub transformer, the loop with STDiT2-XL cut to
depth 2 against the fp32 oracle, and the per-frame VAE decode.

Real-model bounds. The pipeline's STDiT2 runs bf16 GEMMs and a bf16 residual stream; the oracle is fp32 (TF32 off).
Three steps of 2 samples (caption lengths 120 and 57, latent 4 x 16 x 24) with the same Philox noise, cfg_scale 7 on
3 channels, which multiplies the model's error on those channels by up to 15. Measured on an H100 80GB HBM3 (700 W power
limit): normwise error of the final latents 1.85e-2, largest element error 0.091 rms of the reference. The bounds
(4e-2, 0.2 rms) leave about 2x headroom. On the same card the kernel's 2^20 Philox normals matched the oracle's bit for
bit, and the stub loop matched the oracle's 2B-row loop exactly (the bound there is 1e-6 relative).
"""
import math

import pytest
import torch

from oracle import iddpm as O

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16


@pytest.fixture(scope="module")
def ops():
    from paddlemix_b200 import ops as _ops
    _ops.init(0)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return _ops


def cfg_combine_ref(m, B, cfg_scale, cc):
    """forward_with_cfg's combine, conditional rows of the result: fp32 [B, 2C, ...]."""
    m = m.float()
    g = m[:B].clone()
    g[:, :cc] = m[B:, :cc] + cfg_scale * (m[:B, :cc] - m[B:, :cc])
    return g


# ---- the step kernel -------------------------------------------------------------------------------------------------
SHAPE = (4, 4, 16, 64, 64)


@pytest.mark.parametrize("i", [99, 50, 0])
@pytest.mark.parametrize("cc", [3, 4])
@pytest.mark.parametrize("dtype", [torch.float32, bf16], ids=["fp32", "bf16"])
def test_step_bit_exact_with_explicit_noise(ops, dtype, cc, i):
    from paddlemix_b200.opensora import IDDPM
    B, C = SHAPE[:2]
    g = torch.Generator().manual_seed(100 + i + cc)
    m = torch.randn(2 * B, 2 * C, *SHAPE[2:], generator=g).to(dtype)
    m[:, C:] = m[:, C:].float().clamp(-1, 1).to(dtype)  # variance values in the model's range
    x = torch.randn(SHAPE, generator=g)
    noise = torch.randn(SHAPE, generator=g)
    s, d = IDDPM(num_sampling_steps=100, cfg_scale=7.0, cfg_channel=cc), O.Diffusion(1000, "100")
    out = s.step(m.cuda(), i, x.cuda(), noise=noise.cuda())
    ref = d.p_sample(cfg_combine_ref(m, B, 7.0, cc), x, i, noise)
    assert torch.equal(out.cpu(), ref)
    # in place, with the second copy for the unconditional half of the model input
    buf = torch.cat([x, x]).cuda()
    s.step(m.cuda(), i, buf[:B], noise=noise.cuda(), out=buf[:B], out_dup=buf[B:])
    assert torch.equal(buf[:B].cpu(), ref) and torch.equal(buf[B:].cpu(), ref)


def philox_normals(ops, seed, step, shape=SHAPE):
    """The kernel's normals: with every scalar 0 the step returns 0 + exp(0) * z = z."""
    B, C = shape[:2]
    m = torch.zeros(2 * B, 2 * C, *shape[2:], device="cuda")
    x = torch.zeros(shape, device="cuda")
    return ops.iddpm_step(m, x, 1.0, C, (0.0,) * 6, add_noise=True, seed=seed, step=step)


def test_philox_normals_match_oracle(ops):
    seed, step = 0x1234_5678_9ABC_DEF0 & (2 ** 63 - 1), 77
    z = philox_normals(ops, seed, step).cpu().reshape(-1)
    ref = O.philox_normal(seed, step, z.numel())
    ulp = (z.view(torch.int32).long() - ref.view(torch.int32).long()).abs()
    n_diff = int((ulp != 0).sum())
    print(f"philox normals: {n_diff} of {z.numel()} differ from the oracle, max {int(ulp.max())} ulp")
    assert int(ulp.max()) <= 1 and n_diff <= 16
    assert torch.equal(philox_normals(ops, seed, step).cpu().reshape(-1), z)       # same seed and step: same bits
    for other in (philox_normals(ops, seed, step + 1), philox_normals(ops, seed + 1, step)):
        assert (other.cpu().reshape(-1) != z).float().mean().item() > 0.99
    n = z.numel()
    zd = z.double()
    assert abs(zd.mean().item()) < 5 / math.sqrt(n)
    assert abs(zd.std().item() - 1) < 5 / math.sqrt(2 * n)


def test_step_philox_and_index_zero(ops):
    """With Philox noise the step is the oracle's with the oracle's normals (within 1 ulp of them); at index 0 no
    noise is added, whatever the seed."""
    from paddlemix_b200.opensora import IDDPM
    B, C = SHAPE[:2]
    g = torch.Generator().manual_seed(5)
    m = torch.randn(2 * B, 2 * C, *SHAPE[2:], generator=g).clamp(-1, 1)
    x = torch.randn(SHAPE, generator=g)
    s, d = IDDPM(num_sampling_steps=100, cfg_scale=4.0), O.Diffusion(1000, "100")
    out = s.step(m.cuda(), 50, x.cuda(), seed=9).cpu()
    ref = d.p_sample(cfg_combine_ref(m, B, 4.0, C), x, 50, O.philox_normal(9, 50, x.numel()).reshape(SHAPE))
    assert (out - ref).abs().max().item() <= 1e-6 * ref.abs().max().item()
    z0 = [s.step(m.cuda(), 0, x.cuda(), seed=sd).cpu() for sd in (1, 2)]
    ref0 = d.p_sample(cfg_combine_ref(m, B, 4.0, C), x, 0, None)
    assert torch.equal(z0[0], ref0) and torch.equal(z0[1], ref0)


# ---- the loop's plumbing ---------------------------------------------------------------------------------------------
class StubSTDiT2:
    """STDiT2's forward signature; per-row output from + and * only (rounded the same on CPU and GPU). On the GPU it
    checks what the pipeline hands over: cond rows first, the null caption, the mask at B rows, the 2B size tensors."""

    def __init__(self, B, null=None, prompt=None, mask=None):
        self.B, self.prompt, self.mask, self.null_y = B, prompt, mask, null
        self.device = torch.device("cuda")
        self.calls = 0

    def null_caption(self, n):
        return self.null_y[None, None].repeat(n, 1, 1, 1)

    def __call__(self, x, t, y, mask=None, num_frames=None, height=None, width=None, ar=None, fps=None, **kw):
        B = self.B
        if x.is_cuda:
            self.calls += 1
            assert x.shape[0] == 2 * B and torch.equal(x[:B], x[B:])
            assert torch.equal(y[:B], self.prompt.to(bf16)) and torch.equal(y[B:], self.null_caption(B).to(bf16))
            assert (mask is None and self.mask is None) or torch.equal(mask, self.mask)
            for v in (num_frames, height, width, ar, fps, t):
                assert v.shape == (2 * B,)
        C = x.shape[1]
        yv = y[:, 0, 0, 0].float().reshape(-1, 1, 1, 1, 1)
        tv = (t.float() * 0.001).reshape(-1, 1, 1, 1, 1)
        eps = x * 0.5 + yv * (1.0 - tv)
        var = x[:, :C] * 0.01 + yv * 0.3 - tv * 0.2
        return torch.cat([eps, var], 1).contiguous()


def test_pipeline_loop_matches_reference_2b_loop(ops):
    from paddlemix_b200.opensora import IDDPM, OpenSoraPipeline
    from paddlemix_b200.sampling import seed_from
    B, L, T, H, W = 2, 12, 3, 64, 96
    g = torch.Generator().manual_seed(11)
    prompt = torch.randn(B, 1, L, 16, generator=g).to(bf16).float()
    null = torch.randn(L, 16, generator=g).to(bf16).float()
    mask = torch.ones(B, L, dtype=torch.long)
    mask[1, 7:] = 0
    lat = torch.randn(B, 4, T, H // 8, W // 8, generator=g)
    stub = StubSTDiT2(B, null.cuda(), prompt.cuda(), mask.cuda())
    pipe = OpenSoraPipeline(stub, IDDPM(num_sampling_steps=10, cfg_scale=7.0, cfg_channel=3))
    out = pipe(prompt.cuda(), prompt_attention_mask=mask, num_frames=T, height=H, width=W, latents=lat,
               generator=torch.Generator().manual_seed(12))
    assert stub.calls == 10 and out.shape == lat.shape and out.dtype == torch.float32
    seed = seed_from(torch.Generator().manual_seed(12))
    ref = O.sample_2b(O.Diffusion(1000, "10"), stub, lat, prompt, null[None, None].repeat(B, 1, 1, 1), 7.0, 3,
                      O.philox_noise_fn(seed))
    err = (out.cpu() - ref).abs().max().item() / ref.abs().max().item()
    print(f"stub loop: max rel err {err:.3g}")
    assert err <= 1e-6


# ---- the real model --------------------------------------------------------------------------------------------------
REAL_L2, REAL_MAX_RMS = 4e-2, 0.2


@pytest.mark.slow
def test_pipeline_stdit2_xl_depth2_vs_oracle(ops):
    from oracle import stdit2 as OS
    from paddlemix_b200.opensora import IDDPM, STDiT2, OpenSoraPipeline
    from paddlemix_b200.sampling import seed_from
    cfg = dict(OS.STDIT2_CONFIGS["stdit2_xl"])
    cfg["depth"] = 2
    P = OS.init_stdit2_params(cfg, seed=3)
    g = torch.Generator().manual_seed(13)
    P["y_embedder.y_embedding"] = (torch.randn(120, 4096, generator=g) / 4096 ** 0.5).to(bf16).float()
    model = STDiT2(cfg).load_state_dict(P, device=0)
    B, T, H, W = 2, 4, 128, 192
    prompt = torch.randn(B, 1, 120, 4096, generator=g).to(bf16).float()
    mask = torch.zeros(B, 120, dtype=torch.long)
    mask[0, :120], mask[1, :57] = 1, 1
    lat = torch.randn(B, 4, T, H // 8, W // 8, generator=g)
    sched = IDDPM(num_sampling_steps=3, cfg_scale=7.0, cfg_channel=3)
    out = OpenSoraPipeline(model, sched)(prompt, prompt_attention_mask=mask, num_frames=T, height=H, width=W, fps=24,
                                         latents=lat, generator=torch.Generator().manual_seed(14))
    seed = seed_from(torch.Generator().manual_seed(14))
    Pd = {k: v.cuda() for k, v in P.items()}
    sizes = {k: torch.full((2 * B,), v, device="cuda") for k, v in
             dict(num_frames=float(T), height=float(H), width=float(W), ar=H / W, fps=24.0).items()}
    m2 = mask.cuda().repeat(2, 1)

    def oracle_model(x, t, y):
        return OS.stdit2_forward(cfg, Pd, x, t.float(), y, m2, **sizes)
    noise = O.philox_noise_fn(seed)
    with torch.device("cuda"), torch.no_grad():
        ref = O.sample_2b(O.Diffusion(1000, "3"), oracle_model, lat.cuda(), prompt.cuda(),
                          Pd["y_embedder.y_embedding"][None, None].repeat(B, 1, 1, 1), 7.0, 3,
                          lambda i, shape: noise(i, shape).cuda())
    d = (out.double() - ref.double())
    l2 = (d.norm() / ref.double().norm()).item()
    mx = (d.abs().max() / ref.double().pow(2).mean().sqrt()).item()
    print(f"stdit2-xl depth 2, 3 steps: normwise {l2:.4g}, max {mx:.4g} rms")
    assert bool(torch.isfinite(out).all()) and l2 <= REAL_L2 and mx <= REAL_MAX_RMS, (l2, mx)


# ---- the video VAE ---------------------------------------------------------------------------------------------------
def test_video_vae_decode_and_pipeline_pt(ops):
    from oracle import vae as OV
    from paddlemix_b200.opensora import IDDPM, OpenSoraPipeline, VideoAutoencoderKL
    from paddlemix_b200.ppdiffusers.autoencoder_kl import AutoencoderKL
    vcfg = OV.VAE_CONFIGS["tiny"]
    keys = ("latent_channels", "out_channels", "block_out_channels", "layers_per_block", "norm_num_groups", "scaling_factor")
    vae = AutoencoderKL(**{k: vcfg[k] for k in keys}).load_state_dict(OV.init_vae_params(vcfg, seed=2), device=0)
    up = 2 ** (len(vcfg["block_out_channels"]) - 1)
    B, T, h, w = 2, 3, 8, 12
    z = torch.randn(B, 4, T, h, w, generator=torch.Generator().manual_seed(3)).cuda()
    frames = ops.scale_model_input(z.permute(0, 2, 1, 3, 4).reshape(B * T, 4, h, w).contiguous(), 0.18215)
    outs = {}
    for mb in (1, 4, None):
        v = VideoAutoencoderKL(vae, micro_batch_size=mb).decode(z)
        assert v.shape == (B, 3, T, h * up, w * up) and v.dtype == torch.float32
        bs = B * T if mb is None else mb
        ref = torch.cat([vae.decode(frames[i:i + bs]).sample for i in range(0, B * T, bs)])
        assert torch.equal(v, ref.reshape(B, T, 3, h * up, w * up).permute(0, 2, 1, 3, 4))
        outs[mb] = v
    for mb in (4, None):
        a, b = outs[mb].flatten().double(), outs[1].flatten().double()
        cos = torch.nn.functional.cosine_similarity(a, b, dim=0).item()
        assert cos >= 0.999 and (a - b).abs().max().item() <= 0.04 * b.abs().max().item()
    # output_type="pt" decodes the loop's latents
    L = 4
    prompt = torch.randn(B, 1, L, 16, generator=torch.Generator().manual_seed(4)).to(bf16).float().cuda()
    null = torch.randn(L, 16, generator=torch.Generator().manual_seed(5)).to(bf16).float().cuda()
    stub = StubSTDiT2(B, null, prompt, None)
    pipe = OpenSoraPipeline(stub, IDDPM(num_sampling_steps=4), vae=VideoAutoencoderKL(vae, micro_batch_size=2))
    kw = dict(num_frames=T, height=8 * h, width=8 * w, latents=z.cpu())
    lat = pipe(prompt, generator=torch.Generator().manual_seed(6), **kw)
    vid = pipe(prompt, generator=torch.Generator().manual_seed(6), output_type="pt", **kw)
    assert torch.equal(vid, VideoAutoencoderKL(vae, micro_batch_size=2).decode(lat))
