"""T2I-Adapter on the GPU: the pixel-unshuffle, 2x2 average-pool, weighted-sum and ReLU kernels against torch,
T2IAdapter / MultiAdapter against the CPU fp32 oracle (tiny and production geometry), and the adapter pipeline (graphed
vs eager, oracle loop, adapter_conditioning_factor, determinism).

Model tolerances are those of test_unet_gpu.py (cosine >= 0.999, max |err| <= 4 % of the output's max magnitude)."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from oracle import adapter as OA
from oracle import unet as O

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16


# ---------------------------------------------------------------------------------------------------------------------
# kernels
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("f", [8, 16])
@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("dtype", [torch.float32, bf16])
@pytest.mark.parametrize("B", [1, 3, 8])
def test_pixel_unshuffle_bit_exact(f, C, dtype, B):
    from paddlemix_b200 import ops
    g = torch.Generator().manual_seed(f * 100 + C * 10 + B)
    H, W = f * 5, f * 3  # H != W
    x = torch.rand(B, C, H, W, generator=g).to(dtype)
    y = ops.pixel_unshuffle(x.cuda(), f)
    ref = F.pixel_unshuffle(x.float(), f).to(bf16).permute(0, 2, 3, 1)
    assert y.shape == (B, H // f, W // f, C * f * f) and y.dtype == bf16
    assert torch.equal(y.cpu(), ref)


@pytest.mark.parametrize("H,W", [(8, 8), (7, 9), (1, 1), (33, 64), (5, 2)])
@pytest.mark.parametrize("C", [8, 320])
def test_avgpool2x2_matches_avg_pool2d(H, W, C):
    from paddlemix_b200 import ops
    g = torch.Generator().manual_seed(H * 1000 + W * 10 + C)
    x = torch.randn(2, H, W, C, generator=g).to(bf16)
    y = ops.avgpool2x2_nhwc(x.cuda()).cpu()
    ref = F.avg_pool2d(x.float().permute(0, 3, 1, 2), 2, 2, ceil_mode=True, count_include_pad=False).permute(0, 2, 3, 1)
    assert y.shape == ref.shape
    # within one bf16 rounding of the fp32 average
    assert ((y.float() - ref).abs() <= ref.abs() * 2.0 ** -8 + 1e-30).all()


def test_weighted_sum_rows_tiles_and_rounds_once():
    from paddlemix_b200 import ops
    g = torch.Generator().manual_seed(3)
    a = torch.randn(2, 4, 6, 16, generator=g).to(bf16)
    b = torch.randn(1, 4, 6, 16, generator=g).to(bf16)
    out = torch.full((4, 4, 6, 16), float("nan"), dtype=bf16, device="cuda")
    ops.weighted_sum_rows([a.cuda(), b.cuda()], [0.3, 1.7], out=out)
    rows = torch.arange(4)
    ref = (torch.tensor(0.3) * a.float()[rows % 2] + torch.tensor(1.7) * b.float()[rows % 1]).to(bf16)
    assert torch.equal(out.cpu(), ref)


def test_relu_activation_bit_exact():
    from paddlemix_b200 import ops
    from paddlemix_b200._lib import ACT_RELU
    x = torch.randn(3, 1000, generator=torch.Generator().manual_seed(1))
    for dtype in (torch.float32, bf16):
        xd = x.to(dtype)
        for out_dtype in (None, torch.float32, bf16):
            y = ops.activation(xd.cuda(), ACT_RELU, out_dtype=out_dtype).cpu()
            assert torch.equal(y, torch.relu(xd).to(out_dtype or dtype))


def test_new_entry_points_refuse_bad_arguments():
    """Each bad argument is rejected on the host with B200MIX_ERR_INVALID and a message; no kernel is launched."""
    from paddlemix_b200 import _lib, ops
    lib = _lib.lib
    ops.init(0)
    x = torch.zeros(2, 3, 64, 64, device="cuda")
    y = torch.zeros(2 * 3 * 64 * 64 + 8, device="cuda", dtype=bf16)
    p = lambda t, off=0: ctypes.c_void_p(t.data_ptr() + off)  # noqa: E731
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    good = dict(x=p(x), fp32=1, y=p(y), B=2, C=3, H=64, W=64, f=8)
    for change in [dict(x=None), dict(y=None), dict(x=p(x, 4)), dict(y=p(y, 2)), dict(f=4), dict(f=32), dict(H=60),
                   dict(W=72 - 4), dict(B=0), dict(C=0)]:
        a = {**good, **change}
        rc = lib.b200mix_pixel_unshuffle(a["x"], a["fp32"], a["y"], a["B"], a["C"], a["H"], a["W"], a["f"], st)
        assert rc == -1 and b"pixel_unshuffle" in lib.b200mix_last_error(), change
    good = dict(x=p(y), y=p(x), B=1, H=8, W=8, C=64)
    for change in [dict(x=None), dict(y=None), dict(C=12), dict(C=0), dict(H=0), dict(x=p(y, 2))]:
        a = {**good, **change}
        rc = lib.b200mix_avgpool2x2_nhwc(a["x"], a["y"], a["B"], a["H"], a["W"], a["C"], st)
        assert rc == -1 and b"avgpool2x2_nhwc" in lib.b200mix_last_error(), change
    src = torch.zeros(4, 64, device="cuda", dtype=bf16)
    dst = torch.zeros(8, 64, device="cuda", dtype=bf16)

    def wsum(n=1, ptrs=None, rows=4, w=1.0, out=None, rows_out=8, row=64):
        P = (ctypes.c_void_p * max(n, 1))(*([ptrs or src.data_ptr()] * max(n, 1)))
        R = (ctypes.c_int64 * max(n, 1))(*([rows] * max(n, 1)))
        Wt = (ctypes.c_float * max(n, 1))(*([w] * max(n, 1)))
        return lib.b200mix_weighted_sum_rows(n, P, R, Wt, out or p(dst), rows_out, row, st)

    for kw in [dict(n=0), dict(n=9), dict(rows=0), dict(row=60), dict(rows_out=0), dict(out=p(dst, 2)),
               dict(out=p(src)), dict(ptrs=src.data_ptr() + 2)]:
        assert wsum(**kw) == -1 and b"weighted_sum_rows" in lib.b200mix_last_error(), kw
    h = torch.zeros(16, device="cuda", dtype=bf16)
    assert lib.b200mix_activation(p(h), p(h), 16, 6, 0, 0, st) == -1
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------------
# models
# ---------------------------------------------------------------------------------------------------------------------
def make_adapter(name, seed=1, **kw):
    from paddlemix_b200.ppdiffusers.adapter import T2IAdapter
    cfg = {**OA.ADAPTER_CONFIGS[name], **kw}
    P = O.init_params(OA.adapter_param_shapes(cfg), seed=seed)
    return cfg, P, T2IAdapter(**cfg).load_state_dict(P, device=0)


def image(cfg, B, H, W, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(B, cfg["in_channels"], H, W, generator=g)


def compare(out, ref, what):
    out, ref = out.float().cpu(), ref.float()
    cos = F.cosine_similarity(out.flatten(), ref.flatten(), dim=0).item()
    err = (out - ref).abs().max().item()
    scale = ref.abs().max().item()
    assert cos >= 0.999, f"{what}: cosine {cos}"
    assert err <= 0.04 * scale, f"{what}: max err {err} vs scale {scale}"


def compare_features(feats, refs, what):
    assert len(feats) == len(refs)
    for k, (f, r) in enumerate(zip(feats, refs)):
        assert f.dtype == bf16 and tuple(f.permute(0, 3, 1, 2).shape) == tuple(r.shape), (what, k)
        compare(f.permute(0, 3, 1, 2), r, f"{what} feature {k}")


@pytest.mark.parametrize("name,B,H,W", [("tiny_sd", 2, 128, 96), ("tiny_xl", 2, 128, 160), ("tiny_sd_light", 2, 72, 136),
                                        ("sd15_light", 1, 136, 200)])
def test_adapter_vs_oracle(name, B, H, W):
    """Odd sizes along the way (72 / 8 = 9 -> 5 -> 3) exercise the pool's partial windows."""
    cfg, P, adapter = make_adapter(name)
    img = image(cfg, B, H, W)
    compare_features(adapter(img.cuda()), OA.adapter_forward(cfg, P, img), name)


def test_light_adapter_padding_is_exact():
    """The padded device model equals the unpadded oracle; the padded channels never reach the features."""
    cfg, P, adapter = make_adapter("sd15_light", seed=4)
    assert adapter.blocks[0].resnets[0][0].w.shape[0] == 128
    img = image(cfg, 2, 64, 64, seed=2)
    compare_features(adapter(img.cuda()), OA.adapter_forward(cfg, P, img), "light adapter (80 -> 128 padded)")


def test_multi_adapter_vs_oracle():
    from paddlemix_b200.ppdiffusers.adapter import MultiAdapter
    cfg, P1, a1 = make_adapter("tiny_xl", seed=1)
    _, P2, a2 = make_adapter("tiny_xl", seed=2)
    i1, i2 = image(cfg, 2, 128, 128, seed=1), image(cfg, 1, 128, 128, seed=2)
    multi = MultiAdapter([a1, a2])
    for w in (None, [0.7, 1.3]):
        compare_features(multi([i1.cuda(), i2.cuda()], w), OA.multi_adapter_forward([cfg, cfg], [P1, P2], [i1, i2], w),
                         f"multi-adapter weights {w}")


@pytest.mark.slow
@pytest.mark.parametrize("name,B,H", [("sd15", 2, 512), ("sdxl", 1, 1024)])
def test_adapter_production_geometry_vs_oracle(name, B, H):
    cfg, P, adapter = make_adapter(name)
    img = image(cfg, B, H, H)
    compare_features(adapter(img.cuda()), OA.adapter_forward(cfg, P, img), f"{name} {H}x{H} B={B}")


UNET_KEYS = ("in_channels", "out_channels", "down_block_types", "up_block_types", "block_out_channels",
             "layers_per_block", "cross_attention_dim", "transformer_layers_per_block", "attention_head_dim",
             "use_linear_projection", "addition_embed_type", "addition_time_embed_dim",
             "projection_class_embeddings_input_dim", "resnet_out_scale_factor")


def make_unet(name, seed=11):
    from paddlemix_b200.ppdiffusers.unet_2d_condition import UNet2DConditionModel
    cfg = O.UNET_CONFIGS[name]
    P = O.init_params(O.unet_param_shapes(cfg), seed=seed)
    return cfg, P, UNet2DConditionModel(**{k: cfg[k] for k in UNET_KEYS}).load_state_dict(P, device=0)


def unet_inputs(cfg, B, H, L, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, cfg["in_channels"], H, H, generator=g).to(bf16).float()
    ctx = torch.randn(B, L, cfg["cross_attention_dim"], generator=g).to(bf16).float()
    added = None
    if cfg["addition_embed_type"] == "text_time":
        n_text = cfg["projection_class_embeddings_input_dim"] - 6 * cfg["addition_time_embed_dim"]
        added = {"text_embeds": torch.randn(B, n_text, generator=g).to(bf16).float(),
                 "time_ids": torch.tensor([[H * 8., H * 8., 0, 0, H * 8., H * 8.]] * B)}
    return x, ctx, added


def cuda(d):
    return None if d is None else {k: v.cuda() for k, v in d.items()}


@pytest.mark.slow
def test_sdxl_unet_step_with_adapter_xl_vs_oracle():
    """One SDXL 1024^2 UNet step with FullAdapterXL residuals, adapter and UNet on the device, against the oracle."""
    acfg, aP, adapter = make_adapter("sdxl")
    ucfg, uP, unet = make_unet("sdxl")
    x, ctx, added = unet_inputs(ucfg, 1, 128, 77)
    img = image(acfg, 1, 1024, 1024)
    feats = adapter(img.cuda())
    ref_feats = OA.adapter_forward(acfg, aP, img)
    out = unet.forward_nhwc(x.permute(0, 2, 3, 1).contiguous().cuda(), 701, ctx.to(bf16).cuda(), cuda(added),
                            down_intrablock_additional_residuals=feats, residuals_nchw=False)
    ref = O.unet_forward(ucfg, uP, x, 701, ctx, added, down_intrablock_additional_residuals=ref_feats)
    compare(out.permute(0, 3, 1, 2), ref, "SDXL 1024^2 UNet step with FullAdapterXL residuals")


# ---------------------------------------------------------------------------------------------------------------------
# pipeline
# ---------------------------------------------------------------------------------------------------------------------
SD = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False, set_alpha_to_one=False,
          steps_offset=1)
ADAPTER_FOR = {"tiny_sd": "tiny_sd", "tiny_xl": "tiny_xl"}


def oracle_loop(ucfg, uP, acfgs, aPs, x, ctx, neg, imgs, added, steps, gs, scale, factor):
    """pipeline_stable_diffusion_adapter.py:823-870 (+ the SDXL factor cut-off) on the fp32 oracle models."""
    from oracle.schedulers import DDIMScheduler as ODDIM
    sch = ODDIM(**SD)
    sch.set_timesteps(steps)
    B = x.shape[0]
    do_cfg = gs > 1.0
    if len(acfgs) > 1:
        state = OA.pipeline_residuals(OA.multi_adapter_forward(acfgs, aPs, imgs, scale), 1.0, B, do_cfg)
    else:
        state = OA.pipeline_residuals(OA.adapter_forward(acfgs[0], aPs[0], imgs[0]), scale, B, do_cfg)
    on = OA.residual_steps(steps, factor)
    added2 = added if (added is None or not do_cfg) else {k: torch.cat([v, v], 0) for k, v in added.items()}
    cur = x.clone()
    for i, t in enumerate(sch.timesteps):
        model_in = torch.cat([cur, cur]) if do_cfg else cur
        c = torch.cat([neg, ctx]) if do_cfg else ctx
        eps = O.unet_forward(ucfg, uP, model_in, int(t), c, added2,
                             down_intrablock_additional_residuals=[s.clone() for s in state] if on[i] else None)
        if do_cfg:
            eu, ec = eps.chunk(2)
            eps = eu + gs * (ec - eu)
        cur = sch.step(eps, t, cur)
    return cur


@pytest.mark.parametrize("name", ["tiny_sd", "tiny_xl"])
@pytest.mark.parametrize("n_adapters,gs", [(1, 5.0), (1, 1.0), (2, 5.0), (2, 1.0)])
def test_adapter_pipeline_graphed_eager_oracle(name, n_adapters, gs):
    from paddlemix_b200.ppdiffusers.pipelines import StableDiffusionAdapterPipeline
    from paddlemix_b200.ppdiffusers.schedulers import DDIMScheduler
    ucfg, uP, unet = make_unet(name)
    ads = [make_adapter(ADAPTER_FOR[name], seed=1 + k) for k in range(n_adapters)]
    B, H = 2, 16
    x, ctx, added = unet_inputs(ucfg, B, H, 20)
    imgs = [image(ads[0][0], B if k == 0 else 1, 8 * H, 8 * H, seed=k) for k in range(n_adapters)]
    neg = torch.zeros_like(ctx)
    steps = 4
    scale = 0.8 if n_adapters == 1 else [0.6, 0.9]
    adapter = ads[0][2] if n_adapters == 1 else [a[2] for a in ads]
    kw = dict(prompt_embeds=ctx, negative_prompt_embeds=neg, latents=x, num_inference_steps=steps, guidance_scale=gs,
              added_cond_kwargs=added, image=imgs[0] if n_adapters == 1 else imgs, adapter_conditioning_scale=scale)
    lat = {}
    for graph in (True, False):
        pipe = StableDiffusionAdapterPipeline(unet, adapter, DDIMScheduler(**SD), use_cuda_graph=graph)
        lat[graph] = pipe(**kw).cpu()
        assert torch.equal(pipe(**kw).cpu(), lat[graph]), "two calls with the same inputs must agree bit for bit"
    assert torch.equal(lat[True], lat[False])
    ref = oracle_loop(ucfg, uP, [a[0] for a in ads], [a[1] for a in ads], x, ctx, neg, imgs, added, steps, gs, scale, 1.0)
    compare(lat[True], ref, f"{steps}-step adapter DDIM loop ({name}, adapters={n_adapters}, g={gs})")
    plain = oracle_loop(ucfg, uP, [a[0] for a in ads], [a[1] for a in ads], x, ctx, neg, imgs, added, steps, gs, scale,
                        0.0)
    assert (lat[True] - plain).abs().max() > 1e-2 * plain.abs().max(), "the residuals must change the result"


@pytest.mark.parametrize("name", ["tiny_sd", "tiny_xl"])
def test_adapter_pipeline_factor(name):
    """factor 0 equals StableDiffusionPipeline bit for bit (bf16 h + 0 == h); factor 0.5 matches the oracle loop that
    drops the residuals at the same step."""
    from paddlemix_b200.ppdiffusers.pipelines import StableDiffusionAdapterPipeline, StableDiffusionPipeline
    from paddlemix_b200.ppdiffusers.schedulers import DDIMScheduler
    ucfg, uP, unet = make_unet(name)
    acfg, aP, adapter = make_adapter(ADAPTER_FOR[name])
    x, ctx, added = unet_inputs(ucfg, 2, 16, 20)
    img = image(acfg, 1, 128, 128)
    kw = dict(prompt_embeds=ctx, latents=x, num_inference_steps=4, guidance_scale=4.0, added_cond_kwargs=added)
    for graph in (True, False):
        plain = StableDiffusionPipeline(unet, DDIMScheduler(**SD), use_cuda_graph=graph)(**kw)
        pipe = StableDiffusionAdapterPipeline(unet, adapter, DDIMScheduler(**SD), use_cuda_graph=graph)
        assert torch.equal(pipe(image=img, adapter_conditioning_factor=0.0, **kw), plain)
        half = pipe(image=img, adapter_conditioning_factor=0.5, **kw).cpu()
        full = pipe(image=img, **kw).cpu()
        assert not torch.equal(half, full)
        ref = oracle_loop(ucfg, uP, [acfg], [aP], x, ctx, torch.zeros_like(ctx), [img], added, 4, 4.0, 1.0, 0.5)
        compare(half, ref, f"{name} factor 0.5 (graph={graph})")


def test_graphed_unet_without_adapter_is_unchanged():
    """Constructed without intrablock buffers, GraphedUNet captures exactly the plain UNet: same launches and output."""
    from paddlemix_b200.ppdiffusers.pipelines import GraphedUNet
    ucfg, uP, unet = make_unet("tiny_xl")
    x, ctx, added = unet_inputs(ucfg, 2, 16, 20)
    acfg, aP, adapter = make_adapter("tiny_xl")
    plain = GraphedUNet(unet, tuple(x.shape), tuple(ctx.shape), {k: v.shape for k, v in added.items()})
    bufs = [torch.zeros((2,) + f.shape[1:], device="cuda", dtype=bf16) for f in adapter(image(acfg, 1, 128, 128).cuda())]
    with_ad = GraphedUNet(unet, tuple(x.shape), tuple(ctx.shape), {k: v.shape for k, v in added.items()},
                          intrablock_residuals=bufs)
    assert with_ad.launches_per_replay == plain.launches_per_replay + len(bufs)
    y = plain(x.cuda(), 301, ctx.to(bf16).cuda(), cuda(added)).clone()
    eager = unet(x.cuda(), 301, ctx.cuda(), added_cond_kwargs=cuda(added)).sample
    assert torch.equal(y, eager)
    assert torch.equal(with_ad(x.cuda(), 301, ctx.to(bf16).cuda(), cuda(added)), y)  # zero residuals change nothing
