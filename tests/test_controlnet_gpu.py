"""ControlNet on the GPU: the narrow-channel conv3x3 kernel against torch's fp32 conv2d, ControlNetModel /
MultiControlNetModel against the CPU fp32 oracle, and the ControlNet pipeline (graphed vs eager, oracle loop,
keep = 0 vs no ControlNet, determinism).

Model tolerances are those of test_unet_gpu.py (cosine >= 0.999, max |err| <= 4 % of the output's max magnitude)."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from oracle import controlnet as OC
from oracle import unet as O

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16


# ---------------------------------------------------------------------------------------------------------------------
# kernel
# ---------------------------------------------------------------------------------------------------------------------
NARROW_CASES = [(cin, cout, s, act) for cin, cout in ((3, 16), (16, 16), (16, 32), (32, 96), (96, 96), (96, 256),
                                                       (32, 256), (3, 96))
                for s in (1, 2) for act in (0, 1)]


@pytest.mark.parametrize("cin,cout,stride,act", NARROW_CASES)
def test_conv3x3_narrow_matches_conv2d(cin, cout, stride, act):
    from paddlemix_b200 import ops
    g = torch.Generator().manual_seed(cin * 1000 + cout + 7 * stride + act)
    B, H, W = 2, 38, 52  # H != W, neither a multiple of the 8 x 16 output tile
    x = torch.randn(B, H, W, cin, generator=g).to(bf16)
    w = (torch.randn(cout, 3, 3, cin, generator=g) / (9 * cin) ** 0.5).to(bf16)
    b = 0.1 * torch.randn(cout, generator=g)
    y = ops.conv3x3_narrow(x.cuda(), w.cuda(), b.cuda(), stride=stride, act=act)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2), b, stride=stride, padding=1)
    if act:
        ref = F.silu(ref)
    ref = ref.permute(0, 2, 3, 1)
    assert y.shape == ref.shape and y.dtype == bf16
    rng = (ref.max() - ref.min()).item()
    err = (y.float().cpu() - ref).abs().max().item()
    assert err <= 1e-2 * rng, (err, rng)


def test_conv3x3_narrow_no_bias_and_unaligned_input():
    # bias NULL; an input view starting 2 elements into its buffer takes the scalar staging path
    from paddlemix_b200 import ops
    g = torch.Generator().manual_seed(5)
    buf = torch.randn(2 + 1 * 20 * 24 * 16, generator=g).to(bf16)
    x = buf[2:].reshape(1, 20, 24, 16)
    w = (torch.randn(32, 3, 3, 16, generator=g) / 12).to(bf16)
    y = ops.conv3x3_narrow(buf.cuda()[2:].reshape(1, 20, 24, 16), w.cuda(), None, stride=2)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2), None, stride=2, padding=1)
    ref = ref.permute(0, 2, 3, 1)
    assert (y.float().cpu() - ref).abs().max().item() <= 1e-2 * (ref.max() - ref.min()).item()


def test_conv3x3_narrow_invalid_arguments():
    """Each bad argument is rejected on the host with B200MIX_ERR_INVALID and a message; no kernel is launched."""
    from paddlemix_b200 import _lib, ops
    lib = _lib.lib
    ops.init(0)
    x = torch.zeros(1, 8, 8, 128, device="cuda", dtype=bf16)
    w = torch.zeros(256, 3, 3, 128, device="cuda", dtype=bf16)
    y = torch.zeros(1, 8, 8, 256, device="cuda", dtype=bf16)
    p = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    good = dict(x=p(x), w=p(w), b=None, y=p(y), B=1, H=8, W=8, Cin=16, Cout=16, stride=1, act=0)
    bad = [dict(x=None), dict(w=None), dict(y=None), dict(Cin=0), dict(Cin=129), dict(Cout=12), dict(Cout=264),
           dict(Cout=0), dict(stride=3), dict(act=2), dict(H=7, stride=2), dict(W=9, stride=2), dict(B=0)]
    for change in bad:
        a = {**good, **change}
        rc = lib.b200mix_conv3x3_narrow(a["x"], a["w"], a["b"], a["y"], a["B"], a["H"], a["W"], a["Cin"], a["Cout"],
                                        a["stride"], a["act"], st)
        assert rc == -1, (change, rc)
        assert b"conv3x3_narrow" in lib.b200mix_last_error()
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------------
# models
# ---------------------------------------------------------------------------------------------------------------------
CN_KEYS = ("in_channels", "flip_sin_to_cos", "freq_shift", "down_block_types", "block_out_channels",
           "layers_per_block", "norm_num_groups", "norm_eps", "cross_attention_dim", "transformer_layers_per_block",
           "attention_head_dim", "use_linear_projection", "addition_embed_type", "addition_time_embed_dim",
           "projection_class_embeddings_input_dim")


def make_cn(name, seed=1, data_format="NCHW", **kw):
    from paddlemix_b200.ppdiffusers.controlnet import ControlNetModel
    cfg = {**O.UNET_CONFIGS[name], **kw}
    P = O.init_params(OC.controlnet_param_shapes(cfg), seed=seed)
    extra = {k: cfg[k] for k in ("controlnet_conditioning_channel_order",) if k in cfg}
    model = ControlNetModel(**{k: cfg[k] for k in CN_KEYS}, **extra, data_format=data_format)
    return cfg, P, model.load_state_dict(P, device=0)


def make_unet(name, seed=11):
    from paddlemix_b200.ppdiffusers.unet_2d_condition import UNet2DConditionModel
    cfg = O.UNET_CONFIGS[name]
    P = O.init_params(O.unet_param_shapes(cfg), seed=seed)
    keys = CN_KEYS + ("out_channels", "up_block_types", "resnet_out_scale_factor")
    return cfg, P, UNet2DConditionModel(**{k: cfg[k] for k in keys}).load_state_dict(P, device=0)


def inputs(cfg, B, H, L, seed=0, img_scale=8):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, cfg["in_channels"], H, H, generator=g).to(bf16).float()
    ctx = torch.randn(B, L, cfg["cross_attention_dim"], generator=g).to(bf16).float()
    img = torch.rand(B, 3, H * img_scale, H * img_scale, generator=g).to(bf16).float()
    added = None
    if cfg["addition_embed_type"] == "text_time":
        n_text = cfg["projection_class_embeddings_input_dim"] - 6 * cfg["addition_time_embed_dim"]
        added = {"text_embeds": torch.randn(B, n_text, generator=g).to(bf16).float(),
                 "time_ids": torch.tensor([[H * 8., H * 8., 0, 0, H * 8., H * 8.]] * B)}
    return x, ctx, img, added


def compare(out, ref, what):
    out, ref = out.float().cpu(), ref.float()
    cos = torch.nn.functional.cosine_similarity(out.flatten(), ref.flatten(), dim=0).item()
    err = (out - ref).abs().max().item()
    scale = ref.abs().max().item()
    assert cos >= 0.999, f"{what}: cosine {cos}"
    assert err <= 0.04 * scale, f"{what}: max err {err} vs scale {scale}"


def cuda(d):
    return None if d is None else {k: v.cuda() for k, v in d.items()}


def compare_residuals(out, ref_down, ref_mid, nhwc, what):
    down, mid = out
    assert len(down) == len(ref_down)
    for k, (d, r) in enumerate(zip((*down, mid), (*ref_down, ref_mid))):
        assert d.dtype == bf16
        compare(d.permute(0, 3, 1, 2) if nhwc else d, r, f"{what} residual {k}")


@pytest.mark.parametrize("name,scale,guess,order,nhwc", [
    ("tiny_sd", 1.0, False, "rgb", False), ("tiny_xl", 0.7, False, "rgb", False), ("tiny_sd", "list", False, "bgr", False),
    ("tiny_xl", 0.8, True, "rgb", True), ("tiny_sd", 0.5, True, "bgr", True), ("tiny_xl", "list", False, "bgr", True)])
def test_controlnet_model_vs_oracle(name, scale, guess, order, nhwc):
    cfg, P, model = make_cn(name, controlnet_conditioning_channel_order=order,
                            data_format="NHWC" if nhwc else "NCHW")
    B, H = 2, 16
    x, ctx, img, added = inputs(cfg, B, H, 20)
    if scale == "list":
        scale = [0.3 + 0.1 * k for k in range(model.num_residuals)]
    ref_down, ref_mid = OC.controlnet_forward(cfg, P, x, 481, ctx, img, scale, added, guess_mode=guess)
    xs, im = (x.permute(0, 2, 3, 1).contiguous(), img.permute(0, 2, 3, 1).contiguous()) if nhwc else (x, img)
    out = model(xs.cuda(), 481, ctx.cuda(), im.cuda(), conditioning_scale=scale, added_cond_kwargs=cuda(added),
                guess_mode=guess)
    compare_residuals(tuple(out), ref_down, ref_mid, nhwc, f"{name} {order} guess={guess}")
    down, mid = model(xs.cuda(), 481, ctx.cuda(), im.cuda(), conditioning_scale=scale, added_cond_kwargs=cuda(added),
                      guess_mode=guess, return_dict=False)
    assert all(torch.equal(a, b) for a, b in zip((*down, mid), (*out.down_block_res_samples, out.mid_block_res_sample)))


def test_conditioning_embedding_vs_oracle():
    from paddlemix_b200 import ops
    cfg, P, model = make_cn("tiny_xl")
    _, _, img, _ = inputs(cfg, 2, 16, 8)
    e = model.embed_condition(ops.nchw_to_nhwc(img.cuda()))
    compare(e.permute(0, 3, 1, 2), OC.conditioning_embedding(cfg, P, img), "conditioning embedding")


def test_multi_controlnet_vs_oracle():
    from paddlemix_b200.ppdiffusers.controlnet import MultiControlNetModel
    cfg, P1, n1 = make_cn("tiny_xl", seed=1)
    _, P2, n2 = make_cn("tiny_xl", seed=2)
    B, H = 2, 16
    x, ctx, img1, added = inputs(cfg, B, H, 20)
    img2 = torch.rand(B, 3, H * 8, H * 8, generator=torch.Generator().manual_seed(9)).to(bf16).float()
    scales = [0.6, 1.1]
    ref_down, ref_mid = OC.multi_controlnet_forward([cfg, cfg], [P1, P2], x, 301, ctx, [img1, img2], scales, added)
    multi = MultiControlNetModel([n1, n2])
    out = multi(x.cuda(), 301, ctx.cuda(), [img1.cuda(), img2.cuda()], scales, added_cond_kwargs=cuda(added))
    compare_residuals(tuple(out), ref_down, ref_mid, False, "multi-controlnet")


@pytest.mark.slow
@pytest.mark.parametrize("name,H", [("sd15", 64), ("sdxl", 128)])
def test_controlnet_full_size_vs_oracle(name, H):
    cfg, P, model = make_cn(name)
    x, ctx, img, added = inputs(cfg, 1, H, 77)
    ref_down, ref_mid = OC.controlnet_forward(cfg, P, x, 701, ctx, img, 1.0, added)
    out = model(x.cuda(), 701, ctx.cuda(), img.cuda(), added_cond_kwargs=cuda(added), return_dict=False)
    compare_residuals(out, ref_down, ref_mid, False, f"{name} full size")


# ---------------------------------------------------------------------------------------------------------------------
# pipeline
# ---------------------------------------------------------------------------------------------------------------------
SD = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False, set_alpha_to_one=False,
          steps_offset=1)


def oracle_loop(ucfg, uP, cn_cfgs, cn_Ps, x, ctx, neg, imgs, added, steps, gs, scales, start, end, guess):
    """pipeline_controlnet.py:1047-1130 restated on the fp32 oracle models + the fp32 DDIM oracle."""
    from oracle.schedulers import DDIMScheduler as ODDIM
    sch = ODDIM(**SD)
    sch.set_timesteps(steps)
    multi = len(cn_cfgs) > 1
    keep = OC.controlnet_keep(steps, start, end, multi)
    add2 = None if added is None else {k: torch.cat([v, v], 0) for k, v in added.items()}
    cur = x.clone()
    for i, t in enumerate(sch.timesteps):
        cond_scale = OC.step_conditioning_scale(scales if multi else scales[0], keep[i])
        cond_scale = cond_scale if multi else [cond_scale]
        if guess:
            down, mid = OC.multi_controlnet_forward(cn_cfgs, cn_Ps, cur, int(t), ctx, imgs, cond_scale, added, True)
            down = [torch.cat([torch.zeros_like(d), d]) for d in down]
            mid = torch.cat([torch.zeros_like(mid), mid])
        else:
            down, mid = OC.multi_controlnet_forward(cn_cfgs, cn_Ps, torch.cat([cur, cur]), int(t), torch.cat([neg, ctx]),
                                                    [torch.cat([im, im]) for im in imgs], cond_scale, add2)
        eps = O.unet_forward(ucfg, uP, torch.cat([cur, cur], 0), int(t), torch.cat([neg, ctx], 0), add2,
                             down_block_additional_residuals=down, mid_block_additional_residual=mid)
        eu, ec = eps.chunk(2)
        cur = sch.step(eu + gs * (ec - eu), t, cur)
    return cur


@pytest.mark.parametrize("n_nets,guess", [(1, False), (1, True), (2, False)])
def test_controlnet_pipeline_graphed_eager_oracle(n_nets, guess):
    from paddlemix_b200.ppdiffusers.pipelines import StableDiffusionControlNetPipeline
    from paddlemix_b200.ppdiffusers.schedulers import DDIMScheduler
    ucfg, uP, unet = make_unet("tiny_xl")
    nets = [make_cn("tiny_xl", seed=1 + k) for k in range(n_nets)]
    x, ctx, img, added = inputs(ucfg, 2, 16, 20)
    g = torch.Generator().manual_seed(5)
    imgs = [img] + [torch.rand(img.shape, generator=g).to(bf16).float() for _ in range(n_nets - 1)]
    neg = torch.zeros_like(ctx)
    steps, gs = 4, 5.0
    scales, start, end = [0.8, 0.5][:n_nets], [0.0, 0.25][:n_nets], [0.75, 1.0][:n_nets]
    cn = nets[0][2] if n_nets == 1 else [n[2] for n in nets]
    lat = {}
    for graph in (True, False):
        pipe = StableDiffusionControlNetPipeline(unet, cn, DDIMScheduler(**SD), use_cuda_graph=graph)
        kw = dict(image=img if n_nets == 1 else imgs, controlnet_conditioning_scale=scales[0] if n_nets == 1 else scales,
                  control_guidance_start=start[0] if n_nets == 1 else start,
                  control_guidance_end=end[0] if n_nets == 1 else end, guess_mode=guess)
        lat[graph] = pipe(prompt_embeds=ctx, negative_prompt_embeds=neg, latents=x, num_inference_steps=steps,
                          guidance_scale=gs, added_cond_kwargs=added, **kw).cpu()
        again = pipe(prompt_embeds=ctx, negative_prompt_embeds=neg, latents=x, num_inference_steps=steps,
                     guidance_scale=gs, added_cond_kwargs=added, **kw).cpu()
        assert torch.equal(again, lat[graph]), "two calls with the same inputs must agree bit for bit"
    assert torch.equal(lat[True], lat[False])
    ref = oracle_loop(ucfg, uP, [n[0] for n in nets], [n[1] for n in nets], x, ctx, neg, imgs, added, steps, gs,
                      scales, start, end, guess)
    compare(lat[True], ref, f"{steps}-step ControlNet CFG DDIM loop (nets={n_nets}, guess={guess})")


def test_controlnet_pipeline_keep_zero_equals_plain_pipeline():
    """control_guidance_end = 0.0: every keep is 0, the ControlNet runs at scale 0 and its residuals are exactly 0."""
    from paddlemix_b200.ppdiffusers.pipelines import StableDiffusionControlNetPipeline, StableDiffusionPipeline
    from paddlemix_b200.ppdiffusers.schedulers import DDIMScheduler
    ucfg, uP, unet = make_unet("tiny_xl")
    _, _, cn = make_cn("tiny_xl")
    x, ctx, img, added = inputs(ucfg, 2, 16, 20)
    for graph in (True, False):
        kw = dict(prompt_embeds=ctx, latents=x, num_inference_steps=3, guidance_scale=4.0, added_cond_kwargs=added)
        plain = StableDiffusionPipeline(unet, DDIMScheduler(**SD), use_cuda_graph=graph)(**kw)
        pipe = StableDiffusionControlNetPipeline(unet, cn, DDIMScheduler(**SD), use_cuda_graph=graph)
        with_cn = pipe(image=img, control_guidance_end=0.0, **kw)
        assert torch.equal(with_cn, plain)
