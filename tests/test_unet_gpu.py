"""Model-level parity on the GPU: paddlemix_b200's UNet2DConditionModel (bf16, sm_90a kernels through the C ABI)
against the CPU fp32 oracle on identical seeded inputs and weights.

Tolerance (stated, bf16 vs fp32): every activation is rounded to bf16 (2^-8 relative) after each of ~10^2 fused
ops, so we require cosine similarity >= 0.999 and max |err| <= 4 % of the output's max magnitude; the reference's own
fp16-vs-fp32 pipeline test allows a mean diff of 5e-2 (tests/pipelines/test_pipelines_common.py:567-600)."""
import pytest
import torch

from oracle import unet as O

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16


def make(cfg_name, seed=1):
    from paddlemix_b200.ppdiffusers.unet_2d_condition import UNet2DConditionModel
    cfg = O.UNET_CONFIGS[cfg_name]
    P = O.init_params(O.unet_param_shapes(cfg), seed=seed)
    keys = ("in_channels", "out_channels", "flip_sin_to_cos", "freq_shift", "down_block_types", "up_block_types",
            "block_out_channels", "layers_per_block", "norm_num_groups", "norm_eps", "cross_attention_dim",
            "transformer_layers_per_block", "attention_head_dim", "use_linear_projection", "addition_embed_type",
            "addition_time_embed_dim", "projection_class_embeddings_input_dim", "resnet_out_scale_factor")
    model = UNet2DConditionModel(**{k: cfg[k] for k in keys}).load_state_dict(P, device=0)
    return cfg, P, model


def inputs(cfg, B, H, L, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, cfg["in_channels"], H, H, generator=g)
    ctx = torch.randn(B, L, cfg["cross_attention_dim"], generator=g).to(bf16).float()
    added = None
    if cfg["addition_embed_type"] == "text_time":
        n_text = cfg["projection_class_embeddings_input_dim"] - 6 * cfg["addition_time_embed_dim"]
        added = {"text_embeds": torch.randn(B, n_text, generator=g).to(bf16).float(),
                 "time_ids": torch.tensor([[H * 8., H * 8., 0, 0, H * 8., H * 8.]] * B)}
    return x.to(bf16).float(), ctx, added


def compare(out, ref, what):
    out, ref = out.float().cpu(), ref.float()
    cos = torch.nn.functional.cosine_similarity(out.flatten(), ref.flatten(), dim=0).item()
    err = (out - ref).abs().max().item()
    scale = ref.abs().max().item()
    assert cos >= 0.999, f"{what}: cosine {cos}"
    assert err <= 0.04 * scale, f"{what}: max err {err} vs scale {scale}"
    return cos, err / scale


@pytest.mark.parametrize("name,B,H,L,t", [("tiny_sd", 2, 32, 77, 981), ("tiny_xl", 3, 32, 77, 481), ("tiny_xl", 1, 16, 20, 1)])
def test_unet_tiny_parity(name, B, H, L, t):
    cfg, P, model = make(name)
    x, ctx, added = inputs(cfg, B, H, L)
    ref = O.unet_forward(cfg, P, x, t, ctx, added)
    out = model(x.cuda(), t, ctx.cuda(), added_cond_kwargs=None if added is None else {k: v.cuda() for k, v in added.items()},
                return_dict=False)[0]
    assert out.shape == ref.shape and out.dtype == bf16
    compare(out, ref, f"{name} B{B} H{H}")


def test_unet_batch_vs_single_and_determinism():
    # ModelTesterMixin.test_determinism (test_modeling_common.py:317) / batch-single identical (:478)
    cfg, P, model = make("tiny_sd")
    x, ctx, _ = inputs(cfg, 3, 32, 77)
    a = model(x.cuda(), 10, ctx.cuda()).sample
    b = model(x.cuda(), 10, ctx.cuda()).sample
    assert torch.equal(a, b)
    one = model(x[1:2].cuda(), 10, ctx[1:2].cuda()).sample
    assert (one.float() - a[1:2].float()).abs().max().item() <= 1e-2 * a.float().abs().max().item()
    tt = model(x.cuda(), torch.tensor([10, 10, 10]), ctx.cuda()).sample
    assert torch.equal(tt, a)


def test_special_attn_processor():
    # test_models_unet_2d_condition.py:428-484: a custom processor object receives cross_attention_kwargs and is
    # called once per attention layer; swapping it for the default must not change the result materially
    cfg, P, model = make("tiny_sd")
    x, ctx, _ = inputs(cfg, 2, 32, 77)
    base = model(x.cuda(), 10, ctx.cuda()).sample

    class Proc:
        def __init__(self):
            self.calls, self.number = 0, None

        def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None, number=None, **kw):
            self.calls += 1
            self.number = number
            return attn.fused_forward(hidden_states, encoder_hidden_states)

    p = Proc()
    n_layers = len(model.attn_processors)
    model.set_attn_processor(p)
    out = model(x.cuda(), 10, ctx.cuda(), cross_attention_kwargs={"number": 123}).sample
    assert p.calls == n_layers and p.number == 123
    assert (out.float() - base.float()).abs().max().item() <= 2e-2 * base.float().abs().max().item()
    with pytest.raises(ValueError):
        model.set_attn_processor({"x": p})
    model.set_default_attn_processor()
    assert torch.equal(model(x.cuda(), 10, ctx.cuda()).sample, base)


@pytest.mark.parametrize("mask_dtype", [torch.bool, torch.int64, torch.float32])
def test_model_xattn_mask(mask_dtype):
    """Port of test_models_unet_2d_condition.py:486-519: a keep-all encoder_attention_mask == no mask; dropping the last
    context token changes the output; masking the last token == truncating it out of the condition. The reference's
    rtol 1e-3 / atol 1e-5 is for fp32; here both sides are the same bf16 kernels, so the mask-vs-truncate pair is
    compared at bf16 resolution (2e-2 of the output range), and both against the fp32 oracle with the mask."""
    cfg, P, model = make("tiny_sd")
    x, ctx, _ = inputs(cfg, 2, 32, 77)
    B, L = ctx.shape[:2]
    full = model(x.cuda(), 10, ctx.cuda()).sample
    scale = full.float().abs().max().item()
    keep_all = torch.ones(B, L).to(mask_dtype)
    assert torch.equal(model(x.cuda(), 10, ctx.cuda(), encoder_attention_mask=keep_all.cuda()).sample, full)
    trunc = model(x.cuda(), 10, ctx[:, :-1].contiguous().cuda()).sample
    assert (trunc.float() - full.float()).abs().max().item() > 1e-3 * scale
    mask_last = (torch.arange(L) < L - 1).expand(B, -1).to(mask_dtype)
    masked = model(x.cuda(), 10, ctx.cuda(), encoder_attention_mask=mask_last.cuda()).sample
    assert (masked.float() - trunc.float()).abs().max().item() <= 2e-2 * scale
    ref = O.unet_forward(cfg, P, x, 10, ctx, encoder_attention_mask=mask_last)
    compare(masked, ref, "encoder_attention_mask vs oracle")
    # a ragged key-padding mask (different per batch element) and a self-attention mask over the image tokens
    ragged = torch.ones(B, L)
    ragged[0, 40:] = 0
    ragged[1, 5:9] = 0
    out = model(x.cuda(), 10, ctx.cuda(), encoder_attention_mask=ragged.cuda()).sample
    compare(out, O.unet_forward(cfg, P, x, 10, ctx, encoder_attention_mask=ragged), "ragged encoder_attention_mask")


def test_controlnet_and_adapter_residuals():
    """down_block_additional_residuals + mid_block_additional_residual (ControlNet) and
    down_intrablock_additional_residuals (T2I-Adapter), unet_2d_condition.py:1078-1155, against the oracle."""
    cfg, P, model = make("tiny_xl")
    B, H = 2, 32
    x, ctx, added = inputs(cfg, B, H, 77)
    addc = {k: v.cuda() for k, v in added.items()}
    L = O.unet_layout(cfg)
    g = torch.Generator().manual_seed(7)
    # skip tensors: conv_in output, then per down block its resnet outputs (+ the downsampler output)
    shapes, hw, ch = [(cfg["block_out_channels"][0], H)], H, None
    for d in L["down"]:
        for _ in range(d["layers"]):
            shapes.append((d["out_ch"], hw))
        if d["downsample"]:
            hw //= 2
            shapes.append((d["out_ch"], hw))
    down_res = [(0.3 * torch.randn(B, c, s, s, generator=g)).to(bf16).float() for c, s in shapes]
    mid_res = (0.3 * torch.randn(B, L["mid"]["ch"], hw, hw, generator=g)).to(bf16).float()
    out = model(x.cuda(), 481, ctx.cuda(), added_cond_kwargs=addc, down_block_additional_residuals=[r.cuda() for r in down_res],
                mid_block_additional_residual=mid_res.cuda()).sample
    ref = O.unet_forward(cfg, P, x, 481, ctx, added, down_block_additional_residuals=down_res,
                         mid_block_additional_residual=mid_res)
    compare(out, ref, "controlnet residuals")
    base = model(x.cuda(), 481, ctx.cuda(), added_cond_kwargs=addc).sample
    assert (out.float() - base.float()).abs().max().item() > 1e-2 * base.float().abs().max().item()
    # T2I-Adapter: one residual per down block (block output resolution / channels)
    intra, hw = [], H
    for d in L["down"]:
        if d["type"] == "CrossAttnDownBlock2D":
            intra.append((0.3 * torch.randn(B, d["out_ch"], hw, hw, generator=g)).to(bf16).float())
            if d["downsample"]:
                hw //= 2
        else:
            if d["downsample"]:
                hw //= 2
            intra.append((0.3 * torch.randn(B, d["out_ch"], hw, hw, generator=g)).to(bf16).float())
    out2 = model(x.cuda(), 481, ctx.cuda(), added_cond_kwargs=addc,
                 down_intrablock_additional_residuals=[r.cuda() for r in intra]).sample
    ref2 = O.unet_forward(cfg, P, x, 481, ctx, added, down_intrablock_additional_residuals=list(intra))
    compare(out2, ref2, "t2i-adapter residuals")


def test_graphed_pipeline_matches_eager_and_oracle_loop():
    from oracle.schedulers import DDIMScheduler as ODDIM
    from paddlemix_b200.ppdiffusers.pipelines import StableDiffusionPipeline
    from paddlemix_b200.ppdiffusers.schedulers import DDIMScheduler
    SD = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False,
              set_alpha_to_one=False, steps_offset=1)
    cfg, P, model = make("tiny_xl")
    x, ctx, added = inputs(cfg, 2, 16, 20)
    neg = torch.zeros_like(ctx)
    steps, gs = 4, 5.0
    lat = {}
    for graph in (True, False):
        pipe = StableDiffusionPipeline(model, DDIMScheduler(**SD), use_cuda_graph=graph)
        lat[graph] = pipe(prompt_embeds=ctx, negative_prompt_embeds=neg, latents=x, num_inference_steps=steps,
                          guidance_scale=gs, added_cond_kwargs=added).cpu()
    assert torch.equal(lat[True], lat[False])
    # oracle loop (pipeline_stable_diffusion.py:858-908 restated): fp32 UNet + fp32 DDIM
    sch = ODDIM(**SD)
    sch.set_timesteps(steps)
    cur = x.clone()
    add2 = {k: torch.cat([v, v], 0) for k, v in added.items()}
    for t in sch.timesteps:
        eps = O.unet_forward(cfg, P, torch.cat([cur, cur], 0), int(t), torch.cat([neg, ctx], 0), add2)
        eu, ec = eps.chunk(2)
        cur = sch.step(eu + gs * (ec - eu), t, cur)
    compare(lat[True], cur, "4-step CFG DDIM loop")


def test_euler_discrete_pipeline_matches_oracle_loop():
    """SDXL's default sampler: EulerDiscreteScheduler (host numpy + b200mix_scale_model_input / b200mix_euler_step) driven
    by the pipeline (graph and eager bit-identical) against the oracle's fp32 UNet + fp32 Euler loop; the device step
    itself is bit-exact against the oracle on identical fp32 inputs."""
    from oracle.schedulers import EulerDiscreteScheduler as OEuler
    from paddlemix_b200 import ops
    from paddlemix_b200.ppdiffusers.pipelines import StableDiffusionPipeline
    from paddlemix_b200.ppdiffusers.schedulers import EulerDiscreteScheduler
    XL = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", timestep_spacing="leading", steps_offset=1)
    # (1) one step, bit-exact
    o, s = OEuler(**XL), EulerDiscreteScheduler(**XL)
    o.set_timesteps(8), s.set_timesteps(8)
    g = torch.Generator().manual_seed(3)
    xs, e = torch.randn(2, 4, 16, 16, generator=g) * s.init_noise_sigma, torch.randn(2, 4, 16, 16, generator=g)
    for t in s.timesteps[:3]:
        scaled = s.scale_model_input(xs.cuda(), t)
        assert torch.equal(scaled.cpu(), o.scale_model_input(xs, torch.tensor(t)))
        nxt = s.step(e.cuda(), t, xs.cuda())
        xs = o.step(e, torch.tensor(t), xs)
        assert torch.equal(nxt.cpu(), xs)
    # (2) the pipeline loop
    cfg, P, model = make("tiny_xl")
    x, ctx, added = inputs(cfg, 2, 16, 20)
    neg = torch.zeros_like(ctx)
    steps, gs = 4, 5.0
    lat = {}
    for graph in (True, False):
        pipe = StableDiffusionPipeline(model, EulerDiscreteScheduler(**XL), use_cuda_graph=graph)
        lat[graph] = pipe(prompt_embeds=ctx, negative_prompt_embeds=neg, latents=x, num_inference_steps=steps,
                          guidance_scale=gs, added_cond_kwargs=added).cpu()
    assert torch.equal(lat[True], lat[False])
    sch = OEuler(**XL)
    sch.set_timesteps(steps)
    cur = x.clone() * sch.init_noise_sigma
    add2 = {k: torch.cat([v, v], 0) for k, v in added.items()}
    for t in sch.timesteps:
        xin = sch.scale_model_input(cur, t)
        eps = O.unet_forward(cfg, P, torch.cat([xin, xin], 0), float(t), torch.cat([neg, ctx], 0), add2)
        eu, ec = eps.chunk(2)
        cur = sch.step(eu + gs * (ec - eu), t, cur)
    compare(lat[True], cur, "4-step CFG Euler loop")


@pytest.mark.slow
def test_sd15_parity_config_c1():
    """BASELINE.json configs[0]: SD1.5 UNet, 1 x 512x512 (latent 64x64), one timestep, against the fp32 CPU oracle."""
    cfg, P, model = make("sd15")
    x, ctx, _ = inputs(cfg, 1, 64, 77)
    for t in (981,):
        ref = O.unet_forward(cfg, P, x, t, ctx)
        out = model(x.cuda(), t, ctx.cuda()).sample
        cos, rel = compare(out, ref, f"sd15 t={t}")
        print(f"sd15 C1 parity t={t}: cosine {cos:.6f}, max rel err {rel:.4f}")


def test_load_pretrained_from_safetensors_and_pdparams(tmp_path):
    """weights.load_pretrained: a torch-layout .safetensors (diffusers export, Linear [out, in]) and a paddle .pdparams
    of the same parameters must give bit-identical outputs to loading the reference-layout dict directly."""
    import pickle

    from paddlemix_b200 import weights as W
    cfg, P, model = make("tiny_xl", seed=5)
    x, ctx, added = inputs(cfg, 2, 32, 77)
    kw = dict(added_cond_kwargs={k: v.cuda() for k, v in added.items()}, return_dict=False)
    base = model(x.cuda(), 481, ctx.cuda(), **kw)[0]
    lin = W.linear_weight_keys(model)
    torch_sd = {("unet." + k): (v.t().contiguous() if k in lin else v) for k, v in P.items()}
    st = str(tmp_path / "diffusion_pytorch_model.safetensors")
    W.write_safetensors(st, torch_sd, {"format": "pt"})
    _, _, m2 = make("tiny_xl", seed=6)  # different weights, then overwritten from the file
    rep = W.load_pretrained(m2, st, device=0, prefix="unet.")
    assert rep["missing"] == [] and rep["unexpected"] == []
    assert torch.equal(m2(x.cuda(), 481, ctx.cuda(), **kw)[0], base)
    pd = str(tmp_path / "model_state.pdparams")
    with open(pd, "wb") as f:
        pickle.dump({k: v.numpy() for k, v in P.items()}, f, protocol=4)
    _, _, m3 = make("tiny_xl", seed=7)
    W.load_pretrained(m3, pd, device=0)
    assert torch.equal(m3(x.cuda(), 481, ctx.cuda(), **kw)[0], base)
    with pytest.raises(W.CheckpointError):
        W.load_pretrained(m3, st, device=0, layout="paddle", prefix="unet.")  # wrong layout is caught by the shape check


def test_dpm_solver_pp_2m_device_step_and_pipeline():
    """DPM-Solver++ 2M: the fused device step (b200mix_dpmpp_2m_step, x0 history kept on the device) is bit-exact against
    the oracle's fp32 step over a whole trajectory, with and without the fused CFG combine; the pipeline loop (graph and
    eager bit-identical) tracks the oracle's fp32 UNet + fp32 solver."""
    from oracle.schedulers import DPMSolverMultistepScheduler as ODPM
    from paddlemix_b200.ppdiffusers.pipelines import StableDiffusionPipeline
    from paddlemix_b200.ppdiffusers.schedulers import DPMSolverMultistepScheduler
    SD = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", timestep_spacing="leading", steps_offset=1)
    for kw, n in ((SD, 12), (dict(SD, use_karras_sigmas=True), 20)):
        o, s = ODPM(**kw), DPMSolverMultistepScheduler(**kw)
        o.set_timesteps(n), s.set_timesteps(n)
        g = torch.Generator().manual_seed(11)
        x = torch.randn(2, 4, 16, 16, generator=g)
        xd = x.cuda()
        for t in s.timesteps:
            eu, ec = torch.randn(2, 4, 16, 16, generator=g), torch.randn(2, 4, 16, 16, generator=g)
            xd = s.step(eu.cuda(), int(t), xd, model_output_cond=ec.cuda(), guidance_scale=7.5)
            x = o.step(eu + 7.5 * (ec - eu), torch.tensor(int(t)), x)
            assert torch.equal(xd.cpu(), x), f"DPM-Solver++ step at t={int(t)} is not bit-exact"
    cfg, P, model = make("tiny_xl")
    x, ctx, added = inputs(cfg, 2, 16, 20)
    neg = torch.zeros_like(ctx)
    steps, gs = 5, 5.0
    lat = {}
    for graph in (True, False):
        pipe = StableDiffusionPipeline(model, DPMSolverMultistepScheduler(**SD), use_cuda_graph=graph)
        lat[graph] = pipe(prompt_embeds=ctx, negative_prompt_embeds=neg, latents=x, num_inference_steps=steps,
                          guidance_scale=gs, added_cond_kwargs=added).cpu()
    assert torch.equal(lat[True], lat[False])
    sch = ODPM(**SD)
    sch.set_timesteps(steps)
    cur = x.clone()
    add2 = {k: torch.cat([v, v], 0) for k, v in added.items()}
    for t in sch.timesteps:
        eps = O.unet_forward(cfg, P, torch.cat([cur, cur], 0), int(t), torch.cat([neg, ctx], 0), add2)
        eu, ec = eps.chunk(2)
        cur = sch.step(eu + gs * (ec - eu), t, cur)
    compare(lat[True], cur, "5-step CFG DPM-Solver++ loop")
