"""Stochastic DDIM (eta > 0) and DPM-Solver++ 2M SDE on the device: both fused steps bit for bit against the CPU oracle
given the same noise (bf16 / fp32 model outputs, CFG on and off, every DDIM prediction type with clip_sample and
use_clipped_model_output, DPM orders 1 and 2 with Karras sigmas, an odd element count and SDXL's [16, 4, 128, 128] CFG
batch into an [8, 4, 128, 128] state), the in-kernel Philox noise against oracle.iddpm.philox_normal, 20-step loops
against the oracle loops, and the pipelines (graphed = eager, equal generators give equal bits, another generator
changes them, ControlNet and T2I-Adapter)."""
import pytest
import torch

from oracle import stochastic as OSa
from oracle import unet as O
from oracle.iddpm import philox_normal

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16
XL = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", timestep_spacing="leading", steps_offset=1)
SHAPES = {"small": (2, 4, 16, 16), "odd": (3, 3, 5, 7), "sdxl": (8, 4, 128, 128)}


def model_outputs(shape, dtype, cfg, g):
    """(m_u, m_c or None) on the device and the guided fp32 model output the oracle sees (u + g*(c - u), each operation
    rounded as the kernels round it)."""
    u = torch.randn(shape, generator=g).to(dtype)
    c = torch.randn(shape, generator=g).to(dtype) if cfg else None
    gs = 5.0
    ref = u.float() if c is None else u.float() + gs * (c.float() - u.float())
    pair = torch.cat([u, c], 0).cuda() if cfg else u.cuda()  # one [2B, ...] model batch, as the pipelines produce it
    B = shape[0]
    return (pair[:B], pair[B:] if cfg else None), ref, gs


def production_only(shape, dtype, cfg):
    if shape == "sdxl" and (dtype, cfg) != (bf16, True):
        pytest.skip("the production shape runs the production inputs: bf16 CFG")


def ddim_pair(**kw):
    from paddlemix_b200.ppdiffusers.schedulers import DDIMScheduler
    kw = dict(XL, set_alpha_to_one=False, **kw)
    return DDIMScheduler(**kw), OSa.DDIMScheduler(**kw)


def sde_pair(**kw):
    from paddlemix_b200.ppdiffusers.schedulers import DPMSolverMultistepScheduler
    kw = dict(XL, algorithm_type="sde-dpmsolver++", **kw)
    return DPMSolverMultistepScheduler(**kw), OSa.DPMSolverSDEScheduler(**kw)


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("dtype", [bf16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("cfg", [True, False], ids=["cfg", "nocfg"])
@pytest.mark.parametrize("prediction_type,clip_sample,use_clipped", [
    ("epsilon", False, False), ("epsilon", True, True), ("sample", True, False), ("v_prediction", False, False),
    ("v_prediction", True, True)])
def test_ddim_eta_step_is_bit_exact(shape, dtype, cfg, prediction_type, clip_sample, use_clipped):
    production_only(shape, dtype, cfg)
    if shape == "sdxl" and prediction_type != "epsilon":
        pytest.skip("the production shape runs the production inputs: epsilon prediction")
    shp = SHAPES[shape]
    s, o = ddim_pair(prediction_type=prediction_type, clip_sample=clip_sample)
    s.set_timesteps(6), o.set_timesteps(6)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(shp, generator=g)
    xd = x.cuda()
    for k, t in enumerate(s.timesteps):
        (mu, mc), m, gs = model_outputs(shp, dtype, cfg, g)
        noise = torch.randn(shp, generator=g)
        eta = (0.3, 0.5, 1.0)[k % 3]
        out = s.step(mu, t, xd, eta=eta, model_output_cond=mc, guidance_scale=gs, use_clipped_model_output=use_clipped,
                     variance_noise=noise.cuda(), out=xd if k % 2 else None)
        x = o.step(m, t, x, eta=eta, use_clipped_model_output=use_clipped, variance_noise=noise)
        assert torch.equal(out.cpu(), x), (shape, k)
        xd = out


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("dtype", [bf16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("cfg", [True, False], ids=["cfg", "nocfg"])
@pytest.mark.parametrize("karras", [False, True], ids=["linear", "karras"])
def test_dpm_sde_step_is_bit_exact(shape, dtype, cfg, karras):
    """Six steps: orders 1, 2, 2, 2, 2, 1 (lower_order_final)."""
    production_only(shape, dtype, cfg)
    shp = SHAPES[shape]
    s, o = sde_pair(use_karras_sigmas=karras)
    s.set_timesteps(6), o.set_timesteps(6)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(shp, generator=g)
    xd, nxt = x.cuda(), torch.empty(shp, device="cuda")
    for k, t in enumerate(s.timesteps):
        (mu, mc), m, gs = model_outputs(shp, dtype, cfg, g)
        noise = torch.randn(shp, generator=g)
        out = s.step(mu, t, xd, model_output_cond=mc, guidance_scale=gs, noise=noise.cuda(), out=nxt if k % 2 else xd)
        x = o.step(m, torch.tensor(t), x, noise=noise)
        assert torch.equal(out.cpu(), x), (shape, k)
        if k % 2:
            xd, nxt = out, xd  # the pipeline's buffer swap: the scheduler's x0 history must not live in them


@pytest.mark.parametrize("shape", list(SHAPES))
def test_philox_noise_is_the_oracles_stream(shape):
    """noise=None draws philox_normal(seed, step, n) inside each kernel: the same bits as passing that stream."""
    from paddlemix_b200 import ops
    shp = SHAPES[shape]
    n = torch.Size(shp).numel()
    g = torch.Generator().manual_seed(4)
    x = torch.randn(shp, generator=g).cuda()
    m = torch.randn(shp, generator=g).to(bf16).cuda()
    prev = torch.randn(shp, generator=g).cuda()
    seed = 0x9E3779B97F4A7C15
    for step in (0, 7):
        z = philox_normal(seed, step, n).reshape(shp).cuda()
        a = ops.ddim_eta_step(m, None, 0.0, x, None, 0.9, 0.43, 0.95, 0.2, 0.25, seed=seed, step=step)
        b = ops.ddim_eta_step(m, None, 0.0, x, z, 0.9, 0.43, 0.95, 0.2, 0.25)
        assert torch.equal(a, b)
        mo_a, mo_b = torch.empty_like(x), torch.empty_like(x)
        a = ops.dpmpp_2m_sde_step(m, None, 0.0, x, None, prev, mo_a, 0.9, 0.6, 0.8, 0.1, 0.05, 0.7, 0.3, seed=seed,
                                  step=step)
        b = ops.dpmpp_2m_sde_step(m, None, 0.0, x, z, prev, mo_b, 0.9, 0.6, 0.8, 0.1, 0.05, 0.7, 0.3)
        assert torch.equal(a, b) and torch.equal(mo_a, mo_b)
        assert z.std().item() == pytest.approx(1.0, abs=0.05 if n > 1000 else 0.3)


@pytest.mark.parametrize("sampler", ["ddim_eta", "dpm_sde", "dpm_sde_karras"])
def test_twenty_step_loop_matches_the_oracle_loop(sampler):
    """A 20-step SDXL-latent CFG loop with a synthetic model output and the in-kernel noise seeded from a generator,
    against the oracle fed the same seed."""
    from paddlemix_b200.sampling import seed_from
    shp = (2, 4, 64, 64)
    if sampler == "ddim_eta":
        s, o = ddim_pair()
    else:
        s, o = sde_pair(use_karras_sigmas=sampler == "dpm_sde_karras")
    s.set_timesteps(20), o.set_timesteps(20)
    seed = seed_from(torch.Generator().manual_seed(31))
    g = torch.Generator().manual_seed(6)
    x = torch.randn(shp, generator=g)
    xd, nxt = x.cuda(), torch.empty(shp, device="cuda")
    for k, t in enumerate(s.timesteps):
        (mu, mc), m, gs = model_outputs(shp, bf16, True, g)
        kw = dict(model_output_cond=mc, guidance_scale=gs, out=nxt, generator=torch.Generator().manual_seed(31))
        if sampler == "ddim_eta":
            out = s.step(mu, t, xd, eta=1.0, **kw)
            x = o.step(m, t, x, eta=1.0, seed=seed)
        else:
            out = s.step(mu, t, xd, **kw)
            x = o.step(m, torch.tensor(t), x, seed=seed)
        assert torch.equal(out.cpu(), x), k
        xd, nxt = out, xd
    assert torch.isfinite(x).all()


# ---- pipelines -------------------------------------------------------------------------------------------------------
UNET_KEYS = ("in_channels", "out_channels", "flip_sin_to_cos", "freq_shift", "down_block_types", "up_block_types",
             "block_out_channels", "layers_per_block", "norm_num_groups", "norm_eps", "cross_attention_dim",
             "transformer_layers_per_block", "attention_head_dim", "use_linear_projection", "addition_embed_type",
             "addition_time_embed_dim", "projection_class_embeddings_input_dim", "resnet_out_scale_factor")


@pytest.fixture(scope="module")
def tiny_xl():
    from paddlemix_b200.ppdiffusers.unet_2d_condition import UNet2DConditionModel
    cfg = O.UNET_CONFIGS["tiny_xl"]
    P = O.init_params(O.unet_param_shapes(cfg), seed=1)
    unet = UNet2DConditionModel(**{k: cfg[k] for k in UNET_KEYS}).load_state_dict(P, device=0)
    g = torch.Generator().manual_seed(0)
    B, H, L = 2, 16, 20
    x = torch.randn(B, 4, H, H, generator=g).to(bf16).float()
    ctx = torch.randn(B, L, cfg["cross_attention_dim"], generator=g).to(bf16).float()
    n_text = cfg["projection_class_embeddings_input_dim"] - 6 * cfg["addition_time_embed_dim"]
    added = {"text_embeds": torch.randn(B, n_text, generator=g).to(bf16).float(),
             "time_ids": torch.tensor([[H * 8., H * 8., 0, 0, H * 8., H * 8.]] * B)}
    return cfg, P, unet, x, ctx, added


def new_scheduler(name):
    from paddlemix_b200.ppdiffusers.schedulers import DDIMScheduler, DPMSolverMultistepScheduler
    if name == "ddim_eta":
        return DDIMScheduler(**XL, set_alpha_to_one=False), dict(eta=0.5)
    return DPMSolverMultistepScheduler(**XL, algorithm_type="sde-dpmsolver++", use_karras_sigmas=True), {}


@pytest.mark.parametrize("name", ["ddim_eta", "dpm_sde"])
def test_pipeline_graphed_eager_and_generators(name, tiny_xl):
    from paddlemix_b200.ppdiffusers.pipelines import StableDiffusionPipeline
    cfg, P, unet, x, ctx, added = tiny_xl
    run = dict(prompt_embeds=ctx, negative_prompt_embeds=torch.zeros_like(ctx), latents=x, num_inference_steps=5,
               guidance_scale=5.0, added_cond_kwargs=added)
    lat = {}
    for graph in (True, False):
        sched, extra = new_scheduler(name)
        pipe = StableDiffusionPipeline(unet, sched, use_cuda_graph=graph)
        lat[graph] = pipe(**run, **extra, generator=torch.Generator().manual_seed(21)).cpu()
        again = pipe(**run, **extra, generator=torch.Generator().manual_seed(21)).cpu()
        assert torch.equal(again, lat[graph]), "equal generators must give equal bits: the state is reset per call"
    assert torch.equal(lat[True], lat[False])
    assert torch.isfinite(lat[True]).all()
    sched, extra = new_scheduler(name)
    pipe = StableDiffusionPipeline(unet, sched)
    assert torch.equal(pipe(**run, **extra).cpu(), pipe(**run, **extra).cpu()), "generator=None is the fixed default"
    other = pipe(**run, **extra, generator=torch.Generator().manual_seed(22)).cpu()
    assert not torch.equal(other, lat[True]), "the noise depends on the generator"
    rescaled = pipe(**run, **extra, generator=torch.Generator().manual_seed(21), guidance_rescale=0.7).cpu()
    assert torch.isfinite(rescaled).all() and not torch.equal(rescaled, lat[True])


def test_pipeline_ddim_eta_zero_ignores_the_generator(tiny_xl):
    """eta = 0 is the deterministic sampler: the generator only makes the initial latents."""
    from paddlemix_b200.ppdiffusers.schedulers import DDIMScheduler
    from paddlemix_b200.ppdiffusers.pipelines import StableDiffusionPipeline
    cfg, P, unet, x, ctx, added = tiny_xl
    pipe = StableDiffusionPipeline(unet, DDIMScheduler(**XL, set_alpha_to_one=False))
    run = dict(prompt_embeds=ctx, negative_prompt_embeds=torch.zeros_like(ctx), latents=x, num_inference_steps=4,
               guidance_scale=5.0, added_cond_kwargs=added)
    a = pipe(**run, generator=torch.Generator().manual_seed(1)).cpu()
    assert torch.equal(a, pipe(**run, eta=0.0, generator=torch.Generator().manual_seed(2)).cpu())
    assert not torch.equal(a, pipe(**run, eta=0.5, generator=torch.Generator().manual_seed(1)).cpu())


@pytest.mark.parametrize("name", ["ddim_eta", "dpm_sde"])
def test_controlnet_and_adapter_pipelines_run_both_samplers(name, tiny_xl):
    from oracle import adapter as OA
    from oracle import controlnet as OC
    from paddlemix_b200.ppdiffusers.adapter import T2IAdapter
    from paddlemix_b200.ppdiffusers.controlnet import ControlNetModel
    from paddlemix_b200.ppdiffusers.pipelines import StableDiffusionAdapterPipeline, StableDiffusionControlNetPipeline
    cfg, P, unet, x, ctx, added = tiny_xl
    cn_keys = ("in_channels", "flip_sin_to_cos", "freq_shift", "down_block_types", "block_out_channels",
               "layers_per_block", "norm_num_groups", "norm_eps", "cross_attention_dim", "transformer_layers_per_block",
               "attention_head_dim", "use_linear_projection", "addition_embed_type", "addition_time_embed_dim",
               "projection_class_embeddings_input_dim")
    cn = ControlNetModel(**{k: cfg[k] for k in cn_keys}).load_state_dict(
        O.init_params(OC.controlnet_param_shapes(cfg), seed=2), device=0)
    acfg = OA.ADAPTER_CONFIGS["tiny_xl"]
    adapter = T2IAdapter(**acfg).load_state_dict(O.init_params(OA.adapter_param_shapes(acfg), seed=3), device=0)
    img = torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(6)).to(bf16).float()
    run = dict(prompt_embeds=ctx, negative_prompt_embeds=torch.zeros_like(ctx), latents=x, image=img,
               num_inference_steps=4, guidance_scale=5.0, added_cond_kwargs=added)
    for make in (lambda s, graph: StableDiffusionControlNetPipeline(unet, cn, s, use_cuda_graph=graph),
                 lambda s, graph: StableDiffusionAdapterPipeline(unet, adapter, s, use_cuda_graph=graph)):
        lat = {}
        for graph in (True, False):
            sched, extra = new_scheduler(name)
            lat[graph] = make(sched, graph)(**run, **extra, generator=torch.Generator().manual_seed(9)).cpu()
        assert torch.isfinite(lat[True]).all() and torch.equal(lat[True], lat[False])
        sched, extra = new_scheduler(name)
        other = make(sched, True)(**run, **extra, generator=torch.Generator().manual_seed(10)).cpu()
        assert not torch.equal(other, lat[True])
