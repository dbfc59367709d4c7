"""Euler-ancestral and UniPC on the device: both fused steps bit for bit against the CPU oracle on identical fp32
inputs (bf16 / fp32 model outputs, CFG on and off, every prediction type, UniPC orders 1-3 with the corrector on and
off, a small shape and SDXL's [16, 4, 128, 128] CFG batch into an [8, 4, 128, 128] state), the in-kernel Philox noise
against the oracle's restatement of its stream, the UniPC goldens of the reference on the device, and the pipelines
driven by both schedulers against the oracle UNet + oracle scheduler loop."""
import json
import os

import pytest
import torch

from oracle import samplers as OSa
from oracle import unet as O
from oracle.iddpm import philox_normal

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16
XL = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", timestep_spacing="leading", steps_offset=1)
SHAPES = {"small": (2, 4, 16, 16), "sdxl": (8, 4, 128, 128)}


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


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("dtype", [bf16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("cfg", [True, False], ids=["cfg", "nocfg"])
@pytest.mark.parametrize("prediction_type", ["epsilon", "v_prediction"])
def test_euler_ancestral_step_is_bit_exact(shape, dtype, cfg, prediction_type):
    from paddlemix_b200.ppdiffusers.schedulers import EulerAncestralDiscreteScheduler
    if shape == "sdxl" and (dtype, cfg) != (bf16, True):
        pytest.skip("the production shape runs the production inputs: bf16 CFG")
    shp = SHAPES[shape]
    kw = dict(XL, prediction_type=prediction_type)
    s, o = EulerAncestralDiscreteScheduler(**kw), OSa.EulerAncestralDiscreteScheduler(**kw)
    s.set_timesteps(6), o.set_timesteps(6)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(shp, generator=g) * s.init_noise_sigma
    xd = x.cuda()
    for k, t in enumerate(s.timesteps[:4]):
        (mu, mc), m, gs = model_outputs(shp, dtype, cfg, g)
        noise = torch.randn(shp, generator=g)
        out = s.step(mu, t, xd, noise=noise.cuda(), model_output_cond=mc, guidance_scale=gs, out=xd if k % 2 else None)
        x = o.step(m, torch.tensor(t), x, noise)
        assert torch.equal(out.cpu(), x), (shape, k)
        xd = out


@pytest.mark.parametrize("shape", list(SHAPES))
def test_euler_ancestral_philox_noise_is_the_oracles_stream(shape):
    """noise=NULL draws philox_normal(seed, step, n) inside the kernel: the same bits as passing that stream."""
    from paddlemix_b200 import ops
    shp = SHAPES[shape]
    n = torch.Size(shp).numel()
    g = torch.Generator().manual_seed(4)
    x = torch.randn(shp, generator=g).cuda()
    m = torch.randn(shp, generator=g).to(bf16).cuda()
    seed = 0x9E3779B97F4A7C15
    for step in (0, 7):
        a = ops.euler_ancestral_step(m, None, 0.0, x, None, 3.5, -0.96, 13.25, -1.25, 0.75, seed=seed, step=step)
        z = philox_normal(seed, step, n).reshape(shp)
        b = ops.euler_ancestral_step(m, None, 0.0, x, z.cuda(), 3.5, -0.96, 13.25, -1.25, 0.75)
        assert torch.equal(a, b)
        assert z.std().item() == pytest.approx(1.0, abs=0.05)


def unipc_pair(**kw):
    from paddlemix_b200.ppdiffusers.schedulers import UniPCMultistepScheduler
    return UniPCMultistepScheduler(**kw), OSa.UniPCMultistepScheduler(**kw)


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("dtype", [bf16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("cfg", [True, False], ids=["cfg", "nocfg"])
@pytest.mark.parametrize("prediction_type", ["epsilon", "sample", "v_prediction"])
@pytest.mark.parametrize("corrector", [True, False], ids=["unic", "nounic"])
@pytest.mark.parametrize("solver_type", ["bh1", "bh2"])
def test_unipc_step_is_bit_exact(shape, dtype, cfg, prediction_type, corrector, solver_type):
    """solver_order 3 over 6 steps with lower_order_final: predictor orders 1, 2, 3, 3, 2, 1 and corrector orders
    1, 2, 3, 3, 2 (none with every step in disable_corrector)."""
    if shape == "sdxl" and ((dtype, cfg) != (bf16, True) or solver_type == "bh1" or prediction_type == "sample"):
        pytest.skip("the production shape runs the production inputs: bf16 CFG, bh2")
    shp = SHAPES[shape]
    kw = dict(XL, solver_order=3, prediction_type=prediction_type, solver_type=solver_type,
              disable_corrector=[] if corrector else list(range(6)))
    s, o = unipc_pair(**kw)
    s.set_timesteps(6), o.set_timesteps(6)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(shp, generator=g)
    xd, nxt = x.cuda(), torch.empty(shp, device="cuda")
    for k, t in enumerate(s.timesteps):
        (mu, mc), m, gs = model_outputs(shp, dtype, cfg, g)
        out = s.step(mu, t, xd, model_output_cond=mc, guidance_scale=gs, out=nxt)
        x = o.step(m, torch.tensor(t), x)
        assert torch.equal(out.cpu(), x), (shape, k)
        xd, nxt = out, xd  # the pipeline's buffer swap: the scheduler's state must not live in them


GOLD = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "unipc_goldens.json")))


def deter(kind, flip=False):  # test_schedulers.py:261-290 (4d), test_scheduler_unipc.py:299-325 (1d)
    shape = (3, 8, 8, 4) if kind == "4d" else (3, 8, 4)
    n = torch.Size(shape).numel()
    s = torch.arange(n)
    s = (s.flip(-1) if flip else s).reshape(shape) / n
    return s.permute(3, 0, 1, 2).contiguous() if kind == "4d" else s.permute(2, 0, 1).contiguous()


@pytest.mark.parametrize("kind", ["4d", "1d"])
def test_unipc_full_loop_reproduces_the_goldens_on_the_device(kind):
    from paddlemix_b200.ppdiffusers.schedulers import UniPCMultistepScheduler
    fx = GOLD["fixtures"][kind]
    cases = [(c["config"], None) for c in fx["full_loop"]] + [({}, fx["full_loop_with_noise"])]
    for config, noisy in cases:
        sch = UniPCMultistepScheduler(**{**GOLD["config"], **config})
        sch.set_timesteps(GOLD["num_inference_steps"])
        timesteps = sch.timesteps
        x = deter(kind)
        if noisy:
            o = OSa.UniPCMultistepScheduler(**GOLD["config"])
            o.set_timesteps(GOLD["num_inference_steps"])
            timesteps = timesteps[noisy["t_start"]:]
            x = o.add_noise(x, deter(kind, flip=True), torch.from_numpy(timesteps[:1]))
        x = x.cuda()
        for t in timesteps:
            x = sch.step(x * float(t) / (float(t) + 1), t, x)
        mean = x.abs().mean().item()
        if noisy:
            assert abs(x.abs().sum().item() - noisy["sum"]) < GOLD["sum_atol"]
            assert abs(mean - noisy["mean"]) < GOLD["mean_atol"]
        else:
            assert abs(mean - [c for c in fx["full_loop"] if c["config"] == config][0]["mean"]) < GOLD["mean_atol"], mean


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


def compare(out, ref, what):  # the tolerance of test_unet_gpu.py's pipeline-vs-oracle loops
    out, ref = out.float().cpu(), ref.float()
    cos = torch.nn.functional.cosine_similarity(out.flatten(), ref.flatten(), dim=0).item()
    err = (out - ref).abs().max().item()
    scale = ref.abs().max().item()
    assert cos >= 0.999, f"{what}: cosine {cos}"
    assert err <= 0.04 * scale, f"{what}: max err {err} vs scale {scale}"


def new_scheduler(name):
    from paddlemix_b200.ppdiffusers import EulerAncestralDiscreteScheduler, UniPCMultistepScheduler
    if name == "euler_a":
        return EulerAncestralDiscreteScheduler(**XL)
    return UniPCMultistepScheduler(**XL, solver_order=3)


@pytest.mark.parametrize("name", ["euler_a", "unipc"])
def test_pipeline_graphed_eager_oracle(name, tiny_xl):
    from paddlemix_b200.ppdiffusers.pipelines import StableDiffusionPipeline
    from paddlemix_b200.sampling import seed_from
    cfg, P, unet, x, ctx, added = tiny_xl
    neg = torch.zeros_like(ctx)
    steps, gs = 5, 5.0
    run = dict(prompt_embeds=ctx, negative_prompt_embeds=neg, latents=x, num_inference_steps=steps, guidance_scale=gs,
               added_cond_kwargs=added)
    lat = {}
    for graph in (True, False):
        pipe = StableDiffusionPipeline(unet, new_scheduler(name), use_cuda_graph=graph)
        lat[graph] = pipe(**run, generator=torch.Generator().manual_seed(21)).cpu()
        again = pipe(**run, generator=torch.Generator().manual_seed(21)).cpu()
        assert torch.equal(again, lat[graph]), "equal generators must give equal bits: the state is reset per call"
    assert torch.equal(lat[True], lat[False])
    pipe = StableDiffusionPipeline(unet, new_scheduler(name))
    assert torch.equal(pipe(**run).cpu(), pipe(**run).cpu()), "generator=None is the pipeline's fixed default"
    other = pipe(**run, generator=torch.Generator().manual_seed(22)).cpu()
    assert torch.equal(other, lat[True]) == (name != "euler_a"), "only Euler a depends on the seed"
    rescaled = pipe(**run, generator=torch.Generator().manual_seed(21), guidance_rescale=0.7).cpu()
    assert torch.isfinite(rescaled).all() and not torch.equal(rescaled, lat[True])

    sch = (OSa.EulerAncestralDiscreteScheduler(**XL) if name == "euler_a"
           else OSa.UniPCMultistepScheduler(**XL, solver_order=3))
    sch.set_timesteps(steps)
    seed = seed_from(torch.Generator().manual_seed(21))
    cur = x.clone() * float(sch.init_noise_sigma)
    add2 = {k: torch.cat([v, v], 0) for k, v in added.items()}
    for i, t in enumerate(sch.timesteps):
        xin = sch.scale_model_input(cur, t) if name == "euler_a" else cur
        eps = O.unet_forward(cfg, P, torch.cat([xin, xin], 0), float(t), torch.cat([neg, ctx], 0), add2)
        eu, ec = eps.chunk(2)
        m = eu + gs * (ec - eu)
        if name == "euler_a":
            cur = sch.step(m, t, cur, philox_normal(seed, i, cur.numel()).reshape(cur.shape))
        else:
            cur = sch.step(m, t, cur)
    compare(lat[True], cur, f"{steps}-step CFG {name} loop")


@pytest.mark.parametrize("name", ["euler_a", "unipc"])
def test_controlnet_pipeline_runs_both_samplers(name, tiny_xl):
    from oracle import controlnet as OC
    from paddlemix_b200.ppdiffusers.controlnet import ControlNetModel
    from paddlemix_b200.ppdiffusers.pipelines import StableDiffusionControlNetPipeline
    cfg, P, unet, x, ctx, added = tiny_xl
    cn_keys = ("in_channels", "flip_sin_to_cos", "freq_shift", "down_block_types", "block_out_channels",
               "layers_per_block", "norm_num_groups", "norm_eps", "cross_attention_dim", "transformer_layers_per_block",
               "attention_head_dim", "use_linear_projection", "addition_embed_type", "addition_time_embed_dim",
               "projection_class_embeddings_input_dim")
    cP = O.init_params(OC.controlnet_param_shapes(cfg), seed=2)
    cn = ControlNetModel(**{k: cfg[k] for k in cn_keys}).load_state_dict(cP, device=0)
    img = torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(6)).to(bf16).float()
    lat = {}
    for graph in (True, False):
        pipe = StableDiffusionControlNetPipeline(unet, cn, new_scheduler(name), use_cuda_graph=graph)
        lat[graph] = pipe(prompt_embeds=ctx, negative_prompt_embeds=torch.zeros_like(ctx), latents=x, image=img,
                          num_inference_steps=4, guidance_scale=5.0, added_cond_kwargs=added,
                          generator=torch.Generator().manual_seed(9)).cpu()
    assert torch.isfinite(lat[True]).all() and torch.equal(lat[True], lat[False])
