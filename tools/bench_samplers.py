"""Cost of the Euler-ancestral, UniPC, stochastic DDIM and DPM-Solver++ 2M SDE steps. Prints one JSON line:
  * the GPU's name, power limit and max SM clock, read in the same run;
  * the time of b200mix_euler_ancestral_step, b200mix_ddim_eta_step and b200mix_dpmpp_2m_sde_step (order 2; all three
    with in-kernel Philox noise) and of b200mix_unipc_step (order 3 with the order-3 corrector: the most history it
    reads) at SDXL 1024^2 and SD1.5 512^2, B = 8 with CFG (bf16 model output [2B, 4, h, w] into an fp32 [B, 4, h, w]
    state), with the bytes each reads and writes once and their share of the H100 SXM data-sheet 3.35 TB/s;
  * ms per denoising step (graph replay of the UNet + scale_model_input + scheduler step) of the SDXL 1024^2 B = 8 CFG
    pipeline loop with synthetic weights, for Euler a, UniPC, DDIM with eta = 0.5 and DPM-Solver++ 2M SDE against
    Euler, DDIM (eta = 0) and DPM-Solver++ 2M, alternated over `--repeats` rounds: median, min and max.
Writes nothing to the tree.

    python tools/bench_samplers.py [--batch 8] [--steps 10] [--repeats 3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_TBS = 3.35
XL = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", timestep_spacing="leading", steps_offset=1)
UNET_KEYS = ("in_channels", "out_channels", "down_block_types", "up_block_types", "block_out_channels",
             "layers_per_block", "cross_attention_dim", "transformer_layers_per_block", "attention_head_dim",
             "use_linear_projection", "addition_embed_type", "addition_time_embed_dim",
             "projection_class_embeddings_input_dim")


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=False).stdout.strip()
    name, power, clock = (q.split(", ") + ["?", "?", "?"])[:3]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def event_ms(fn, n):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(n):
        fn(i)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / n


def spread(v):
    return {"median": round(statistics.median(v), 3), "min": round(min(v), 3), "max": round(max(v), 3)}


def schedulers():
    from paddlemix_b200.ppdiffusers.schedulers import (DDIMScheduler, DPMSolverMultistepScheduler,
                                                       EulerAncestralDiscreteScheduler, EulerDiscreteScheduler,
                                                       UniPCMultistepScheduler)
    return {"euler_a": EulerAncestralDiscreteScheduler(**XL), "unipc": UniPCMultistepScheduler(**XL, solver_order=3),
            "ddim_eta": DDIMScheduler(**XL, set_alpha_to_one=False),
            "dpmpp_2m_sde": DPMSolverMultistepScheduler(**XL, algorithm_type="sde-dpmsolver++"),
            "euler": EulerDiscreteScheduler(**XL), "ddim": DDIMScheduler(**XL, set_alpha_to_one=False),
            "dpmpp_2m": DPMSolverMultistepScheduler(**XL)}


def kernel_times(B, g):
    """Per-kernel ms and bytes at SDXL 1024^2 and SD1.5 512^2 latents (B images, CFG)."""
    import torch

    from paddlemix_b200 import ops
    out = {}
    for model, h in (("sdxl_1024", 128), ("sd15_512", 64)):
        shape = (B, 4, h, h)
        n = B * 4 * h * h
        eps = torch.randn((2 * B, 4, h, h), generator=g).to(torch.bfloat16).cuda()
        x = torch.randn(shape, generator=g).cuda()
        bufs = [torch.randn(shape, generator=g).cuda() for _ in range(6)]
        coeffs = dict(alpha_t=0.5, sigma_t=0.8, A_c=0.9, K_c=-0.1, E_c=-0.1, rc_last=0.45, rc=[0.25, -0.1],
                      rk_c=[-0.9, -1.7], A_p=0.9, K_p=-0.1, E_p=-0.1, rp=[1.7, -1.1], rk_p=[-0.9, -1.7])
        runs = {
            # reads m_u, m_c (bf16) and x, writes x_prev: 2 + 2 + 4 + 4 bytes per element
            "euler_ancestral_step": (lambda i: ops.euler_ancestral_step(eps[:B], eps[B:], 5.0, x, None, 3.5, -0.96, 13.25,
                                                                        -1.25, 0.75, seed=1234, step=i, out=bufs[0]),
                                     12 * n),
            # reads m_u, m_c, x, last_sample, m_prev and the two older x0 (hp0 = m_prev, hp1 = hc0), writes x_next,
            # x_corr (in place over last_sample) and m_out: 2 + 2 + 4 * 5 read, 4 * 3 written
            "unipc_step": (lambda i: ops.unipc_step(eps[:B], eps[B:], 5.0, x, coeffs, bufs[1], bufs[2],
                                                    last_sample=bufs[2], m_prev=bufs[3], hist_c=[bufs[4], bufs[5]],
                                                    hist_p=[bufs[3], bufs[4]], out=bufs[0]), 36 * n),
            # reads m_u, m_c (bf16) and x, writes x_prev: 2 + 2 + 4 + 4 bytes per element
            "ddim_eta_step": (lambda i: ops.ddim_eta_step(eps[:B], eps[B:], 5.0, x, None, 0.9, 0.43, 0.95, 0.2, 0.25,
                                                          seed=1234, step=i, out=bufs[0]), 12 * n),
            # order 2: reads m_u, m_c, x and m_prev, writes x_next and m_out: 2 + 2 + 4 * 2 read, 4 * 2 written
            "dpmpp_2m_sde_step": (lambda i: ops.dpmpp_2m_sde_step(eps[:B], eps[B:], 5.0, x, None, bufs[1], bufs[2], 0.9,
                                                                  0.6, 0.8, 0.1, 0.05, 0.7, 0.3, seed=1234, step=i,
                                                                  out=bufs[0]), 20 * n),
        }
        for name, (fn, nbytes) in runs.items():
            for i in range(20):
                fn(i)
            ms = statistics.median([event_ms(fn, 200) for _ in range(5)])
            out[f"{model}_{name}"] = {"ms": round(ms, 4), "bytes": nbytes,
                                      "hbm_share": round(nbytes / (ms * 1e-3) / (HBM_TBS * 1e12), 3)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--steps", type=int, default=10, help="timed steps per sampler and round")
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()

    import torch

    from oracle.unet import UNET_CONFIGS
    from paddlemix_b200.ppdiffusers.pipelines import GraphedUNet
    from paddlemix_b200.ppdiffusers.unet_2d_condition import UNet2DConditionModel

    if not torch.cuda.is_available():
        raise SystemExit("bench_samplers.py needs a GPU")
    B, L, H = args.batch, 77, 128
    g = torch.Generator().manual_seed(0)
    kernels = kernel_times(B, g)

    cfg = UNET_CONFIGS["sdxl"]
    unet = UNet2DConditionModel(**{k: cfg[k] for k in UNET_KEYS}).init_synthetic_weights(seed=1, device=0)
    dev, D = unet.device, cfg["cross_attention_dim"]
    ctx = torch.randn(2 * B, L, D, generator=g).to(torch.bfloat16).to(dev)
    added = {"text_embeds": torch.randn(2 * B, 1280, generator=g).to(torch.bfloat16).to(dev),
             "time_ids": torch.tensor([[1024.0, 1024.0, 0.0, 0.0, 1024.0, 1024.0]] * (2 * B)).to(dev)}
    den = GraphedUNet(unet, (2 * B, 4, H, H), (2 * B, L, D), {k: v.shape for k, v in added.items()})
    lat0 = torch.randn(B, 4, H, H, generator=g).to(dev)
    den(torch.cat([lat0, lat0], 0), 981.0, ctx, added)
    scheds = schedulers()
    state = {k: dict(x=lat0.clone(), nxt=torch.empty_like(lat0), model_in=torch.empty(2 * B, 4, H, H, device=dev))
             for k in scheds}

    def stepper(key):
        sch, st = scheds[key], state[key]
        gen = torch.Generator().manual_seed(7)

        def step(i):
            if i % 50 == 0:
                sch.set_timesteps(50)
                st["x"].copy_(lat0)
            t = sch.timesteps[i % 50]
            scaled = sch.scale_model_input(st["x"], t)
            st["model_in"][:B].copy_(scaled)
            st["model_in"][B:].copy_(scaled)
            eps = den(st["model_in"], float(t))
            kw = {"generator": gen} if getattr(sch, "takes_generator", False) else {}  # the pipelines' rule
            if key == "ddim_eta":
                kw["eta"] = 0.5
            sch.step(eps[:B], t, st["x"], model_output_cond=eps[B:], guidance_scale=5.0, out=st["nxt"], **kw)
            st["x"], st["nxt"] = st["nxt"], st["x"]
        return step

    steps = {k: stepper(k) for k in scheds}
    for k in scheds:
        event_ms(steps[k], 3)
    times = {k: [] for k in scheds}
    for _ in range(args.repeats):
        for k in scheds:
            times[k].append(event_ms(steps[k], args.steps))
    print(json.dumps({"gpu": gpu_info(), "batch": B, "cfg": True, "kernels": kernels,
                      "sdxl_1024_step_ms": {k: spread(v) for k, v in times.items()},
                      "hbm_tb_s_datasheet": HBM_TBS}))


if __name__ == "__main__":
    main()
