"""ControlNet cost on the SDXL workload of bench.py (1024^2 images -> 128^2 latents, B = 8, DDIM, CUDA graph,
synthetic weights). Prints one JSON line:
  * the GPU's name and power limit, read in the same run;
  * ms per denoising step (graph replay + scheduler step) of UNet alone and of ControlNet + UNet, without and with CFG
    (16 rows), the four variants alternated in one process over `--repeats` rounds: median, min, max;
  * the conditioning embedding's time per pipeline call (B control images of 1024^2);
  * every conditioning-embedding conv's kernel time with its achieved TB/s and TFLOP/s, using the byte and FLOP
    counts of oracle.controlnet.controlnet_flops, against the H100 SXM data-sheet 3.35 TB/s and 989 TFLOP/s (bf16
    dense).
Writes nothing to the tree.

    python tools/bench_controlnet.py [--batch 8] [--height 1024] [--steps 10] [--repeats 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_TBS, BF16_TFLOPS = 3.35, 989.0
DDIM = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False,
            set_alpha_to_one=False, steps_offset=1)


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--height", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=10, help="timed steps per variant and round")
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()

    import torch

    from oracle.controlnet import controlnet_flops
    from oracle.unet import UNET_CONFIGS, unet_flops
    from paddlemix_b200 import ops
    from paddlemix_b200.ppdiffusers.controlnet import ControlNetModel
    from paddlemix_b200.ppdiffusers.pipelines import GraphedUNet
    from paddlemix_b200.ppdiffusers.schedulers import DDIMScheduler
    from paddlemix_b200.ppdiffusers.unet_2d_condition import UNet2DConditionModel

    if not torch.cuda.is_available():
        raise SystemExit("bench_controlnet.py needs a GPU")
    cfg = UNET_CONFIGS["sdxl"]
    ukeys = ("in_channels", "out_channels", "down_block_types", "up_block_types", "block_out_channels",
             "layers_per_block", "cross_attention_dim", "transformer_layers_per_block", "attention_head_dim",
             "use_linear_projection", "addition_embed_type", "addition_time_embed_dim",
             "projection_class_embeddings_input_dim")
    unet = UNet2DConditionModel(**{k: cfg[k] for k in ukeys}).init_synthetic_weights(seed=1, device=0)
    cn = ControlNetModel(**{k: cfg[k] for k in ukeys if k not in ("out_channels", "up_block_types")})
    cn.init_synthetic_weights(seed=2, device=0)
    dev = unet.device
    B, H, L = args.batch, args.height // 8, 77
    g = torch.Generator().manual_seed(0)
    lat = torch.randn(B, 4, H, H, generator=g).to(dev)
    ctx = torch.randn(B, L, 2048, generator=g).to(torch.bfloat16).to(dev)
    te = torch.randn(B, 1280, generator=g).to(torch.bfloat16).to(dev)
    ids = torch.tensor([[float(args.height)] * 2 + [0.0, 0.0] + [float(args.height)] * 2] * B).to(dev)
    img = torch.rand(B, 3, args.height, args.height, generator=g).to(dev)
    cond_nhwc = ops.nchw_to_nhwc(img)
    emb = cn.embed_condition(cond_nhwc)
    table = cn.scale_table(cn.residual_scales(1.0))
    sched = DDIMScheduler(**DDIM)
    sched.set_timesteps(50)
    timesteps = [int(t) for t in sched.timesteps]

    variants = {}
    for cfg_rows, tag in ((1, "no_cfg"), (2, "cfg")):
        rows = B * cfg_rows
        r = lambda t: torch.cat([t] * cfg_rows, 0)  # noqa: E731
        added = {"text_embeds": r(te), "time_ids": r(ids)}
        shapes = {k: v.shape for k, v in added.items()}
        for name, kw in (("unet", {}), ("controlnet_unet", {"controlnet": cn})):
            den = GraphedUNet(unet, (rows, 4, H, H), (rows, L, 2048), shapes, **kw)
            extra = {"cond_embeddings": [r(emb)]} if kw else {}
            den(r(lat), 981.0, r(ctx), added, **extra)
            variants[f"{name}_{tag}"] = (den, bool(kw), rows)
    state = {k: lat.clone() for k in variants}
    nxt = torch.empty_like(lat)

    def stepper(key):
        den, with_cn, rows = variants[key]

        def step(i):
            t = timesteps[i % len(timesteps)]
            x = state[key]
            model_in = x if rows == B else torch.cat([x, x], 0)
            eps = den(model_in, float(t), scale_tables=[table] if with_cn else None)
            if rows == B:
                sched.step(eps, t, x, out=nxt)
            else:
                sched.step(eps[:B], t, x, model_output_cond=eps[B:], guidance_scale=5.0, out=nxt)
            state[key].copy_(nxt)
        return step

    steps = {k: stepper(k) for k in variants}
    for k in variants:  # warm-up
        event_ms(steps[k], 3)
    times = {k: [] for k in variants}
    for _ in range(args.repeats):
        for k in variants:
            times[k].append(event_ms(steps[k], args.steps))
    step_ms = {k: {"median": round(statistics.median(v), 3), "min": round(min(v), 3), "max": round(max(v), 3)}
               for k, v in times.items()}
    ratio = {tag: round(step_ms[f"controlnet_unet_{tag}"]["median"] / step_ms[f"unet_{tag}"]["median"], 3)
             for tag in ("no_cfg", "cfg")}

    # conditioning embedding: once per pipeline call
    for _ in range(3):
        cn.embed_condition(cond_nhwc)
    embed_ms = event_ms(lambda i: cn.embed_condition(cond_nhwc), 10)

    # each conditioning-embedding conv at its real shape
    fl = controlnet_flops(cfg, B, H, H, L, (args.height, args.height))
    layers, e = [], cond_nhwc
    for (conv, stride), acc in zip(cn.cond_convs, fl["cond_layers"]):
        narrow = conv.cin % 64 != 0
        fn = ops.conv3x3_narrow if narrow else ops.conv3x3
        x_in = e
        for _ in range(3):
            e = fn(x_in, conv.w, conv.b, stride=stride)
        ms = event_ms(lambda i: fn(x_in, conv.w, conv.b, stride=stride), 20)
        tbs, tfl = acc["bytes"] / ms / 1e9, acc["flops"] / ms / 1e9
        layers.append({"layer": conv.name, "kernel": "conv3x3_narrow" if narrow else "conv3x3",
                       "cin": conv.cin, "cout": conv.cout, "stride": stride, "in_hw": list(acc["in_hw"]),
                       "ms": round(ms, 4), "TB/s": round(tbs, 3), "TFLOP/s": round(tfl, 2),
                       "frac_hbm": round(tbs / HBM_TBS, 3), "frac_bf16_peak": round(tfl / BF16_TFLOPS, 3),
                       "bound": "bytes" if acc["bytes"] / (HBM_TBS * 1e12) > acc["flops"] / (BF16_TFLOPS * 1e12)
                       else "flops"})
    out = {"metric": "controlnet_sdxl_step", "gpu": gpu_info(), "batch": B, "image": args.height, "latent": H,
           "steps_per_round": args.steps, "repeats": args.repeats, "ms_per_step": step_ms,
           "controlnet_over_unet": ratio,
           "flops_per_step_tflop": {"unet": round(unet_flops(cfg, B, H, H, L) / 1e12, 3), "controlnet_encoder": round(fl["encoder"] / 1e12, 3),
                                    "zero_convs": round(fl["zero_convs"] / 1e12, 3)},
           "cond_embedding_ms_per_call": round(embed_ms, 3),
           "cond_embedding_tflop_per_call": round(fl["cond_embedding"] / 1e12, 4), "cond_layers": layers,
           "peaks": {"hbm_TB/s": HBM_TBS, "bf16_dense_TFLOP/s": BF16_TFLOPS}}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
