"""T2I-Adapter cost per denoising step and per call (DDIM, CUDA graph, synthetic weights). Prints one JSON line:
  * the GPU's name, power limit and max SM clock, read in the same run;
  * ms per denoising step (graph replay + scheduler step) of the UNet alone and of the UNet with adapter residuals,
    without and with CFG, for SDXL 1024^2 with FullAdapterXL and SD1.5 512^2 with FullAdapter: all variants alternated
    in one process over `--repeats` rounds, median, min and max;
  * the adapter's forward time per pipeline call (B images) and the residual write (b200mix_weighted_sum_rows);
  * the achieved bytes/s of the pixel-unshuffle, 2x2 average-pool and weighted-sum kernels at the call shapes (bytes
    read + written once), against the H100 SXM data-sheet 3.35 TB/s.
Writes nothing to the tree.

    python tools/bench_adapter.py [--batch 8] [--steps 10] [--repeats 3]
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
DDIM = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False,
            set_alpha_to_one=False, steps_offset=1)
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--steps", type=int, default=10, help="timed steps per variant and round")
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()

    import torch

    from oracle.adapter import ADAPTER_CONFIGS
    from oracle.unet import UNET_CONFIGS
    from paddlemix_b200 import ops
    from paddlemix_b200.ppdiffusers.adapter import T2IAdapter
    from paddlemix_b200.ppdiffusers.pipelines import GraphedUNet
    from paddlemix_b200.ppdiffusers.schedulers import DDIMScheduler
    from paddlemix_b200.ppdiffusers.unet_2d_condition import UNet2DConditionModel

    if not torch.cuda.is_available():
        raise SystemExit("bench_adapter.py needs a GPU")
    B, L = args.batch, 77
    sched = DDIMScheduler(**DDIM)
    sched.set_timesteps(50)
    timesteps = [int(t) for t in sched.timesteps]
    g = torch.Generator().manual_seed(0)
    variants, models, nxt = {}, {}, {}
    for model, image in (("sdxl", 1024), ("sd15", 512)):
        cfg = UNET_CONFIGS[model]
        unet = UNet2DConditionModel(**{k: cfg[k] for k in UNET_KEYS}).init_synthetic_weights(seed=1, device=0)
        adapter = T2IAdapter(**ADAPTER_CONFIGS[model]).init_synthetic_weights(seed=2, device=0)
        dev, H, D = unet.device, image // 8, cfg["cross_attention_dim"]
        lat = torch.randn(B, 4, H, H, generator=g).to(dev)
        ctx = torch.randn(B, L, D, generator=g).to(torch.bfloat16).to(dev)
        img = torch.rand(B, 3, image, image, generator=g).to(dev)
        added = None
        if cfg["addition_embed_type"] == "text_time":
            added = {"text_embeds": torch.randn(B, 1280, generator=g).to(torch.bfloat16).to(dev),
                     "time_ids": torch.tensor([[float(image)] * 2 + [0.0, 0.0] + [float(image)] * 2] * B).to(dev)}
        feats = adapter(img)
        models[model] = (unet, adapter, img, feats)
        nxt[model] = torch.empty_like(lat)
        for rows_per, tag in ((1, "no_cfg"), (2, "cfg")):
            rows = B * rows_per
            r = lambda t: torch.cat([t] * rows_per, 0)  # noqa: E731
            add = None if added is None else {k: r(v) for k, v in added.items()}
            shapes = None if add is None else {k: v.shape for k, v in add.items()}
            for with_adapter in (False, True):
                kw = {}
                if with_adapter:
                    bufs = [torch.empty((rows,) + tuple(f.shape[1:]), device=dev, dtype=torch.bfloat16) for f in feats]
                    for f, buf in zip(feats, bufs):
                        ops.weighted_sum_rows([f], [1.0], out=buf)
                    kw["intrablock_residuals"] = bufs
                den = GraphedUNet(unet, (rows, 4, H, H), (rows, L, D), shapes, **kw)
                den(r(lat), 981.0, r(ctx), add)
                name = f"{model}_{'adapter_unet' if with_adapter else 'unet'}_{tag}"
                variants[name] = dict(den=den, rows=rows, model=model, x=lat.clone())

    def stepper(key):
        v = variants[key]

        def step(i):
            t = timesteps[i % len(timesteps)]
            x, out = v["x"], nxt[v["model"]]
            model_in = x if v["rows"] == B else torch.cat([x, x], 0)
            eps = v["den"](model_in, float(t))
            if v["rows"] == B:
                sched.step(eps, t, x, out=out)
            else:
                sched.step(eps[:B], t, x, model_output_cond=eps[B:], guidance_scale=5.0, out=out)
            x.copy_(out)
        return step

    steps = {k: stepper(k) for k in variants}
    for k in variants:
        event_ms(steps[k], 3)
    times = {k: [] for k in variants}
    for _ in range(args.repeats):
        for k in variants:
            times[k].append(event_ms(steps[k], args.steps))
    step_ms = {k: spread(v) for k, v in times.items()}
    overhead = {f"{m}_{tag}": round(step_ms[f"{m}_adapter_unet_{tag}"]["median"] - step_ms[f"{m}_unet_{tag}"]["median"], 3)
                for m in ("sdxl", "sd15") for tag in ("no_cfg", "cfg")}

    per_call, kernels = {}, []
    for model, (unet, adapter, img, feats) in models.items():
        f = adapter.downscale_factor
        for _ in range(3):
            adapter(img)
        per_call[f"{model}_adapter_forward_ms"] = spread([event_ms(lambda i: adapter(img), 5) for _ in range(3)])
        bufs = [torch.empty((2 * B,) + tuple(x.shape[1:]), device=img.device, dtype=torch.bfloat16) for x in feats]

        def write(i):
            for x, buf in zip(feats, bufs):
                ops.weighted_sum_rows([x], [0.8], out=buf)
        write(0)
        per_call[f"{model}_residual_write_ms"] = spread([event_ms(write, 20) for _ in range(3)])
        h = ops.pixel_unshuffle(img, f)
        pooled_in = feats[0] if model == "sd15" else feats[1]
        for kname, fn, nbytes in (
                (f"pixel_unshuffle f={f} {tuple(img.shape)} fp32", lambda i: ops.pixel_unshuffle(img, f),
                 img.numel() * 4 + h.numel() * 2),
                (f"avgpool2x2 {tuple(pooled_in.shape)}", lambda i: ops.avgpool2x2_nhwc(pooled_in),
                 2 * pooled_in.numel() * 5 // 4),
                (f"weighted_sum_rows {tuple(feats[0].shape)} -> {2 * B} rows",
                 lambda i: ops.weighted_sum_rows([feats[0]], [0.8], out=bufs[0]), 2 * feats[0].numel() * 3)):
            fn(0)
            ms = min(event_ms(fn, 50) for _ in range(3))
            kernels.append({"model": model, "kernel": kname, "ms": round(ms, 4), "bytes": int(nbytes),
                            "TB/s": round(nbytes / ms / 1e9, 3), "frac_hbm": round(nbytes / ms / 1e9 / HBM_TBS, 3)})
    print(json.dumps({"metric": "t2i_adapter_step", "gpu": gpu_info(), "batch": B, "steps_per_round": args.steps,
                      "repeats": args.repeats, "ms_per_step": step_ms, "adapter_overhead_ms_per_step": overhead,
                      "per_call": per_call, "kernels": kernels, "peaks": {"hbm_TB/s": HBM_TBS}}))


if __name__ == "__main__":
    main()
