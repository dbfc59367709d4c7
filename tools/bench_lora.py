"""LoRA cost on the SDXL UNet (synthetic weights, a LoRA on every LoRA-compatible layer). Prints one JSON line:
  * the GPU's name, power limit and max SM clock, read in the same run;
  * per rank (--ranks): the b200mix_lora_apply launch time (CUDA events, median of --repeats) and its bytes moved
    (bf16 base read + bf16 weight written + fp32 U and D read once) as a share of the H100 SXM data-sheet 3.35 TB/s;
    the wall time of a set_adapters switch and of a call-scale change (host factor assembly + the launch, ending in a
    device synchronise); the snapshot bytes;
  * the graphed 1024^2 pipeline step (CFG, DDIM) with the LoRA realised against none (the same adapter at weight 0),
    alternated over --repeats rounds.
Writes nothing to the tree.

    python tools/bench_lora.py [--ranks 4 32 128] [--steps 5] [--repeats 3]
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_adapter import DDIM, UNET_KEYS, event_ms, gpu_info, spread  # noqa: E402

HBM_TBS = 3.35


def synthetic_lora(unet, rank, seed):
    """ppdiffusers-format, Paddle-layout factors on every LoRA-compatible layer, drawn on the device."""
    import torch
    from paddlemix_b200.ppdiffusers.lora import lora_layer_shapes
    g = torch.Generator(device="cuda").manual_seed(seed)
    sd = {}
    for layer, shape in lora_layer_shapes(unet.state_dict_shapes()).items():
        n_out, n_in = shape[:2]
        fan = n_in * (shape[2] * shape[3] if len(shape) == 4 else 1)
        down = torch.randn(rank, fan, generator=g, device="cuda") / fan ** 0.5
        up = torch.randn(n_out, rank, generator=g, device="cuda") * 0.1 / rank ** 0.5
        if len(shape) == 2:
            sd[f"{layer}.lora.down.weight"], sd[f"{layer}.lora.up.weight"] = down.t(), up.t()
        else:
            sd[f"{layer}.lora.down.weight"] = down.reshape(rank, n_in, shape[2], shape[3])
            sd[f"{layer}.lora.up.weight"] = up.reshape(n_out, rank, 1, 1)
    return sd


def wall_ms(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ranks", type=int, nargs="+", default=[4, 32, 128])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import torch
    from oracle import unet as O
    from paddlemix_b200 import ops
    from paddlemix_b200.ppdiffusers.pipelines import StableDiffusionPipeline
    from paddlemix_b200.ppdiffusers.schedulers import DDIMScheduler
    from paddlemix_b200.ppdiffusers.unet_2d_condition import UNet2DConditionModel

    cfg = O.UNET_CONFIGS["sdxl"]
    unet = UNet2DConditionModel(**{k: cfg[k] for k in UNET_KEYS}).init_synthetic_weights(seed=1, device=0)
    res = {"gpu": gpu_info(), "ranks": {}}
    for r in args.ranks:
        unet.load_attn_procs(synthetic_lora(unet, r, 10 + r), adapter_name="a")
        unet.load_attn_procs(synthetic_lora(unet, r, 20 + r), adapter_name="b")
        st = unet._lora
        ops.profile_begin()
        st.realise()
        prof = ops.profile_end()["lora"]
        kernel = []
        for _ in range(args.repeats):
            ops.profile_begin()
            st.realise()
            kernel.append(ops.profile_end()["lora"]["ms"])
        ms = statistics.median(kernel)
        switch = [wall_ms(lambda i=i: unet.set_adapters(["a", "b"][i % 2])) for i in range(args.repeats)]
        scale = [wall_ms(lambda i=i: unet._set_lora_scale(0.5 + 0.25 * (i % 2))) for i in range(args.repeats)]
        unet._set_lora_scale(1.0)
        res["ranks"][r] = {"apply_ms": spread(kernel), "bytes": prof["work"],
                           "share_of_3.35TB/s": round(prof["work"] / (ms * 1e-3) / (HBM_TBS * 1e12), 3),
                           "set_adapters_ms": spread(switch), "scale_change_ms": spread(scale),
                           "snapshot_bytes": st.snapshot_bytes(), "targets": len(st.snap)}
        unet.unload_lora_weights()

    # graphed SDXL 1024^2 step, LoRA realised (weight 1) against none (weight 0), alternated
    r = max(args.ranks)
    unet.load_attn_procs(synthetic_lora(unet, r, 7), adapter_name="a")
    g = torch.Generator().manual_seed(0)
    ctx = torch.randn(1, 77, 2048, generator=g).to(torch.bfloat16)
    added = {"text_embeds": torch.randn(1, 1280, generator=g).to(torch.bfloat16),
             "time_ids": torch.tensor([[1024., 1024., 0, 0, 1024., 1024.]])}
    lat = torch.randn(1, 4, 128, 128, generator=g)
    pipe = StableDiffusionPipeline(unet, DDIMScheduler(**DDIM))
    run = dict(prompt_embeds=ctx, latents=lat, num_inference_steps=args.steps, guidance_scale=5.0,
               added_cond_kwargs=added)
    times = {"lora": [], "none": []}
    for i in range(2 * args.repeats + 2):
        kind = ("none", "lora")[i % 2]
        unet.set_adapters("a", 1.0 if kind == "lora" else 0.0)
        pipe(**run)  # warm (the first round captures the graph)
        ms = event_ms(lambda _: pipe(**run), 1) / args.steps
        if i >= 2:
            times[kind].append(ms)
    res["sdxl_1024_step_ms"] = {k: spread(v) for k, v in times.items()}
    unet.unload_lora_weights()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
