"""Open-Sora text-to-video sampling cost: STDiT2-XL (qk_norm, synthetic weights), 16 frames at 512^2 (latent
16 x 64 x 64), 120 caption tokens, B = 1 and 4 (2 and 8 model rows under CFG). Prints one JSON line:
  * the GPU's name, power limit and maximum SM clock, read in the same run;
  * ms per step of OpenSoraPipeline's loop (forward + IDDPM step) against the bare STDiT2 forward at the same rows,
    alternated over `--repeats` rounds: median, min, max;
  * the iddpm_step kernel's time from CUDA events over 200 launches, its bytes and their rate against the H100 SXM
    data-sheet 3.35 TB/s;
  * the SD-VAE decode of B*16 frames at 512^2, micro-batch 1 and all frames at once.
Writes nothing to the tree.

    python tools/bench_opensora.py [--steps 5] [--repeats 3] [--batches 1,4]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_TBS = 3.35


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=False).stdout.strip()
    name, power, clock = (q.split(", ") + ["?", "?", "?"])[:3]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def wall_ms(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def stats(v):
    return {"median": round(statistics.median(v), 3), "min": round(min(v), 3), "max": round(max(v), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5, help="timed sampling steps per variant and round")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--batches", default="1,4")
    args = ap.parse_args()

    import torch

    from oracle.stdit2 import STDIT2_CONFIGS
    from oracle.vae import VAE_CONFIGS
    from paddlemix_b200 import ops
    from paddlemix_b200.opensora import IDDPM, STDiT2, OpenSoraPipeline, VideoAutoencoderKL
    from paddlemix_b200.ppdiffusers.autoencoder_kl import AutoencoderKL

    if not torch.cuda.is_available():
        raise SystemExit("bench_opensora needs a GPU")
    res = {"gpu": gpu_info(), "geometry": "STDiT2-XL qk_norm, 16 x 512^2 (latent 16x64x64), 120 tokens"}
    model = STDiT2(STDIT2_CONFIGS["stdit2_xl"]).init_synthetic_weights(seed=1, device=0)
    g = torch.Generator(device="cuda").manual_seed(2)
    model.y_embedding = (torch.randn(120, 4096, generator=g, device="cuda") * 0.02).to(torch.bfloat16)
    T, H = 16, 512
    for B in (int(b) for b in args.batches.split(",")):
        emb = torch.randn(B, 1, 120, 4096, generator=g, device="cuda") * 0.5
        lat = torch.randn(B, 4, T, H // 8, H // 8, generator=g, device="cuda")
        sched = IDDPM(num_sampling_steps=100, cfg_scale=7.0, cfg_channel=3)
        sched.indices = lambda: range(99, 99 - args.steps, -1)  # the first `steps` steps of the 100-step loop
        pipe = OpenSoraPipeline(model, sched)
        x2 = torch.cat([lat, lat])
        y2 = torch.cat([emb, model.null_caption(B).float()]).to(torch.bfloat16)
        sizes = {k: torch.full((2 * B,), v, device="cuda") for k, v in
                 dict(num_frames=float(T), height=float(H), width=float(H), ar=1.0, fps=24.0).items()}
        t2 = torch.full((2 * B,), 999.0, device="cuda")

        def loop():
            pipe(emb, num_frames=T, height=H, width=H, latents=lat, generator=torch.Generator().manual_seed(0))

        def forward():
            for _ in range(args.steps):
                model(x2, t2, y2, None, **sizes)
        loop(), forward()  # warm-up of every shape
        lo, fw = [], []
        for _ in range(args.repeats):
            lo.append(wall_ms(loop) / args.steps)
            fw.append(wall_ms(forward) / args.steps)
        # the step kernel alone
        out = model(x2, t2, y2, None, **sizes)
        x = lat.clone()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        sched.step(out, 50, x, seed=1, out=x)
        e0.record()
        for i in range(200):
            sched.step(out, 50, x, seed=i, out=x)
        e1.record()
        e1.synchronize()
        k_us = e0.elapsed_time(e1) / 200 * 1e3
        C, N = 4, T * (H // 8) ** 2
        nbytes = B * N * 4 * (2 * C + 3 + C + C)  # cond eps+var, uncond guided eps, x in, x out
        # the decode of B*16 frames
        dec = {}
        vae = AutoencoderKL(**VAE_CONFIGS["sd_vae"]).init_synthetic_weights(seed=3, device=0)
        for mb in (1, None):
            v = VideoAutoencoderKL(vae, micro_batch_size=mb)
            v.decode(lat[:, :, :2])
            dec["mb1" if mb else "all"] = round(wall_ms(lambda: v.decode(lat)), 1)
        torch.cuda.empty_cache()
        res[f"B{B}"] = {"model_rows": 2 * B, "loop_ms_per_step": stats(lo), "forward_ms": stats(fw),
                        "step_overhead_ms": round(statistics.median(lo) - statistics.median(fw), 3),
                        "iddpm_step_us": round(k_us, 2), "iddpm_step_MB": round(nbytes / 1e6, 2),
                        "iddpm_step_TBps": round(nbytes / (k_us * 1e-6) / 1e12, 3),
                        "iddpm_step_share_of_3.35TBps": round(nbytes / (k_us * 1e-6) / 1e12 / HBM_TBS, 3),
                        "vae_decode_ms": dec, "frames": B * T}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
