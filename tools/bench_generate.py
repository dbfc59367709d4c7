"""Cost of on-device sampling in Qwen2-VL-7B generate() (synthetic weights, 512-token text prompt, 128 new tokens,
B = 1, 8, 32). Prints one JSON line:
  * the GPU's name, power limit and max SM clock, read in the same run;
  * b200mix_sample_tokens on [B, 152064] fp32 logits, greedy + penalty and sampling (top_k=50, top_p=0.9, T=0.7,
    penalty 1.05): CUDA-event time over many launches, the bytes it must read (the logits once, plus the presence
    bitmap) and the bandwidth that implies; `row_passes` is how many times the sampling path reads each row (the
    repeated reads hit L2);
  * per-token time of the graphed decode loop: plain greedy (graph replay + argmax, what generate() does without
    processors) against sampling (graph replay with the sampler inside), alternated over `--repeats` rounds;
  * device-to-host copies per generated token of a whole sampling generate() call, from a torch.profiler trace taken
    in a separate pass after the timings.
Writes nothing to the tree.

    python tools/bench_generate.py [--batches 1 8 32] [--prompt 512] [--new 128] [--repeats 3]
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

SAMPLING = dict(do_sample=True, temperature=0.7, top_k=50, top_p=0.9, repetition_penalty=1.05)
EOS, PAD = [151645, 151643], 151643  # two EOS ids and a pad id, Instruct-style


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=False).stdout.strip()
    name, power, clock = (q.split(", ") + ["?", "?", "?"])[:3]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 8, 32])
    ap.add_argument("--prompt", type=int, default=512)
    ap.add_argument("--new", type=int, default=128)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--kernel-launches", type=int, default=200)
    args = ap.parse_args()

    import torch

    from oracle.qwen2vl import QWEN2VL_CONFIGS
    from paddlemix_b200.qwen2_vl import GraphedDecodeStep, Qwen2VLForConditionalGeneration
    from paddlemix_b200.sampling import TokenSampler, resolve_generation_args

    if not torch.cuda.is_available():
        raise SystemExit("bench_generate.py needs a GPU")
    info = gpu_info()
    cfg = QWEN2VL_CONFIGS["qwen2vl_7b"]
    V = cfg["vocab_size"]
    model = Qwen2VLForConditionalGeneration(cfg).init_synthetic_weights(seed=1, device=0)
    s_args = resolve_generation_args(eos_token_id=EOS, pad_token_id=PAD, **SAMPLING)
    g_args = resolve_generation_args(repetition_penalty=1.05, eos_token_id=EOS, pad_token_id=PAD)
    g = torch.Generator().manual_seed(0)
    result = {"gpu": info, "model": "qwen2vl_7b synthetic", "prompt": args.prompt, "new_tokens": args.new, "batches": {}}

    def events(fn, n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) / n

    for B in args.batches:
        r = {}
        prompt = torch.randint(0, 150000, (B, args.prompt), generator=g)
        # ---- the sampler kernel alone ---------------------------------------------------------------------------
        logits = (torch.randn(B, V, generator=g) * 3).cuda()
        n = args.kernel_launches
        for name, a in (("greedy_penalty", g_args), ("sampling", s_args)):
            smp = TokenSampler(prompt, V, 2 * n + 8, a, 5, model.device)
            for _ in range(5):
                smp(logits)
            ms = events(lambda: smp(logits), n)
            read = B * V * 4 + B * ((V + 31) // 32) * 4
            r[f"kernel_{name}"] = {"us": round(ms * 1e3, 2), "bytes_read": read,
                                   "GBps_on_bytes_read": round(read / (ms * 1e-3) / 1e9, 1)}
        r["kernel_sampling"]["row_passes"] = 9  # max, sum, 3 top-k digits, 3 top-p digits, <= 1 inverse-CDF scan
        del logits
        # ---- graphed decode loops, alternated ---------------------------------------------------------------------
        loops = {}
        for name in ("greedy", "sampling"):
            model.cache_headroom = args.new
            out = model(input_ids=prompt, use_cache=True)
            last = out.logits[:, -1].clone()
            cache, deltas = out.past_key_values, out.rope_deltas
            del out
            smp = None
            if name == "sampling":
                smp = TokenSampler(prompt, V, args.new * (args.repeats + 1), s_args, 7, model.device)
                smp(last)
            stepper = GraphedDecodeStep(model, cache, deltas, sampler=smp)
            loops[name] = (stepper, cache, last.argmax(-1))
            torch.cuda.empty_cache()
        P = args.prompt
        times = {"greedy": [], "sampling": []}
        steps = args.new - 1
        for _ in range(args.repeats):
            for name in ("greedy", "sampling"):
                stepper, cache, first = loops[name]
                for t, t0 in zip((stepper.pos, stepper.rows, stepper.kv_lens), stepper._state0):  # rewind the cache
                    t.copy_(t0)
                cache.length = P
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                if name == "greedy":
                    tok = first
                    for _ in range(steps):
                        tok = stepper.step(tok).argmax(-1)
                else:
                    for _ in range(steps):
                        stepper.step()
                torch.cuda.synchronize()
                times[name].append((time.perf_counter() - t0) * 1e3 / steps)
        for name, v in times.items():
            r[f"ms_per_token_{name}"] = {"median": round(statistics.median(v), 3), "min": round(min(v), 3),
                                         "max": round(max(v), 3)}
        r["sampling_over_greedy"] = round(statistics.median(times["sampling"]) / statistics.median(times["greedy"]), 4)
        del loops
        torch.cuda.empty_cache()
        result["batches"][B] = r

    # ---- D2H copies per generated token, in a profiled pass of its own ----------------------------------------------
    from torch.profiler import ProfilerActivity, profile
    B = args.batches[0]
    prompt = torch.randint(0, 150000, (B, args.prompt), generator=g)
    model.generate(prompt, max_new_tokens=args.new, eos_token_id=EOS, pad_token_id=PAD, **SAMPLING)  # warm-up
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        gen = model.generate(prompt, max_new_tokens=args.new, eos_token_id=EOS, pad_token_id=PAD, **SAMPLING)
        torch.cuda.synchronize()
    d2h = sum(e.count for e in prof.key_averages() if "Memcpy DtoH" in e.key)
    n_new = gen.shape[1] - args.prompt
    result["d2h_per_token"] = {"batch": B, "tokens": n_new, "d2h_copies": d2h, "per_token": round(d2h / n_new, 3)}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
