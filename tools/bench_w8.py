"""Weight-only int8 against bf16 on the Qwen2-VL-7B decoder (synthetic weights). Prints one JSON line:
  * the GPU's name, power limit and max SM clock, read in the same run;
  * per-kernel CUDA-event time of b200mix_linear_w8 against b200mix_linear on the bf16 weight for the four projections
    of a layer (q|k|v + bias, o + residual, gate|up + SwiGLU, down + residual). Both int8 paths are timed at
    M = 1 .. 64 (the weight-streaming kernel and the expand + wgmma path, forced with the debug hook), so the crossover
    in linear_w8.cu can be read off; the default path alone at M = 128, 512, 3072. Bytes moved = weights + scales +
    activations + outputs (+ residual), as the algorithm needs them; the fraction is of 3.35 TB/s (H100 SXM data sheet).
    Each launch reads a different copy of the weights (copies together > 160 MB, larger than L2);
  * graphed greedy decode ms/token (512-token text prompt, 128 new tokens, B = 1 / 8 / 32), bf16 against int8, medians of
    alternated rounds with min / max; and, report-only, how many of the greedy tokens the two models agree on;
  * prefill tokens/s at bench.py's Qwen2-VL config (4 x (448x448 image + 512 text tokens)), alternated rounds;
  * device bytes of the decoder layers' weights in both modes (and the int8 mode's shared workspace).
Writes nothing to the tree.

    python tools/bench_w8.py [--batches 1 8 32] [--prompt 512] [--new 128] [--repeats 3]
"""
import argparse
import ctypes
import json
import math
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BPS = 3.35e12
PROJ = ("qkv", "o", "gu", "down")


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=False).stdout.strip()
    name, power, clock = (q.split(", ") + ["?", "?", "?"])[:3]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def events(fn, n):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(n):
        fn(i)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / n


def kernel_section(cfg, ops, lib):
    import torch
    bf16 = torch.bfloat16
    H, I = cfg["hidden_size"], cfg["intermediate_size"]
    kv = cfg["num_key_value_heads"] * (H // cfg["num_attention_heads"])
    shapes = {"qkv": (H + 2 * kv, H, "bias"), "o": (H, H, "res"), "gu": (2 * I, H, "swiglu"), "down": (H, I, "res")}
    ws = torch.empty(max(n * k for n, k, _ in shapes.values()), device="cuda", dtype=bf16)
    g = torch.Generator(device="cuda").manual_seed(0)
    out = {}
    for name, (N, K, epi) in shapes.items():
        w = torch.randn(N, K, generator=g, device="cuda") * K ** -0.5
        copies = max(1, math.ceil(160e6 / (N * K)))
        w8 = [ops.quantize_w8(w, ws) for _ in range(copies)]
        wb = [w.to(bf16) for _ in range(max(1, math.ceil(160e6 / (2 * N * K))))]
        del w
        bias = torch.randn(N, generator=g, device="cuda")
        r = {}
        for M in (1, 8, 16, 32, 64, 128, 512, 3072):
            a = torch.randn(M, K, generator=g, device="cuda").to(bf16)
            res = torch.randn(M, N, generator=g, device="cuda").to(bf16)
            kw = dict(bias=dict(bias=bias), res=dict(residual=res), swiglu=dict(glu=2))[epi]
            n_out = N // 2 if epi == "swiglu" else N
            act_bytes = M * K * 2 + M * n_out * 2 + (M * N * 2 if epi == "res" else 0)
            n = max(20, min(200, int(2e9 / (N * K * max(1, M // 64)))))

            def timed(ws_list, byte_w, small_max=None):
                if small_max is not None:
                    lib.b200mix_debug_w8_small_max(small_max)
                try:
                    for i in range(3):
                        ops.linear(a, ws_list[i % len(ws_list)], **kw)
                    ms = events(lambda i: ops.linear(a, ws_list[i % len(ws_list)], **kw), n)
                finally:
                    lib.b200mix_debug_w8_small_max(-1)
                b = byte_w + act_bytes
                return {"us": round(ms * 1e3, 2), "bytes": b, "frac_of_3.35TBps": round(b / (ms * 1e-3) / HBM_BPS, 3),
                        "tflops": round(2.0 * M * N * K / (ms * 1e-3) / 1e12, 1)}
            row = {"bf16": timed(wb, 2 * N * K)}
            if M <= 64:
                row["w8_small"] = timed(w8, N * K + 4 * N, 1 << 30)
                row["w8_large"] = timed(w8, N * K + 4 * N, 0)
            else:
                row["w8"] = timed(w8, N * K + 4 * N)
            best = min(v["us"] for k, v in row.items() if k != "bf16")
            row["w8_over_bf16"] = round(best / row["bf16"]["us"], 3)
            r[M] = row
            del a, res
        out[name] = {"N": N, "K": K, "epilogue": epi, "M": r}
        del w8, wb
        torch.cuda.empty_cache()
    return out


def layer_bytes(model):
    tot = 0
    for L in model.decoder.layers:
        for n in PROJ:
            w = L[n]
            tot += (w.q.nbytes + w.scale.nbytes) if hasattr(w, "q") else w.nbytes
    return tot


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 8, 32])
    ap.add_argument("--prompt", type=int, default=512)
    ap.add_argument("--new", type=int, default=128)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--prefill-steps", type=int, default=10)
    args = ap.parse_args()

    import torch

    from oracle.qwen2vl import QWEN2VL_CONFIGS
    from paddlemix_b200 import ops
    from paddlemix_b200._lib import lib
    from paddlemix_b200.qwen2_vl import GraphedDecodeStep, Qwen2VLForConditionalGeneration

    if not torch.cuda.is_available():
        raise SystemExit("bench_w8.py needs a GPU")
    lib.b200mix_debug_w8_small_max.argtypes, lib.b200mix_debug_w8_small_max.restype = [ctypes.c_int], None
    result = {"gpu": gpu_info(), "model": "qwen2vl_7b synthetic"}
    cfg = QWEN2VL_CONFIGS["qwen2vl_7b"]
    ops.init(0)
    result["kernels"] = kernel_section(cfg, ops, lib)
    torch.cuda.empty_cache()

    models = {"bf16": Qwen2VLForConditionalGeneration(cfg).init_synthetic_weights(seed=1, device=0)}
    torch.cuda.empty_cache()
    models["w8"] = Qwen2VLForConditionalGeneration(dict(cfg, quant_type="weight_only_int8")).init_synthetic_weights(
        seed=1, device=0)
    torch.cuda.empty_cache()
    ws = models["w8"].decoder.layers[0]["qkv"].workspace
    result["decoder_layer_weight_bytes"] = {"bf16": layer_bytes(models["bf16"]), "w8": layer_bytes(models["w8"]),
                                            "w8_shared_workspace": ws.nbytes}
    result["decoder_layer_weight_bytes"]["ratio"] = round(result["decoder_layer_weight_bytes"]["w8"] /
                                                          result["decoder_layer_weight_bytes"]["bf16"], 4)

    # ---- graphed greedy decode, alternated -----------------------------------------------------------------------
    g = torch.Generator().manual_seed(0)
    result["decode"] = {}
    for B in args.batches:
        prompt = torch.randint(0, 150000, (B, args.prompt), generator=g)
        loops = {}
        for name, model in models.items():
            model.cache_headroom = args.new
            out = model(input_ids=prompt, use_cache=True)
            first = out.logits[:, -1].argmax(-1)
            stepper = GraphedDecodeStep(model, out.past_key_values, out.rope_deltas)
            loops[name] = (stepper, out.past_key_values, first)
            del out
        steps = args.new - 1
        times, toks = {n: [] for n in models}, {}
        for rnd in range(args.repeats):
            for name in models:
                stepper, cache, first = loops[name]
                for t, t0 in zip((stepper.pos, stepper.rows, stepper.kv_lens), stepper._state0):  # rewind the cache
                    t.copy_(t0)
                cache.length = args.prompt
                seq = [first]
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                tok = first
                for _ in range(steps):
                    tok = stepper.step(tok).argmax(-1)
                    seq.append(tok)
                torch.cuda.synchronize()
                times[name].append((time.perf_counter() - t0) * 1e3 / steps)
                if rnd == 0:
                    toks[name] = torch.stack(seq, 1).cpu()
        r = {f"ms_per_token_{n}": {"median": round(statistics.median(v), 3), "min": round(min(v), 3),
                                   "max": round(max(v), 3)} for n, v in times.items()}
        r["w8_over_bf16"] = round(statistics.median(times["w8"]) / statistics.median(times["bf16"]), 4)
        same = toks["w8"] == toks["bf16"]
        first_diff = [int((~row).int().argmax()) if not bool(row.all()) else row.numel() for row in same]
        r["greedy_agreement"] = {"tokens_equal": round(same.float().mean().item(), 4),
                                 "median_first_divergence": statistics.median(first_diff), "of": args.new}
        result["decode"][B] = r
        del loops
        torch.cuda.empty_cache()

    # ---- prefill at bench.py's Qwen2-VL config, alternated -------------------------------------------------------
    B, n_img_tok, n_txt = 4, 256, 510
    grid = [[1, 32, 32]] * B
    c = models["bf16"].config
    pv = torch.randn(B * 1024, 1176, generator=g).to(torch.bfloat16).cuda()
    rows = [[c.vision_start_token_id] + [c.image_token_id] * n_img_tok + [c.vision_end_token_id] +
            torch.randint(0, 151643, (n_txt,), generator=g).tolist() for _ in range(B)]
    ids_h = torch.tensor(rows)
    S = ids_h.shape[1]
    pos, _ = models["bf16"].get_rope_index(ids_h, torch.tensor(grid))
    cos, sin = models["bf16"]._mrope_tables(pos)
    ids_d = ids_h.cuda().reshape(-1)
    idx_d = (ids_h.reshape(-1) == c.image_token_id).nonzero().reshape(-1).cuda()
    ptimes = {n: [] for n in models}
    for name, model in models.items():  # warm-up
        for _ in range(3):
            model.prefill_device(ids_d, B, S, cos, sin, pv, grid, idx_d)
    for _ in range(args.repeats):
        for name, model in models.items():
            ms = events(lambda i: model.prefill_device(ids_d, B, S, cos, sin, pv, grid, idx_d), args.prefill_steps)
            ptimes[name].append(B * S / (ms * 1e-3))
    result["prefill_tokens_per_sec"] = {n: {"median": round(statistics.median(v), 1), "min": round(min(v), 1),
                                            "max": round(max(v), 1)} for n, v in ptimes.items()}
    result["prefill_tokens_per_sec"]["tokens"] = B * S
    print(json.dumps(result))


if __name__ == "__main__":
    main()
