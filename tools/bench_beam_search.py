"""Cost of on-device beam search in Qwen2-VL-7B generate() (synthetic weights, 512-token text prompt, 128 new tokens,
B = 1 and 8 prompts with num_beams = 4). Prints one JSON line:
  * the GPU's name, power limit and max SM clock, read in the same run;
  * b200mix_beam_search_step on [B * nb, 152064] fp32 logits (repetition penalty 1.05): CUDA-event time over many
    launches, the bytes it must read (the logits once, plus the presence bitmaps) and the bandwidth that implies;
  * b200mix_kv_reorder of new - 1 = 127 generated positions (an upper bound on any reorder of the run), every beam
    taking another beam's history: time against the bytes it moves (every staged row read once, every moved row written once, 28 layers x K and V);
  * per-token time of the graphed decode loop: beam search (graph replay with selection and cache reorder inside)
    against greedy decoding of the same B * nb rows (graph replay + argmax), alternated over `--repeats` rounds;
  * device-to-host copies per generated token of a whole beam-search generate() call, from a torch.profiler trace taken
    in a separate pass after the timings.
Writes nothing to the tree.

    python tools/bench_beam_search.py [--batches 1 8] [--beams 4] [--prompt 512] [--new 128] [--repeats 3]
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

PENALTY = 1.05


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=False).stdout.strip()
    name, power, clock = (q.split(", ") + ["?", "?", "?"])[:3]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 8])
    ap.add_argument("--beams", type=int, default=4)
    ap.add_argument("--prompt", type=int, default=512)
    ap.add_argument("--new", type=int, default=128)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()

    import torch

    from oracle.qwen2vl import QWEN2VL_CONFIGS
    from paddlemix_b200 import ops
    from paddlemix_b200.beam_search import BEAM_INIT, WORST_INIT, BeamSearcher, expand_cache, resolve_beam_search_args
    from paddlemix_b200.qwen2_vl import GraphedDecodeStep, Qwen2VLForConditionalGeneration

    if not torch.cuda.is_available():
        raise SystemExit("bench_beam_search.py needs a GPU")
    info = gpu_info()
    cfg = QWEN2VL_CONFIGS["qwen2vl_7b"]
    V, nb = cfg["vocab_size"], args.beams
    model = Qwen2VLForConditionalGeneration(cfg).init_synthetic_weights(seed=1, device=0)
    b_args = resolve_beam_search_args(num_beams=nb, repetition_penalty=PENALTY)
    g = torch.Generator().manual_seed(0)
    result = {"gpu": info, "model": "qwen2vl_7b synthetic", "prompt": args.prompt, "new_tokens": args.new,
              "num_beams": nb, "repetition_penalty": PENALTY, "batches": {}}

    def events(fn, n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) / n

    def reset(searcher, presence0):
        B = searcher.prompt_ids.shape[0]
        searcher.arena.zero_()
        searcher.t["beam_scores"].view(B, nb)[:, 1:] = BEAM_INIT
        searcher.t["hyp_worst"].fill_(WORST_INIT)
        searcher.presence.copy_(presence0)

    for B in args.batches:
        r = {}
        rows = B * nb
        prompt = torch.randint(0, 150000, (B, args.prompt), generator=g)
        # ---- prefill once per prompt, cache expanded to B * nb rows ------------------------------------------------
        model.cache_headroom = args.new
        out = model(input_ids=prompt, use_cache=True)
        last = out.logits[:, -1].repeat_interleave(nb, 0)
        cache = expand_cache(out.past_key_values, nb)
        deltas = out.rope_deltas.repeat_interleave(nb, 0)
        del out
        searcher = BeamSearcher(prompt, V, args.new, b_args, cache, model.device)
        t = searcher.t
        presence_init = searcher.presence.clone()
        # ---- the step kernel alone --------------------------------------------------------------------------------
        logits = (torch.randn(rows, V, generator=g) * 3).cuda()
        step = lambda: ops.beam_search_step(  # noqa: E731
            logits, nb, searcher.workspace, state=t["state"], next_ids=t["ids"], beam_scores=t["beam_scores"],
            tokens=t["tokens"], parents=t["parents"], hyp_score=t["hyp_score"], hyp_step=t["hyp_step"],
            hyp_slot=t["hyp_slot"], hyp_count=t["hyp_count"], hyp_worst=t["hyp_worst"], done=t["done"],
            presence=searcher.presence, repetition_penalty=PENALTY)
        for _ in range(5):
            step()
        reset(searcher, presence_init)
        ms = events(step, args.new - 1)  # every launch an active step (the step counter stays below max_new)
        read = rows * V * 4 + rows * ((V + 31) // 32) * 4
        r["kernel_beam_step"] = {"us": round(ms * 1e3, 2), "bytes_read": read,
                                 "GBps_on_bytes_read": round(read / (ms * 1e-3) / 1e9, 1), "row_passes": 2}
        del logits
        # ---- the reorder kernel at the last step: every beam takes the next beam's history ------------------------
        n_pos = args.new - 1
        parents = torch.zeros(args.new, rows, dtype=torch.int32, device=model.device)
        parents[n_pos] = ((torch.arange(rows) + 1) % nb).to(torch.int32).cuda()
        state = torch.tensor([n_pos + 1, 0, 0, n_pos], dtype=torch.int64, device=model.device)
        done = torch.zeros(B, dtype=torch.int32, device=model.device)
        reorder = lambda: ops.kv_reorder(searcher.layer_kv, cache.k[0], nb, args.prompt, parents, state, done)  # noqa
        for _ in range(3):
            reorder()
        ms = events(reorder, 50)
        row_bytes = cache.k[0][0, 0].numel() * 2
        moved = len(cache.k) * 2 * rows * n_pos * row_bytes * 2  # staged read + write back
        r["kernel_kv_reorder_last_step"] = {"us": round(ms * 1e3, 2), "positions": n_pos, "bytes_moved": moved,
                                            "GBps": round(moved / (ms * 1e-3) / 1e9, 1)}
        # ---- graphed decode loops, alternated -----------------------------------------------------------------------
        reset(searcher, presence_init)
        searcher(last)
        beam_stepper = GraphedDecodeStep(model, cache, deltas, sampler=searcher)
        first_state = searcher.arena.clone()
        first_presence = searcher.presence.clone()
        out = model(input_ids=prompt.repeat_interleave(nb, 0), use_cache=True)
        g_cache, g_first = out.past_key_values, out.logits[:, -1].argmax(-1)
        greedy_stepper = GraphedDecodeStep(model, g_cache, out.rope_deltas)
        del out
        torch.cuda.empty_cache()
        loops = {"greedy": (greedy_stepper, g_cache), "beam_search": (beam_stepper, cache)}
        P = args.prompt
        times = {"greedy": [], "beam_search": []}
        steps = args.new - 1
        for _ in range(args.repeats):
            for name in ("greedy", "beam_search"):
                stepper, c = loops[name]
                for x, x0 in zip((stepper.pos, stepper.rows, stepper.kv_lens), stepper._state0):  # rewind the cache
                    x.copy_(x0)
                c.length = P
                if name == "beam_search":
                    searcher.arena.copy_(first_state)
                    searcher.presence.copy_(first_presence)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                if name == "greedy":
                    tok = g_first
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
        r["beam_search_over_greedy"] = round(statistics.median(times["beam_search"]) /
                                             statistics.median(times["greedy"]), 4)
        r["rows"] = rows
        del loops, greedy_stepper, beam_stepper, g_cache, cache, searcher, presence_init
        torch.cuda.empty_cache()
        result["batches"][B] = r

    # ---- D2H copies per generated token, in a profiled pass of its own ----------------------------------------------
    from torch.profiler import ProfilerActivity, profile
    B = args.batches[0]
    prompt = torch.randint(0, 150000, (B, args.prompt), generator=g)
    kw = dict(max_new_tokens=args.new, decode_strategy="beam_search", num_beams=nb, repetition_penalty=PENALTY)
    model.generate(prompt, **kw)  # warm-up
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        gen = model.generate(prompt, **kw)
        torch.cuda.synchronize()
    d2h = sum(e.count for e in prof.key_averages() if "Memcpy DtoH" in e.key)
    n_new = gen.shape[1] - args.prompt
    result["d2h_per_token"] = {"batch": B, "tokens": n_new, "d2h_copies": d2h, "per_token": round(d2h / n_new, 3)}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
