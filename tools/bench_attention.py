"""Per-problem timing of the attention kernel (attn_kernel, csrc/attention.cu) on the SDXL workload of bench.py (batch 8,
1024^2 images -> 128^2 latents, bf16, synthetic weights), plus SD3-medium's joint attention at batch 32.

  * the distinct sdpa problems (B, heads, Sq, Sk, D, causal) and their call counts are recorded from one eager UNet
    forward (ops.profile_begin / profile_end see every launch), not listed by hand; SD3's B = 32 joint attention
    (4096 image + 154 text tokens, 24 heads of 64, 24 layers per step) is added to them;
  * every problem is timed with CUDA events over enough launches to fill --min-seconds, rotating over buffer sets that
    together exceed the 50 MB L2, so a launch does not find its operands left there by the previous one;
  * printed per problem: calls per step, us, TFLOP/s from 4 B H Sq Sk D (half of it when causal), and the card's name,
    power limit and max SM clock read in the same run;
  * --other-lib PATH loads a second build of libb200mix.so and alternates the two per problem in the same process over
    --rounds rounds (median and min-max of each), and compares the two builds' outputs bit for bit on every problem and
    on a fixed set that covers D = 128 / 192, causal, varlen, kv_lens, an additive mask and GQA.
Writes nothing to the tree unless --json PATH is given.

    python tools/bench_attention.py [--other-lib /path/to/libb200mix.so] [--rounds 3] [--json out.json]
"""
import argparse
import json
import math
import os
import re
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_igemm import gpu_info, load_lib  # noqa: E402

L2_SPAN_BYTES = 160 << 20
SD3_B32 = "attn B32 H24 Sq4250 Sk4250 D64"
TAG = re.compile(r"attn B(\d+) H(\d+) Sq(\d+) Sk(\d+) D(\d+)( causal)?$")


def flop_of(tag):
    m = TAG.match(tag)
    B, H, Sq, Sk, D = (int(m.group(i)) for i in range(1, 6))
    return 4.0 * B * H * Sq * Sk * D * (0.5 if m.group(6) else 1.0)


def record_problems(batch, height):
    """{tag: calls per step} of the sdpa launches of one eager SDXL forward, plus SD3's B = 32 joint attention."""
    import torch

    from bench import SDXL
    from paddlemix_b200 import ops
    from paddlemix_b200.ppdiffusers.unet_2d_condition import UNet2DConditionModel
    unet = UNet2DConditionModel(**SDXL).init_synthetic_weights(seed=1, device=0)
    H = height // 8
    g = torch.Generator().manual_seed(3)
    x = ops.nchw_to_nhwc(torch.randn(batch, 4, H, H, generator=g).cuda())
    added = {"text_embeds": torch.randn(batch, 1280, generator=g).to(torch.bfloat16).cuda(),
             "time_ids": torch.tensor([[float(height), float(height), 0, 0, float(height), float(height)]] * batch).cuda()}
    tt = torch.full((batch,), 981.0, device="cuda")
    ctx = torch.randn(batch, 77, 2048, generator=g).to(torch.bfloat16).cuda()
    unet.forward_nhwc(x, tt, ctx, added)
    torch.cuda.synchronize()
    ops.profile_begin()
    unet.forward_nhwc(x, tt, ctx, added)
    prof = ops.profile_end(by_tag=True)
    del unet
    torch.cuda.empty_cache()
    probs = {t: v["calls"] for t, v in prof.items() if TAG.match(t)}
    probs[SD3_B32] = 24
    return probs


class Problem:
    """One sdpa problem on contiguous [B, S, H, D] bf16 operands, optionally with GQA, kv_lens, varlen or a mask."""

    def __init__(self, tag, hkv=None, kv_lens=None, cu=None, mask=None, sets=None, seed=0):
        import torch
        m = TAG.match(tag)
        if not m:
            raise ValueError(f"unrecognised attention tag {tag!r}")
        self.tag = tag
        self.B, self.H, self.Sq, self.Sk, self.D = (int(m.group(i)) for i in range(1, 6))
        self.causal = bool(m.group(6))
        self.hkv = hkv or self.H
        self.flop = flop_of(tag)
        span = 2 * (2 * self.B * self.Sq * self.H * self.D + 2 * self.B * self.Sk * self.hkv * self.D)
        n = sets or max(2, min(16, math.ceil(L2_SPAN_BYTES / span)))
        g = torch.Generator(device="cuda").manual_seed(1000 + seed)
        bf = torch.bfloat16
        rnd = lambda *s: torch.randn(*s, generator=g, device="cuda").to(bf)  # noqa: E731
        self.sets = [dict(q=rnd(self.B, self.Sq, self.H, self.D), k=rnd(self.B, self.Sk, self.hkv, self.D),
                          v=rnd(self.B, self.Sk, self.hkv, self.D),
                          out=torch.empty(self.B, self.Sq, self.H, self.D, device="cuda", dtype=bf)) for _ in range(n)]
        self.kw = {}
        if kv_lens is not None:
            self.kw["kv_lens"] = torch.tensor(kv_lens, dtype=torch.int32, device="cuda")
        if cu is not None:
            self.kw["cu_seqlens"] = torch.tensor(cu, dtype=torch.int32, device="cuda")
        if mask is not None:
            self.kw["attn_mask"] = mask(g)

    def launch(self, i):
        from paddlemix_b200 import ops
        d = self.sets[i % len(self.sets)]
        ops.sdpa(d["q"], d["k"], d["v"], causal=self.causal, out=d["out"], **self.kw)
        return d["out"]


def time_us(prob, lib, min_seconds):
    """Mean us per launch of `prob` through build `lib`, over enough launches to fill min_seconds."""
    import torch

    from paddlemix_b200 import ops
    saved, ops.lib = ops.lib, lib
    try:
        def run(n):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(n):
                prob.launch(i)
            e1.record()
            e1.synchronize()
            return e0.elapsed_time(e1) * 1e-3 / n
        per = run(2 * len(prob.sets))
        return run(max(2 * len(prob.sets), math.ceil(min_seconds / per))) * 1e6
    finally:
        ops.lib = saved


def outputs(prob, lib):
    """The output of every buffer set of `prob` through build `lib` (copies)."""
    import torch

    from paddlemix_b200 import ops
    saved, ops.lib = ops.lib, lib
    try:
        outs = [prob.launch(i).clone() for i in range(len(prob.sets))]
        torch.cuda.synchronize()
        return outs
    finally:
        ops.lib = saved


def coverage_problems():
    """A fixed set of the kernel's other features, compared bit for bit between two builds."""
    import torch

    def keypad(B, Sk):
        def make(g):
            keep = (torch.rand(B, Sk, generator=g, device="cuda") > 0.3).float()
            keep[:, 0] = 1.0
            return ((1 - keep) * -10000.0)[:, None, None, :]
        return make

    full_bias = lambda g: torch.randn(2, 3, 300, 333, generator=g, device="cuda").to(torch.bfloat16)  # noqa: E731
    return [
        Problem("attn B2 H4 Sq1000 Sk1000 D128", sets=1, seed=1),
        Problem("attn B2 H3 Sq520 Sk700 D192", sets=1, seed=2),
        Problem("attn B2 H4 Sq700 Sk900 D64 causal", sets=1, seed=3),
        Problem("attn B1 H8 Sq900 Sk900 D128 causal", hkv=2, sets=1, seed=4),
        Problem("attn B1 H4 Sq1500 Sk1500 D64", cu=[0, 100, 613, 614, 1500], sets=1, seed=5),
        Problem("attn B1 H2 Sq1500 Sk1500 D128 causal", cu=[0, 400, 1100, 1500], sets=1, seed=6),
        Problem("attn B4 H3 Sq300 Sk700 D64", kv_lens=[700, 129, 1, 0], sets=1, seed=7),
        Problem("attn B3 H4 Sq256 Sk333 D64", mask=keypad(3, 333), sets=1, seed=8),
        Problem("attn B2 H3 Sq300 Sk333 D128", mask=full_bias, sets=1, seed=9),
        Problem("attn B2 H16 Sq1024 Sk1024 D64", hkv=4, sets=1, seed=10),
    ]


def spread(v):
    return {"median": round(statistics.median(v), 2), "min": round(min(v), 2), "max": round(max(v), 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--height", type=int, default=1024)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--min-seconds", type=float, default=0.2, help="timed window per problem, build and round")
    ap.add_argument("--other-lib", default=None, help="a second build of libb200mix.so to alternate with the tree's")
    ap.add_argument("--json", default=None, help="also write the result as JSON to this path")
    args = ap.parse_args()

    import torch

    from paddlemix_b200 import ops
    if not torch.cuda.is_available():
        raise SystemExit("bench_attention.py needs a GPU")
    ops.init(0)
    info = gpu_info()
    print(f"# {info['name']}, power limit {info['power_limit']}, max SM clock {info['max_sm_clock']}", flush=True)
    libs = {"tree": ops.lib}
    if args.other_lib:
        libs["other"] = load_lib(os.path.abspath(args.other_lib))

    calls = record_problems(args.batch, args.height)
    probs = [Problem(t, seed=i) for i, t in enumerate(sorted(calls, key=lambda t: -flop_of(t) * calls[t]))]
    rows = []
    times = {name: {p.tag: [] for p in probs} for name in libs}
    for _ in range(args.rounds):
        for p in probs:
            for name, lib in libs.items():
                times[name][p.tag].append(time_us(p, lib, args.min_seconds))

    hdr = f"{'problem':<40} {'calls':>5}"
    for name in libs:
        hdr += f" {name + ' us':>12} {'TFLOP/s':>8} {'min-max us':>17}"
    print(hdr)
    step_ms = {name: 0.0 for name in libs}
    step_flop = 0.0
    for p in probs:
        row = {"problem": p.tag, "calls_per_step": calls[p.tag], "tflop_per_call": p.flop / 1e12}
        line = f"{p.tag:<40} {calls[p.tag]:>5}"
        for name in libs:
            s = spread(times[name][p.tag])
            row[name] = dict(s, tflops=round(p.flop / (s["median"] * 1e-6) / 1e12, 1))
            if p.tag != SD3_B32:
                step_ms[name] += s["median"] * calls[p.tag] * 1e-3
            line += f" {s['median']:>12.1f} {row[name]['tflops']:>8.1f} {s['min']:>8.1f}-{s['max']:<8.1f}"
        if p.tag != SD3_B32:
            step_flop += p.flop * calls[p.tag]
        rows.append(row)
        print(line, flush=True)
    summary = {name: {"sdxl_ms_per_step": round(step_ms[name], 3),
                      "sdxl_tflops": round(step_flop / (step_ms[name] * 1e-3) / 1e12, 1)} for name in libs}
    for name, s in summary.items():
        print(f"# {name}: SDXL attention {s['sdxl_ms_per_step']} ms per step ({step_flop / 1e12:.2f} TFLOP), "
              f"{s['sdxl_tflops']} TFLOP/s")

    identical = None
    if args.other_lib:
        identical = {}
        for p in probs + coverage_problems():
            a, b = outputs(p, libs["tree"]), outputs(p, libs["other"])
            identical[p.tag + "".join(f" +{k}" for k in p.kw) + (f" Hkv{p.hkv}" if p.hkv != p.H else "")] = all(
                torch.equal(x, y) for x, y in zip(a, b))
        for t, same in identical.items():
            print(f"# bit-identical {'yes' if same else 'NO '}  {t}")
        print(f"# outputs bit-identical on {sum(identical.values())} / {len(identical)} problems")
    result = {"gpu": info, "problems": rows, "summary": summary, "bit_identical": identical}
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)
    if identical is not None and not all(identical.values()):
        sys.exit(1)


if __name__ == "__main__":
    main()
