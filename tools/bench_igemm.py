"""Per-problem timing of the implicit-GEMM kernel (igemm_kernel: Linear + conv3x3) on the SDXL workload of bench.py
(batch 8, 1024^2 images -> 128^2 latents, bf16, synthetic weights).

  * the distinct igemm problems (M, N, K, taps, epilogue flavour) and their call counts are recorded from one eager
    UNet forward (ops.profile_begin / profile_end see every launch), not listed by hand;
  * every problem is rebuilt from its tag on fresh buffers and timed with CUDA events over enough launches to fill
    --min-seconds, rotating over buffer sets that together exceed the 50 MB L2, so a launch does not find its operands
    left there by the previous one;
  * printed per problem: calls per step, us, TFLOP/s from 2 M N K taps, the tile width BN the heuristic picks, its
    super-tiles (256 x BN) and rounds = super-tiles / clusters, the FLOP-weighted time of all calls, and the card's
    name, power limit and max SM clock read in the same run;
  * --other-lib PATH loads a second build of libb200mix.so and alternates the two per problem in the same process over
    --rounds rounds: median and min-max of each, which is how a kernel change is compared against its parent;
  * --force-bn 128,64 also times the --top heaviest problems with the tile width forced (b200mix_debug_force_bn);
  * --gemm-pair 0 runs every build without 2-CTA clusters (b200mix_debug_gemm_pair: each CTA loads its whole B tile,
    no multicast and no cross-CTA release of ring stages), except the folded-LayerNorm problems, which exist only
    clustered; the default 1 is the shipped schedule.
Writes nothing to the tree unless --json PATH is given.

    python tools/bench_igemm.py [--other-lib /path/to/libb200mix.so] [--rounds 3] [--force-bn 128,64] [--gemm-pair 0]
                                [--json out.json]
"""
import argparse
import json
import math
import os
import re
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

L2_SPAN_BYTES = 160 << 20  # operands + outputs of the rotating buffer sets of one problem cover at least this much
ACTS = {"act1": 1, "act2": 2, "act3": 3, "act4": 4}
BN_CANDIDATES = (256, 224, 192, 160, 128, 64, 32)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=False).stdout.strip()
    name, power, clock = (q.split(", ") + ["?", "?", "?"])[:3]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def load_lib(path):
    """A second ctypes binding of the same C ABI from another build of the library."""
    from paddlemix_b200 import _lib
    saved, _lib.LIB_PATH = _lib.LIB_PATH, path
    try:
        return _lib._load()
    finally:
        _lib.LIB_PATH = saved


def tile_schedule(m_tiles, n, kblocks, sms, force_bn=0):
    """(BN, super-tiles, rounds) as gemm.cu's pick_bn / launch_igemm choose them (a mirror for reporting only)."""
    clusters = sms // 2
    best, best_bn = 1e30, 256
    for bn in BN_CANDIDATES:
        eff = (128.0 * bn / (128.0 + bn / 2.0)) / (128.0 * 256 / 256.0)
        tiles = ((m_tiles + 1) // 2) * ((n + bn - 1) // bn)
        waves = float((tiles + clusters - 1) // clusters)
        if kblocks >= 64 and tiles > clusters and tiles % clusters:
            waves = tiles / clusters + 0.2
        cost = waves * bn / eff
        if cost < best * 0.999:
            best, best_bn = cost, bn
    bn = force_bn or best_bn
    tiles = ((m_tiles + 1) // 2) * ((n + bn - 1) // bn)
    return bn, tiles, tiles / min(clusters, tiles)


def record_problems(batch, height):
    """{tag: calls} and {tag: flop per call} of the igemm launches of one eager SDXL forward."""
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
    return {t: dict(calls=v["calls"], flop=v["work"] / v["calls"], eager_ms=v["ms"])
            for t, v in prof.items() if re.match(r"(lin|conv1|conv2|convup) ", t)}


class Problem:
    """One igemm problem rebuilt from its profile tag ("lin 8192x1280x640 bias+res", "conv1 32768x640x5760 bias")."""

    def __init__(self, tag, batch):
        import torch
        m = re.match(r"(\w+) (\d+)x(\d+)x(\d+)(?: (\S+))?$", tag)
        if not m:
            raise ValueError(f"unrecognised igemm tag {tag!r}")
        self.tag, self.kind = tag, m.group(1)
        self.M, self.N, self.K = int(m.group(2)), int(m.group(3)), int(m.group(4))
        self.flags = set((m.group(5) or "").split("+")) - {""}
        self.batch = batch
        # the folded-LayerNorm epilogues exist only in the clustered (multicast) kernel
        self.pair_only = bool(self.flags & {"ln", "stats"})
        self.act = next((ACTS[f] for f in self.flags if f in ACTS), 0)
        self.glu = next((int(f[3:]) for f in self.flags if f.startswith("glu")), 0)
        self.taps = {"lin": 1, "conv1": 9, "conv2": 9, "convup": 4}[self.kind]
        self.flop = 2.0 * self.M * self.N * self.K
        self.kblocks = self.taps * math.ceil(self.K / self.taps / 64)
        n_out = self.N // 2 if self.glu else self.N
        elem = 4 if "f32" in self.flags else 2
        span = self.M * self.K * 2 // (1 if self.kind == "lin" else self.taps) + self.N * self.K * 2 + self.M * n_out * elem
        if "res" in self.flags:
            span += self.M * n_out * 2
        self.sets = [self._make_set(torch, s) for s in range(max(2, min(24, math.ceil(L2_SPAN_BYTES / span))))]

    def _make_set(self, torch, seed):
        from paddlemix_b200 import ops
        g = torch.Generator(device="cuda").manual_seed(seed)
        bf = torch.bfloat16
        rnd = lambda *s, scale=1.0: (torch.randn(*s, generator=g, device="cuda") * scale)  # noqa: E731
        M, N, K, B = self.M, self.N, self.K, self.batch
        d = {"bias": rnd(N) if "bias" in self.flags else None}
        n_out = N // 2 if self.glu else N
        if self.kind == "lin":
            d["a"] = rnd(M, K).to(bf)
            d["w"] = rnd(N, K, scale=K ** -0.5).to(bf)
            d["res"] = rnd(M, n_out).to(bf) if "res" in self.flags else None
            d["radd"] = rnd(B, N) if "radd" in self.flags else None
            d["gate"] = rnd(B, N) if "gate" in self.flags else None
            d["out"] = torch.empty(M, n_out, device="cuda", dtype=torch.float32 if "f32" in self.flags else bf)
            if "ln" in self.flags:  # statistics of the input rows, as the producing GEMM would have left them
                af = d["a"].float()
                buf = torch.stack([af.sum(1), (af * af).sum(1)], 1).mul(ops.RowStats.SCALE).round().to(torch.int64)
                d["ln"] = (ops.RowStats(buf.contiguous(), K), d["w"].float().sum(1).contiguous(), 1e-5)
            if "stats" in self.flags:
                d["stats"] = torch.zeros(M, 2, device="cuda", dtype=torch.int64)
        else:
            cin = K // self.taps
            stride = 2 if self.kind == "conv2" else 1
            pix = M // B // (4 if self.kind == "convup" else 1) * stride * stride  # input pixels per image
            hw = math.isqrt(pix)
            assert hw * hw == pix, self.tag
            d["x"] = rnd(B, hw, hw, cin).to(bf)
            d["w"] = rnd(N, 16 if self.kind == "convup" else 9, cin, scale=K ** -0.5).to(bf)
            if self.kind != "convup":
                d["w"] = d["w"].reshape(N, 3, 3, cin)
            ho = hw * 2 if self.kind == "convup" else hw // stride
            d["res"] = rnd(B, ho, ho, N).to(bf) if "res" in self.flags else None
            d["radd"] = rnd(B, N) if "radd" in self.flags else None
            d["out"] = torch.empty(B, ho, ho, N, device="cuda", dtype=bf)
        return d

    @property
    def m_tiles(self):
        return (self.M // 4 + 127) // 128 * 4 if self.kind == "convup" else (self.M + 127) // 128

    def launch(self, i):
        from paddlemix_b200 import ops
        d = self.sets[i % len(self.sets)]
        if self.kind == "lin":
            ops.linear(d["a"], d["w"], d["bias"], act=self.act, glu=self.glu, residual=d["res"], row_add=d["radd"],
                       row_gate=d["gate"], rows_per_group=self.M // self.batch if (d["radd"] is not None or d["gate"] is not None) else 0,
                       out_fp32="f32" in self.flags, out=d["out"], stats=d.get("stats", False), ln=d.get("ln"))
        elif self.kind == "convup":
            ops.conv3x3_up2x(d["x"], d["w"], d["bias"], row_add=d["radd"], residual=d["res"], act=self.act, out=d["out"])
        else:
            ops.conv3x3(d["x"], d["w"], d["bias"], stride=2 if self.kind == "conv2" else 1, row_add=d["radd"],
                        residual=d["res"], act=self.act, out=d["out"])


def time_us(prob, lib, min_seconds, force_bn=0, gemm_pair=1):
    """Mean us per launch of `prob` through build `lib`, over enough launches to fill min_seconds."""
    import torch

    from paddlemix_b200 import ops
    saved, ops.lib = ops.lib, lib
    lib.b200mix_debug_force_bn(force_bn)
    lib.b200mix_debug_gemm_pair(1 if prob.pair_only else gemm_pair)
    try:
        def run(n):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(n):
                prob.launch(i)
            e1.record()
            e1.synchronize()
            return e0.elapsed_time(e1) * 1e-3 / n
        per = run(2 * len(prob.sets))  # warm-up of every buffer set, and the estimate that sizes the timed window
        return run(max(2 * len(prob.sets), math.ceil(min_seconds / per))) * 1e6
    finally:
        lib.b200mix_debug_force_bn(0)
        lib.b200mix_debug_gemm_pair(1)
        ops.lib = saved


def spread(v):
    return {"median": round(statistics.median(v), 2), "min": round(min(v), 2), "max": round(max(v), 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--height", type=int, default=1024)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--min-seconds", type=float, default=0.2, help="timed window per problem, build and round")
    ap.add_argument("--other-lib", default=None, help="a second build of libb200mix.so to alternate with the tree's")
    ap.add_argument("--force-bn", default="", help="comma-separated tile widths to force on the --top heaviest problems")
    ap.add_argument("--top", type=int, default=5)
    ap.add_argument("--gemm-pair", type=int, default=1, choices=[0, 1],
                    help="1: 2-CTA clusters sharing the B tile through multicast (default); 0: independent CTAs")
    ap.add_argument("--json", default=None, help="also write the result as JSON to this path")
    args = ap.parse_args()

    import torch

    from paddlemix_b200 import ops
    if not torch.cuda.is_available():
        raise SystemExit("bench_igemm.py needs a GPU")
    builds = {"tree": ops.lib}
    if args.other_lib:
        builds["other"] = load_lib(args.other_lib)
    sms = ops.lib.b200mix_num_sms()
    info = gpu_info()
    print(json.dumps({"gpu": info, "sms": sms, "gemm_pair": args.gemm_pair,
                      "builds": {"tree": ops._lib.LIB_PATH, "other": args.other_lib}}), flush=True)

    rec = record_problems(args.batch, args.height)
    order = sorted(rec, key=lambda t: -rec[t]["flop"] * rec[t]["calls"])
    forced = [int(b) for b in args.force_bn.split(",") if b]
    rows = []
    hdr = f"{'problem':44s} {'calls':>5s} {'BN':>4s} {'tiles':>6s} {'rounds':>6s}"
    for name in builds:
        hdr += f" | {name + ' us (min-max)':>26s} {'TFLOP/s':>7s}"
    print(hdr, flush=True)
    for rank, tag in enumerate(order):
        prob = Problem(tag, args.batch)
        bn, tiles, rounds = tile_schedule(prob.m_tiles, prob.N, prob.kblocks, sms)
        t = {name: [] for name in builds}
        for _ in range(args.rounds):
            for name, lib in builds.items():
                t[name].append(time_us(prob, lib, args.min_seconds, gemm_pair=args.gemm_pair))
        row = {"problem": tag, "calls": rec[tag]["calls"], "flop": prob.flop, "bn": bn, "tiles": tiles,
               "rounds": round(rounds, 2), "us": {n: spread(v) for n, v in t.items()}, "forced": {}}
        line = f"{tag:44s} {row['calls']:5d} {bn:4d} {tiles:6d} {rounds:6.2f}"
        for name in builds:
            s = row["us"][name]
            line += f" | {s['median']:9.1f} ({s['min']:.1f}-{s['max']:.1f})".ljust(29) + f" {prob.flop / s['median'] / 1e6:7.1f}"
        print(line, flush=True)
        if rank < args.top:
            for fbn in forced:
                fb, ftiles, frounds = tile_schedule(prob.m_tiles, prob.N, prob.kblocks, sms, fbn)
                for name, lib in builds.items():
                    v = [time_us(prob, lib, args.min_seconds, fbn, args.gemm_pair) for _ in range(args.rounds)]
                    row["forced"].setdefault(str(fbn), {})[name] = spread(v)
                    s = spread(v)
                    print(f"    forced BN {fb:3d} ({name}): tiles {ftiles}, rounds {frounds:.2f}, {s['median']:.1f} us "
                          f"({s['min']:.1f}-{s['max']:.1f}), {prob.flop / s['median'] / 1e6:.1f} TFLOP/s", flush=True)
        rows.append(row)
        del prob
        torch.cuda.empty_cache()

    total_flop = sum(r["flop"] * r["calls"] for r in rows)
    totals = {}
    for name in builds:
        ms = {k: sum(r["us"][name][k] * r["calls"] for r in rows) * 1e-3 for k in ("median", "min", "max")}
        totals[name] = {"igemm_ms_per_step": {k: round(v, 2) for k, v in ms.items()},
                        "tflops": round(total_flop / ms["median"] / 1e9, 1)}
    out = {"gpu": info, "sms": sms, "gemm_pair": args.gemm_pair, "batch": args.batch, "height": args.height, "rounds": args.rounds,
           "igemm_tflop_per_step": round(total_flop / 1e12, 3), "totals": totals, "problems": rows}
    print(json.dumps({k: out[k] for k in ("gpu", "igemm_tflop_per_step", "totals")}), flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
