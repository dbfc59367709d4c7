"""Where the consumer warpgroups of the implicit-GEMM kernel (igemm_kernel) spend their cycles, per problem of the SDXL
workload of bench.py (batch 8, 1024^2, bf16, synthetic weights).

  * runs a cycle-accounting build of libb200mix.so: gemm.cu compiled with -DIGEMM_CYCLES, whose consumer warpgroups
    add up clock64() intervals per CTA. Unless --lib names such a build, it is compiled from --csrc (default: the tree's
    sources) into a temporary directory; the tree is not written;
  * the problems are the igemm launches of one eager UNet forward (tools/bench_igemm.py records and rebuilds them);
    each runs --launches times on rotating buffer sets after a warm-up, then the counters are read;
  * printed per problem, as shares of a consumer warpgroup's time from its first k-block to its last epilogue:
      wait  - waiting on full_bar for a stage (the ring is empty: TMA / L2 / HBM did not keep up),
      mma   - the rest of the k-loop (issuing MMAs, waiting for the previous k-block's MMAs, releasing stages),
      epi   - the epilogue, stream-K partial exchange included;
    plus cycles per k-block (mma share over k-blocks) and cycles per epilogue (epi over the tiles or stream-K pieces).
    clock64() reads add a few instructions per k-block, so absolute cycles are a little above the shipped kernel's.
Card name, power limit and max SM clock are read in the same run. Writes nothing to the tree unless --json PATH is given.

    python tools/igemm_cycles.py [--lib /path/to/cycle-build/libb200mix.so] [--csrc DIR] [--launches 20] [--json out.json]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

SLOTS, FIELDS = 1024, 5  # gemm.cu: CYC_SLOTS x CYC_FIELDS (wait, k-loop, epilogue, pieces, k-blocks)


def build_cycle_lib(csrc, outdir):
    out = os.path.join(outdir, "libb200mix.so")
    env = dict(os.environ)
    env.setdefault("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.run(["make", "-C", csrc, "-j8", f"BUILD={os.path.join(outdir, 'build')}", f"OUT={out}",
                    "EXTRA_NVFLAGS=-DIGEMM_CYCLES"], check=True, env=env, stdout=subprocess.DEVNULL)
    return out


def read_counters(lib, reset):
    buf = (ctypes.c_ulonglong * (SLOTS * FIELDS))()
    rc = lib.b200mix_debug_igemm_cycles(buf, 1 if reset else 0)
    if rc:
        raise RuntimeError(f"b200mix_debug_igemm_cycles failed ({rc})")
    tot = [0] * FIELDS
    for s in range(SLOTS):
        for f in range(FIELDS):
            tot[f] += buf[s * FIELDS + f]
    return tot


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--height", type=int, default=1024)
    ap.add_argument("--lib", default=None, help="a libb200mix.so built with EXTRA_NVFLAGS=-DIGEMM_CYCLES")
    ap.add_argument("--csrc", default=os.path.join(ROOT, "paddlemix_b200", "csrc"), help="sources to build it from")
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import torch

    from bench_igemm import Problem, gpu_info, load_lib, record_problems
    from paddlemix_b200 import ops
    if not torch.cuda.is_available():
        raise SystemExit("igemm_cycles.py needs a GPU")
    with tempfile.TemporaryDirectory() as tmp:
        path = args.lib or build_cycle_lib(os.path.abspath(args.csrc), tmp)
        lib = load_lib(path)
        if not hasattr(lib, "b200mix_debug_igemm_cycles"):
            raise SystemExit(f"{path} is not a cycle-accounting build (-DIGEMM_CYCLES)")
        lib.b200mix_debug_igemm_cycles.argtypes = [ctypes.c_void_p, ctypes.c_int]
        lib.b200mix_debug_igemm_cycles.restype = ctypes.c_int
        info = gpu_info()
        print(json.dumps({"gpu": info, "lib": path}), flush=True)
        rec = record_problems(args.batch, args.height)
        order = sorted(rec, key=lambda t: -rec[t]["flop"] * rec[t]["calls"])
        print(f"{'problem':44s} {'calls':>5s} {'kblk':>5s} | {'wait':>6s} {'mma':>6s} {'epi':>6s} | "
              f"{'cyc/kblock':>10s} {'cyc/epilogue':>12s}", flush=True)
        rows = []
        saved, ops.lib = ops.lib, lib
        try:
            for tag in order:
                prob = Problem(tag, args.batch)
                for i in range(2 * len(prob.sets)):  # warm-up
                    prob.launch(i)
                read_counters(lib, reset=True)
                for i in range(args.launches):
                    prob.launch(i)
                wait, kloop, epi, pieces, kblocks = read_counters(lib, reset=True)
                busy = max(kloop + epi, 1)
                row = {"problem": tag, "calls": rec[tag]["calls"], "kblocks_per_tile": prob.kblocks,
                       "wait": wait / busy, "mma": (kloop - wait) / busy, "epi": epi / busy,
                       "cycles_per_kblock": (kloop - wait) / max(kblocks, 1), "cycles_per_epilogue": epi / max(pieces, 1),
                       "per_launch": [v / args.launches for v in (wait, kloop, epi)]}
                rows.append(row)
                print(f"{tag:44s} {row['calls']:5d} {prob.kblocks:5d} | {row['wait']:6.1%} {row['mma']:6.1%} "
                      f"{row['epi']:6.1%} | {row['cycles_per_kblock']:10.0f} {row['cycles_per_epilogue']:12.0f}",
                      flush=True)
                del prob
                torch.cuda.empty_cache()
        finally:
            ops.lib = saved
    # over the whole step: every problem's per-launch cycles times its calls per step
    w, k, e = (sum(r["per_launch"][i] * r["calls"] for r in rows) for i in range(3))
    step = {"wait": round(w / (k + e), 4), "mma": round((k - w) / (k + e), 4), "epi": round(e / (k + e), 4)}
    print(json.dumps({"gpu": info, "step_shares": step}), flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"gpu": info, "batch": args.batch, "height": args.height, "launches": args.launches,
                       "step_shares": step, "problems": rows}, f, indent=1)


if __name__ == "__main__":
    main()
