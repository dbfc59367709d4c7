"""Guards on the compiled implicit-GEMM kernel (igemm_kernel, csrc/gemm.cu), read from `cuobjdump -sass` of the built
library; no GPU needed.

Every instantiation's k-loop - from its first HGMMA to the loop's back-branch - must be free of GPU-scope memory
barriers (MEMBAR.*.GPU), L1 invalidates (CCTL.IVALL) and local-memory traffic (LDL / STL spills). The TMA producer's
loop must be free of the first two, and no mbarrier wait may be followed by an L1 invalidate. A cluster-scope
release / acquire on the ring's mbarriers compiles to exactly these instructions and stalls the tensor cores once per
k-block; the ring is written only by TMA and read only by wgmma, so it needs neither.
"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "paddlemix_b200", "libb200mix.so")

INSN = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;")
BRANCH = re.compile(r"^(?:@!?U?P\w+\s+)?BRA(?:\.\w+)*\s+(0x[0-9a-f]+)")
FENCE = re.compile(r"MEMBAR\.[\w.]*GPU|CCTL\.IVALL")
SPILL = re.compile(r"(?:^|\s)(?:LDL|STL)(?:\.\w+)*\s")


def _cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe:
        return exe
    cand = "/usr/local/cuda/bin/cuobjdump"
    return cand if os.path.exists(cand) else None


def _igemm_kernels():
    """{mangled name: [(address, instruction text)]} of every igemm_kernel instantiation in the library."""
    exe = _cuobjdump()
    if exe is None or not os.path.exists(LIB):
        pytest.skip("needs the built library and cuobjdump")
    sass = subprocess.run([exe, "-sass", LIB], capture_output=True, text=True, check=True).stdout
    kernels = {}
    for chunk in re.split(r"\n\s*Function : ", sass)[1:]:
        name = chunk.split("\n", 1)[0].strip()
        if "igemm_kernel" not in name:
            continue
        kernels[name] = [(int(m.group(1), 16), m.group(2).strip()) for m in INSN.finditer(chunk)]
    assert kernels, "no igemm_kernel in the library"
    return kernels


def _branch_target(text):
    m = BRANCH.match(text)
    return int(m.group(1), 16) if m and m.group(1) else None


def _loop_around(ins, first):
    """(start, end) indices of the innermost loop closing over instruction `first`: the first branch after it that
    jumps back to or before it."""
    addr = ins[first][0]
    for i in range(first + 1, len(ins)):
        tgt = _branch_target(ins[i][1])
        if tgt is not None and tgt <= addr:
            start = next(j for j, (a, _) in enumerate(ins) if a >= tgt)
            return start, i
    raise AssertionError(f"no back-branch after {ins[first]}")


@pytest.fixture(scope="module")
def kernels():
    return _igemm_kernels()


def test_every_instantiation_found(kernels):
    # 7 tile widths without clusters, 7 x 3 (plain, LayerNorm consumer, LayerNorm producer) with
    assert len(kernels) >= 28, sorted(kernels)


def test_kloop_has_no_fence_and_no_spill(kernels):
    bad = {}
    for name, ins in kernels.items():
        first = next(i for i, (_, s) in enumerate(ins) if s.startswith("HGMMA"))
        lo, hi = _loop_around(ins, first)
        body = [s for _, s in ins[lo:hi + 1]]
        assert any(s.startswith("HGMMA") for s in body)
        hits = [s for s in body if FENCE.search(s) or SPILL.search(s)]
        if hits:
            bad[name] = hits
    assert not bad, bad


def test_producer_loop_has_no_fence(kernels):
    bad = {}
    for name, ins in kernels.items():
        first = next(i for i, (_, s) in enumerate(ins) if s.startswith("UTMALDG"))
        lo, hi = _loop_around(ins, first)
        hits = [s for _, s in ins[lo:hi + 1] if FENCE.search(s)]
        if hits:
            bad[name] = hits
    assert not bad, bad


def test_no_mbarrier_wait_invalidates_l1(kernels):
    bad = {}
    for name, ins in kernels.items():
        for i, (_, s) in enumerate(ins[:-1]):
            if "TRYWAIT" in s and "CCTL.IVALL" in ins[i + 1][1]:
                bad.setdefault(name, []).append(hex(ins[i][0]))
    assert not bad, bad
