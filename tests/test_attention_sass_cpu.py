"""Guard on the compiled attention kernel (attn_kernel, csrc/attention.cu), read from `cuobjdump -sass` of the built
library; no GPU needed. No instantiation may touch local memory (LDL / STL): a spilled score, probability or output
register would put a local-memory round trip into the softmax that is meant to run under the other warpgroup's MMAs."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "paddlemix_b200", "libb200mix.so")
INSN = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;")
LOCAL = re.compile(r"(?:^|\s)(?:LDL|STL)(?:\.\w+)*\s")


def _attn_kernels():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe) or not os.path.exists(LIB):
        pytest.skip("needs the built library and cuobjdump")
    sass = subprocess.run([exe, "-sass", LIB], capture_output=True, text=True, check=True).stdout
    kernels = {}
    for chunk in re.split(r"\n\s*Function : ", sass)[1:]:
        name = chunk.split("\n", 1)[0].strip()
        if "attn_kernel" in name:
            kernels[name] = [m.group(2).strip() for m in INSN.finditer(chunk)]
    return kernels


def test_no_attention_instantiation_uses_local_memory():
    kernels = _attn_kernels()
    # D = 64 with 128- and 64-key blocks, D = 128, D = 192
    assert len(kernels) == 4, sorted(kernels)
    assert all(any(s.startswith("HGMMA") for s in ins) for ins in kernels.values())
    bad = {name: [s for s in ins if LOCAL.search(s)] for name, ins in kernels.items()}
    assert not any(bad.values()), bad
