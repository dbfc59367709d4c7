"""The path's only collective through the C ABI, on 2 GPUs (needs a machine with 2 GPUs): libb200mix creates its own NCCL
communicator (b200mix_nccl_unique_id / b200mix_comm_init) and b200mix_allgather_latents must return exactly what
torch.distributed's all_gather returns. Spawns 2 ranks; skipped with fewer than 2 GPUs."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

WORKER = r"""
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, %r)
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
from paddlemix_b200 import distributed as bdist
from paddlemix_b200.ppdiffusers.pipelines import all_gather_latents, shard_batch
bdist.init_comm(rank)
assert bdist.comm_ready()
lo, hi = shard_batch(8, rank, world)
full = torch.randn(8, 4, 128, 128, generator=torch.Generator().manual_seed(0))
mine = full[lo:hi].cuda()
got = all_gather_latents(mine)
ref = [torch.empty_like(mine) for _ in range(world)]
dist.all_gather(ref, mine)
assert torch.equal(got, torch.cat(ref, 0)) and torch.equal(got.cpu(), full)
for _ in range(3):
    assert torch.equal(all_gather_latents(mine), got)
torch.cuda.synchronize()
bdist.destroy_comm()
dist.destroy_process_group()
print("rank", rank, "ok")
""" % ROOT


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_allgather_latents_cabi_two_ranks(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                        "--master-port", "29611", str(script)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    assert "rank 0 ok" in r.stdout and "rank 1 ok" in r.stdout
