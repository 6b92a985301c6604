"""Multi-GPU parity under pytest: the NCCL + CUDA-kernel head-parallel path (tests/multi_gpu/tp_check.py), the fused
one-shot all-reduce kernel (tests/multi_gpu/fused_allreduce_check.py) and the sequence-sharded decode
(tests/multi_gpu/seqshard_check.py), each launched with torch.distributed.run on the GPUs of this box.  Skipped on a
one-GPU box; collected by `pytest -m gpu` so the evidence shows up in the driver's GPU test record.  The gloo/CPU twin
of the host logic is tests/test_tp_gloo.py."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_GPUS = torch.cuda.device_count() if torch.cuda.is_available() else 0


def _torchrun(script, world, port, marker, timeout=420, extra_env=None):
    env = dict(os.environ, **(extra_env or {}))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tests", "multi_gpu", script)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, env=env, cwd=ROOT)
    out = r.stdout + r.stderr
    assert r.returncode == 0 and marker in out, out[-4000:]
    return [ln for ln in out.splitlines() if marker in ln][-1]


def _worlds():
    return sorted({2, N_GPUS}) if N_GPUS >= 2 else [2]


@pytest.mark.skipif(N_GPUS < 2, reason="needs >= 2 GPUs")
@pytest.mark.parametrize("world", _worlds())
def test_head_parallel_shards_match_single_gpu_nccl(world):
    if world > N_GPUS:
        pytest.skip(f"needs {world} GPUs")
    _torchrun("tp_check.py", world, 29511 + world, "TP_CHECK_OK")


@pytest.mark.skipif(N_GPUS < 2, reason="needs >= 2 GPUs")
@pytest.mark.parametrize("world", _worlds())
def test_fused_allreduce_kernel(world):
    if world > N_GPUS:
        pytest.skip(f"needs {world} GPUs")
    _torchrun("fused_allreduce_check.py", world, 29531 + world, "FUSED_AR_OK")


@pytest.mark.skipif(N_GPUS < 2, reason="needs >= 2 GPUs")
@pytest.mark.parametrize("world", _worlds())
def test_sequence_sharded_decode_matches_single_gpu(world):
    if world > N_GPUS:
        pytest.skip(f"needs {world} GPUs")
    _torchrun("seqshard_check.py", world, 29551 + world, "SEQSHARD_OK")
