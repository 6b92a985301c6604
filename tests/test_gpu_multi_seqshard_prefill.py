"""Multi-GPU parity of a 1,000-token second turn on a sequence-sharded cache (tests/multi_gpu/seqshard_prefill_check.py),
launched with torch.distributed.run on the GPUs of this box.  Skipped on a one-GPU box; the one-GPU emulation of the
ranks is tests/test_gpu_seqshard_prefill.py and the gloo/CPU twin of the scattered merge is
tests/test_seqshard_prefill_gloo.py."""
import pytest

from test_gpu_multi import N_GPUS, _torchrun

pytestmark = pytest.mark.gpu


@pytest.mark.skipif(N_GPUS < 2, reason="needs >= 2 GPUs")
@pytest.mark.parametrize("world", sorted({2, N_GPUS}) if N_GPUS >= 2 else [2])
def test_sequence_sharded_second_turn_matches_single_gpu(world):
    if world > N_GPUS:
        pytest.skip(f"needs {world} GPUs")
    _torchrun("seqshard_prefill_check.py", world, 29591 + world, "SEQSHARD_PREFILL_OK")
