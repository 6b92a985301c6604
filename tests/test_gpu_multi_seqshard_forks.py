"""Multi-GPU check of forks of a sequence-sharded prompt (tests/multi_gpu/seqshard_forks_check.py), launched with
torch.distributed.run on the GPUs of this box.  Skipped on a one-GPU box; the one-GPU emulations of the ranks are
tests/test_gpu_seqshard_forks.py and tests/test_gpu_seqshard_forks_model.py."""
import pytest

from test_gpu_multi import N_GPUS, _torchrun

pytestmark = pytest.mark.gpu


@pytest.mark.skipif(N_GPUS < 2, reason="needs >= 2 GPUs")
@pytest.mark.parametrize("world", sorted({2, N_GPUS}) if N_GPUS >= 2 else [2])
def test_forks_of_a_sharded_prompt_match_single_gpu(world):
    if world > N_GPUS:
        pytest.skip(f"needs {world} GPUs")
    _torchrun("seqshard_forks_check.py", world, 29611 + world, "SEQSHARD_FORKS_OK")
