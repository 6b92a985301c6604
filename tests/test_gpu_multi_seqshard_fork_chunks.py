"""Multi-GPU check of prefill-sized chunks on forks of a sequence-sharded prompt
(tests/multi_gpu/seqshard_fork_chunks_check.py), launched with torch.distributed.run on the GPUs of this box.  Skipped
on a one-GPU box; the one-GPU emulations of the ranks are tests/test_gpu_seqshard_fork_chunks.py and
tests/test_gpu_seqshard_fork_chunks_model.py."""
import pytest

from test_gpu_multi import N_GPUS, _torchrun

pytestmark = pytest.mark.gpu


@pytest.mark.skipif(N_GPUS < 2, reason="needs >= 2 GPUs")
@pytest.mark.parametrize("world", sorted({2, N_GPUS}) if N_GPUS >= 2 else [2])
def test_questions_on_forks_of_a_sharded_prompt_match_single_gpu(world):
    if world > N_GPUS:
        pytest.skip(f"needs {world} GPUs")
    _torchrun("seqshard_fork_chunks_check.py", world, 29631 + world, "SEQSHARD_FORK_CHUNKS_OK")
