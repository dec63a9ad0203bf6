"""Compaction of the multi-GPU service under torch.distributed.run, one process per GPU, rows re-dealt over NCCL:
scripts/sharded_compact_check.py asserts that the sharded service answers as the single-GPU service through deletes and
updates that compact both.  Runs with 1 rank on a single-GPU box and with 2 (and 4 when present) ranks where the box has
them."""
import pytest

from tests.test_gpu_sharded import _run

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("world", [1, 2, 4])
def test_sharded_service_compaction_equals_single_gpu_service(world):
    import torch
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs, box has {torch.cuda.device_count()}")
    _run(world, "sharded_compact_check.py", "sharded compact check ok")
