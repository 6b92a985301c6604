"""Prefill-sized chunks on a sharer, host side: duo_attention_shared validates before touching CUDA, and row(b).attend
refuses decode-sized chunks and force_mma on a sharer before any launch."""
import ctypes as C
import types

import pytest
import torch

from duo_attention_b200 import _C
from duo_attention_b200.kv_cache import _RaggedRow


def test_duo_attention_shared_validates_before_touching_cuda():
    lib = _C.load()
    st = _C.CacheState(300, 300, 16, None)
    for args in ((None, None), (None, 0x1000), (0x1000, None)):  # a null layer or prefix handle
        rc = lib.duo_attention_shared(*args, 256, C.byref(st), 0x1000, 384, 0x2000, 64, 0.1, None, 0, None)
        assert rc == _C.DUO_EINVAL and "null argument" in _C.last_error()
    rc = lib.duo_attention_shared(0x1000, 0x1000, 256, None, 0x1000, 384, 0x2000, 64, 0.1, None, 0, None)
    assert rc == _C.DUO_EINVAL  # a null state
    rc = lib.duo_attention_shared(0x1000, 0x1000, 256, C.byref(st), None, 384, 0x2000, 64, 0.1, None, 0, None)
    assert rc == _C.DUO_EINVAL  # a null q


class _NoLaunch:
    def __getattr__(self, name):
        raise AssertionError(f"{name} was called")


def _sharer_row(group):
    """Row 1 of a stub parent, sharing the first 256 keys of row 0; nothing behind it may be launched."""
    r = _RaggedRow.__new__(_RaggedRow)
    r._parent = types.SimpleNamespace(pooled=True, _share=[None, (0, 256)], rows_changed=False)
    r._row, r.num_kv_groups, r.lib = 1, group, _NoLaunch()
    r.launch_count = 0
    return r


@pytest.mark.parametrize("group", [1, 4])
def test_sharer_refuses_decode_sized_chunks_and_force_mma(group):
    r = _sharer_row(group)
    width = (8 * group + 16) * 128
    for S in (1, 16 // group):
        qkv = torch.zeros(1, S, width, dtype=torch.bfloat16)
        with pytest.raises(ValueError, match="batched step"):
            r.attend(0, qkv, None, None, _C.ROPE_NONE, torch.empty(1, S, 8 * group, 128, dtype=torch.bfloat16))
    S = 16 // group + 1  # the smallest prefill-sized chunk
    qkv = torch.zeros(1, S, width, dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="force_mma"):
        r.attend(0, qkv, None, None, _C.ROPE_NONE, torch.empty(1, S, 8 * group, 128, dtype=torch.bfloat16),
                 force_mma=True)
    assert r.launch_count == 0 and not r._parent.rows_changed
