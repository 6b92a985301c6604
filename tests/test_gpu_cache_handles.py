"""Every duo_layer handle a KV cache creates is destroyed exactly once when the cache goes away: its layer handles, the
handles of the 16-bit image of an INT4 cache, and for a ragged cache those of the parent and of every row."""
import gc

import pytest
import torch

from duo_attention_b200 import _C
from duo_attention_b200.kv_cache import DuoKVCache, DuoRaggedINT4KVCache

pytestmark = pytest.mark.gpu
D, Hq, Hkv, SINK, RECENT = 128, 8, 2, 16, 48
DEV = torch.device("cuda:0") if torch.cuda.is_available() else None


class CountingLib:
    """libduo_b200 with a record of the handles duo_layer_create* returned and duo_layer_destroy released."""

    def __init__(self, lib):
        self.lib, self.created, self.destroyed = lib, [], []

    def __getattr__(self, name):
        fn = getattr(self.lib, name)
        if name in ("duo_layer_create", "duo_layer_create_pooled"):
            def create(*args):
                rc = fn(*args)
                if rc == _C.DUO_OK:
                    self.created.append(args[-1]._obj.value)  # the handle written through the last argument
                return rc
            return create
        if name == "duo_layer_destroy":
            def destroy(h):
                self.destroyed.append(h)
                fn(h)
            return destroy
        return fn


def chunk(cache, S, g, dtype):
    out = torch.empty(cache.batch_size, S, Hq, D, dtype=dtype, device=DEV)
    qkv = torch.randn(cache.batch_size, S, (Hq + 2 * Hkv) * D, generator=g, device=DEV).to(dtype)
    cache.attend(0, qkv, None, None, _C.ROPE_NONE, out)


def static_16bit(g):
    c = DuoKVCache(1, Hq, Hkv, D, [1], 1, 256, SINK, RECENT, torch.bfloat16, DEV, stage_cap=64)
    for S in (40, 1, 1):
        chunk(c, S, g, torch.bfloat16)
    return c, 1


def growable(g):
    c = DuoKVCache(1, Hq, Hkv, D, [1], 1, 64, SINK, RECENT, torch.bfloat16, DEV, stage_cap=16, growable=True)
    for S in (40, 300, 1):  # the staging area grows, then both, then the retrieval cache
        chunk(c, S, g, torch.bfloat16)
    assert c.full_cap_list[0] >= 341 and c.stage_cap_list[0] == 300
    return c, 4  # at construction and after each growth


def int4(g):
    c = DuoKVCache(1, Hq, Hkv, D, [1], 1, 1024, SINK, RECENT, torch.float16, DEV, stage_cap=200, kv_format="int4")
    for S in (40, 3, 130, 1):  # raw first chunk (16-bit scratch), small chunk, dequantised image, decode
        chunk(c, S, g, torch.float16)
    assert c._scratch is not None and len(c._dq["handles"]) == 1
    return c, 3  # its layer, the first-chunk scratch's, the image's


def ragged_pooled_int4(g):
    c = DuoRaggedINT4KVCache.from_geometry(1, Hq, Hkv, D, [1], 2, [256, 512], SINK, RECENT, torch.float16, DEV,
                                           stage_cap=64)
    for S in (40, 200):  # row 0: raw first chunk, then a chunk on the image (and a longer staging area for every row)
        chunk(c.row(0), S, g, torch.float16)
    c.resize_row(1, 300)
    assert c.row(1)._dq is c.row(0)._dq and len(c.row(0)._dq["handles"]) == 1
    return c, 9  # 3 at construction, the scratch, 3 for the longer staging area, the image, the resized row


@pytest.mark.parametrize("build", [static_16bit, growable, int4, ragged_pooled_int4],
                         ids=["static-16bit", "growable", "int4", "ragged-pooled-int4"])
def test_every_handle_destroyed_once(build, monkeypatch):
    lib = CountingLib(_C.load())
    monkeypatch.setattr(_C, "_lib", lib)
    g = torch.Generator(device=DEV).manual_seed(0)
    cache, creates = build(g)
    torch.cuda.synchronize()
    assert len(lib.created) == creates
    for h in cache.handles:  # created once more than destroyed: a destroyed handle's address may be handed out again
        assert lib.created.count(h) == lib.destroyed.count(h) + 1
    del cache
    gc.collect()
    assert sorted(lib.destroyed) == sorted(lib.created), "handles leaked or destroyed twice"
