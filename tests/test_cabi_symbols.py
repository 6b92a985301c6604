"""The C-ABI shared library loads on a CPU-only host and exports every symbol include/duo_b200.h declares.
No compute calls here (those need a GPU)."""
import ctypes
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HDR = os.path.join(ROOT, "include", "duo_b200.h")


def _ensure_built():
    from duo_attention_b200 import _C

    if not os.path.exists(_C.LIB_PATH):
        import __graft_entry__ as g

        g.build()
    return _C


def declared_symbols():
    src = open(HDR).read()
    return sorted(set(re.findall(r"DUO_API\s+[\w\s\*]+?\b(duo_\w+)\s*\(", src)))


def test_header_symbols_exported_and_bound():
    _C = _ensure_built()
    names = declared_symbols()
    assert len(names) >= 11, names
    assert sorted(_C.SYMBOLS) == names, "python binding table out of sync with the header"
    lib = ctypes.CDLL(_C.LIB_PATH)
    for n in names:
        assert hasattr(lib, n), f"{n} not exported"
    nm = subprocess.run(["nm", "-D", "--defined-only", _C.LIB_PATH], capture_output=True, text=True).stdout
    exported = set(re.findall(r" T (duo_\w+)", nm))
    assert exported == set(names), exported ^ set(names)


def test_header_constants_match_the_binding():
    """#define values of the header == the integers the ctypes binding (and through it the host code) uses."""
    from duo_attention_b200 import _C

    src = open(HDR).read()
    defs = {k: int(v, 0) for k, v in re.findall(r"#define\s+(DUO_\w+)\s+(-?(?:0x[0-9a-fA-F]+|\d+))\s*(?:/|$)", src, re.M)}
    want = dict(DUO_DECODE_MAX_Q=_C.DECODE_MAX_Q, DUO_DECODE_MAX_Q_INT4=_C.DECODE_MAX_Q_INT4)
    for k, v in want.items():
        assert defs.get(k) == v, (k, defs.get(k), v)


def test_host_only_entry_points():
    _C = _ensure_built()
    lib = _C.load()
    assert lib.duo_version() >= 100
    assert isinstance(_C.last_error(), str)
    ws = lib.duo_workspace_bytes(1, 8, 4, 16)
    assert 1 << 20 < ws < 1 << 28
    # argument validation happens before any CUDA call
    rc = lib.duo_layer_create(None, None)
    assert rc == _C.DUO_EINVAL and "null" in _C.last_error()
    with pytest.raises(ValueError):
        _C.check(rc)


def test_sass_has_tma_and_tensor_core_instructions():
    """Static evidence that the kernels are sm_90a code using TMA (UTMALDG) and tensor cores."""
    _C = _ensure_built()
    try:
        sass = subprocess.run(["cuobjdump", "-sass", _C.LIB_PATH], capture_output=True, text=True, timeout=300).stdout
    except FileNotFoundError:
        pytest.skip("cuobjdump not available")
    assert "sm_90a" in sass
    # the SASS names of the PTX the kernels are written in: TMA tiled loads, mbarriers, wgmma (prefill),
    # setmaxnreg (warp-specialised register split), cp.async (INT4 tiles) and the mma.sync of the HBM-bound decode kernel
    for mnemonic in ("UTMALDG", "SYNCS", "HGMMA", "USETMAXREG", "LDGSTS", "HMMA"):
        assert mnemonic in sass, f"{mnemonic} missing from the SASS of libduo_b200.so"


def test_comm_entry_points_validate_before_touching_cuda():
    """duo_comm_* (experimental fused all-reduce): sizes and argument validation are host-only."""
    import ctypes as C

    _C = _ensure_built()
    lib = _C.load()
    assert lib.duo_comm_data_bytes(8, 4096, 16, _C.DT_BF16) == 2 * 8 * 16 * 4096 * 2
    assert lib.duo_comm_flag_bytes(8, 16) == 512
    assert lib.duo_comm_data_bytes(2, 4096, 16, 7) == 0  # unknown dtype
    out = C.c_void_p()
    d = _C.CommDesc()
    d.rank, d.world, d.hidden, d.max_rows, d.dtype = 0, 1, 4096, 16, _C.DT_BF16
    assert lib.duo_comm_create(C.byref(d), C.byref(out)) == _C.DUO_EINVAL  # world < 2
    d.world = 2
    d.local_state = 0x1000
    assert lib.duo_comm_create(C.byref(d), C.byref(out)) == _C.DUO_EINVAL and "peer buffer 0" in _C.last_error()
    d.data[0], d.data[1], d.flags[0], d.flags[1] = 0x10000, 0x20000, 0x30000, 0x40008
    assert lib.duo_comm_create(C.byref(d), C.byref(out)) == _C.DUO_OK
    rc = lib.duo_allreduce_add_rmsnorm(out, 0x100, None, 0x100, 0x100, None, 17, 1e-5, None)
    assert rc == _C.DUO_EOVERFLOW and "max_rows 16" in _C.last_error()
    assert lib.duo_allreduce_add_rmsnorm(out, None, None, None, None, None, 0, 1e-5, None) == _C.DUO_OK
    lib.duo_comm_destroy(out)
    # the descriptor's limits: at most 64 rows; hidden a multiple of 8 in [8, 16384]
    for field, bad, good in (("max_rows", 65, 64), ("hidden", 12, 8), ("hidden", 16392, 16384)):
        setattr(d, field, bad)
        assert lib.duo_comm_create(C.byref(d), C.byref(out)) == _C.DUO_EINVAL, (field, bad)
        assert "bad descriptor" in _C.last_error()
        setattr(d, field, good)
        assert lib.duo_comm_create(C.byref(d), C.byref(out)) == _C.DUO_OK, (field, good)
        lib.duo_comm_destroy(out)
        d.max_rows, d.hidden = 16, 4096


def _seqcomm_desc(**kw):
    """A valid duo_seqcomm_desc (fake, aligned addresses: nothing is dereferenced on the host) with `kw` applied;
    data[i] / flags[i] entries are given as data1=..., flags0=..."""
    _C = _ensure_built()
    d = _C.SeqCommDesc()
    for i in range(8):
        d.data[i], d.flags[i] = 0x100000 * (i + 1), 0x100000 * (i + 1) + 0x80000
    d.local_state, d.rank, d.world, d.max_rows = 0x1000, 0, 2, 16
    for k, v in kw.items():
        if k[:-1] in ("data", "flags"):
            getattr(d, k[:-1])[int(k[-1])] = v
        else:
            setattr(d, k, v)
    return d


def test_seqcomm_entry_points_validate_before_touching_cuda():
    """duo_seqcomm_* / duo_seq_merge: the byte-size formulas and every refusal are host-only."""
    import ctypes as C

    _C = _ensure_built()
    lib = _C.load()
    # data: float [2 slots][world][max_rows][132]; flags: one word per (row, sender), rounded up to 256 bytes
    for w, rows in ((2, 1), (3, 5), (8, 128), (8, 512)):
        assert lib.duo_seqcomm_data_bytes(w, rows) == 2 * w * rows * 132 * 4
        assert lib.duo_seqcomm_flag_bytes(w, rows) == -(-w * rows * 4 // 256) * 256
    assert lib.duo_seqcomm_flag_bytes(3, 5) == 256 and lib.duo_seqcomm_flag_bytes(3, 100) == 1280
    assert lib.duo_seqcomm_data_bytes(0, 16) == 0 and lib.duo_seqcomm_data_bytes(2, 0) == 0
    assert lib.duo_seqcomm_flag_bytes(0, 16) == 0 and lib.duo_seqcomm_flag_bytes(2, 0) == 0
    out = C.c_void_p()
    assert lib.duo_seqcomm_create(None, C.byref(out)) == _C.DUO_EINVAL and "null" in _C.last_error()
    refused = {
        "world 1": dict(world=1), "world 9": dict(world=9), "rank -1": dict(rank=-1), "rank == world": dict(rank=2),
        "max_rows 0": dict(max_rows=0), "max_rows 513": dict(max_rows=513), "no local_state": dict(local_state=None),
    }
    for what, kw in refused.items():
        out = C.c_void_p()
        assert lib.duo_seqcomm_create(C.byref(_seqcomm_desc(**kw)), C.byref(out)) == _C.DUO_EINVAL, what
        assert "bad descriptor" in _C.last_error() and not out.value, what
    peers = {"data1 missing": (1, dict(data1=None)), "data1 misaligned": (1, dict(data1=0x200008)),
             "flags0 missing": (0, dict(flags0=None)), "flags0 misaligned": (0, dict(flags0=0x180002))}
    for what, (peer, kw) in peers.items():
        out = C.c_void_p()
        assert lib.duo_seqcomm_create(C.byref(_seqcomm_desc(**kw)), C.byref(out)) == _C.DUO_EINVAL, what
        assert f"peer buffer {peer} missing or misaligned" in _C.last_error() and not out.value, what
    # only the first `world` entries are read: a missing data[2] does not matter at world 2
    assert lib.duo_seqcomm_create(C.byref(_seqcomm_desc(data2=None)), C.byref(out)) == _C.DUO_OK
    lib.duo_seqcomm_destroy(out)
    for kw in (dict(world=8, rank=7, max_rows=512), dict(flags1=0x200004)):  # the limits; 4-byte aligned flags
        assert lib.duo_seqcomm_create(C.byref(_seqcomm_desc(**kw)), C.byref(out)) == _C.DUO_OK, kw
        lib.duo_seqcomm_destroy(out)

    assert lib.duo_seqcomm_create(C.byref(_seqcomm_desc()), C.byref(out)) == _C.DUO_OK  # max_rows 16
    p = 0x100  # never dereferenced: every call below returns before a launch
    rc = lib.duo_seq_merge(out, p, p, p, 17, 4, 1, _C.DT_BF16, None)
    assert rc == _C.DUO_EOVERFLOW and "17 rows exceed" in _C.last_error() and "max_rows 16" in _C.last_error()
    rc = lib.duo_seq_merge(out, p, p, p, 3, 8, 6, _C.DT_FP16, None)  # 18 rows
    assert rc == _C.DUO_EOVERFLOW and "18 rows" in _C.last_error()
    assert lib.duo_seq_merge(out, None, None, None, 0, 8, 8, _C.DT_BF16, None) == _C.DUO_OK  # no rows
    assert lib.duo_seq_merge(out, None, None, None, 5, 8, 0, _C.DT_BF16, None) == _C.DUO_OK  # no retrieval heads
    for what, args in {"heads_used > heads_total": (1, 4, 5, _C.DT_BF16), "dtype": (1, 4, 4, 7),
                       "tokens < 0": (-1, 4, 4, _C.DT_BF16), "heads_total 0": (1, 0, 0, _C.DT_BF16),
                       "heads_used < 0": (1, 4, -1, _C.DT_BF16)}.items():
        assert lib.duo_seq_merge(out, p, p, p, *args, None) == _C.DUO_EINVAL, what
        assert "bad argument" in _C.last_error(), what
    assert lib.duo_seq_merge(out, None, p, p, 1, 4, 4, _C.DT_BF16, None) == _C.DUO_EINVAL
    assert "null buffer" in _C.last_error()
    assert lib.duo_seq_merge(None, p, p, p, 1, 4, 4, _C.DT_BF16, None) == _C.DUO_EINVAL
    lib.duo_seqcomm_destroy(out)


def test_header_is_plain_c_and_links():
    """include/duo_b200.h is usable from C99 (no torch / C++ types in the boundary) and a C program links against the
    library and calls a host-only entry point."""
    import shutil
    import tempfile

    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    _C = _ensure_built()
    src = ('#include "duo_b200.h"\n#include <stdio.h>\n'
           "int main(void) { duo_comm_desc d; duo_layer_desc l; duo_cache_state s; (void)d; (void)l; (void)s;\n"
           '  printf("%d %zu\\n", duo_version(), duo_workspace_bytes(1, 8, 4, 16)); return 0; }\n')
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "t.c")
        open(c, "w").write(src)
        exe = os.path.join(td, "t")
        libdir = os.path.dirname(_C.LIB_PATH)
        r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"),
                            c, "-o", exe, "-L", libdir, "-l:libduo_b200.so", "-Wl,-rpath," + libdir],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        out = subprocess.run([exe], capture_output=True, text=True)
        assert out.returncode == 0, out.stderr
        ver, ws = out.stdout.split()
        assert int(ver) >= 100 and int(ws) > 1 << 20
