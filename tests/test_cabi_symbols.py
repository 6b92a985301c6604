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
