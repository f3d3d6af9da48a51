"""CPU-side checks of the drop-in boundary: libsrj_b200.so loads, exports every symbol that
include/srj_b200.h declares, and its host-only layout entry point agrees with the oracle."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from oracle import oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _native():
    from srj_b200 import _native as N
    return N


def test_library_exports_every_declared_symbol():
    N = _native()
    hdr = open(os.path.join(ROOT, "include", "srj_b200.h")).read()
    declared = set(re.findall(r"SRJ_API[^;]*?\b(srj_[a-z0-9_]+)\s*\(", hdr))
    assert len(declared) >= 17
    lib = N.lib()
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in srj_b200.h but not exported"
    assert declared == set(N.SYMBOLS), "python binding table and header disagree"
    assert b"sm_90a" in lib.srj_version()
    assert lib.srj_get_max_stack_depth() == 8          # hash/hash.hpp:28
    assert lib.srj_status_string(-3) == b"SRJ_EOVERFLOW"


SCHEMAS = {
    "c1": [O.INT32, O.INT64, O.FLOAT64, O.BOOL8],
    "c2": [O.INT8, O.INT16, O.INT32, O.INT64, O.FLOAT32, O.FLOAT64, O.BOOL8, O.TIMESTAMP_MICROSECONDS] * 4,
    "c3": [O.INT32, O.INT64, O.DECIMAL128, O.STRING] * 64,
    "c4": [O.INT32] * 9 + [O.INT64, O.INT32] + [O.DECIMAL32] * 12,
    "pivot": [O.INT64] * 191 + [O.INT32],
    "javadoc": [O.BOOL8, O.INT16, O.DURATION_DAYS],
    "empty": [],
}


@pytest.mark.parametrize("name", sorted(SCHEMAS))
def test_layout_matches_oracle(name):
    N = _native()
    types = SCHEMAS[name]
    n = len(types)
    t = np.array(types, dtype=np.int32)
    lay = N.SrjLayout()
    st = np.zeros(max(n, 1), np.int32)
    sz = np.zeros(max(n, 1), np.int32)
    rc = N.lib().srj_compute_layout(t.ctypes.data_as(C.c_void_p), n, C.byref(lay), st.ctypes.data_as(C.c_void_p),
                                    sz.ctypes.data_as(C.c_void_p))
    assert rc == 0
    ost, osz, ovoff, ospr = O.compute_layout(types)
    assert list(st[:n]) == list(ost) and list(sz[:n]) == list(osz)
    assert (lay.validity_offset, lay.size_per_row, lay.fixed_row_size) == (ovoff, ospr, (ospr + 7) // 8 * 8)
    assert lay.num_string_columns == sum(1 for x in types if x == O.STRING)


def test_layout_rejects_nested_types():
    N = _native()
    t = np.array([O.INT32, O.LIST], dtype=np.int32)
    lay = N.SrjLayout()
    rc = N.lib().srj_compute_layout(t.ctypes.data_as(C.c_void_p), 2, C.byref(lay), None, None)
    assert rc == N.SRJ_EUNSUPPORTED
    assert b"not supported" in N.lib().srj_last_error()


def test_product_does_not_import_oracle():
    """The product path must never route through the CPU oracle."""
    pkg = os.path.join(ROOT, "spark-rapids-jni_b200")
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh", ".hpp", ".cpp", ".h")):
                src = open(os.path.join(dp, f), errors="replace").read()
                assert "oracle" not in src.replace("test_product_does_not_import_oracle", ""), f"{f} mentions the oracle"


def test_library_reads_no_environment():
    """There is one build: no kernel variant or dispatch choice may hang on an environment variable."""
    csrc = os.path.join(ROOT, "spark-rapids-jni_b200", "csrc")
    for f in sorted(os.listdir(csrc)):
        src = open(os.path.join(csrc, f), errors="replace").read()
        assert not re.search(r"\bgetenv\b", src), f"{f} calls getenv"
        assert "SRJ_KNOB" not in src, f"{f} mentions SRJ_KNOB"


def test_library_holds_the_sm90a_kernels_and_tma_sass():
    """CPU-side evidence that the shipped .so is the hand-written sm_90a path: the kernels DESIGN.md §3.5 names are
    in the cubin, and their SASS uses the bulk-copy (TMA, UBLKCP) and cp.async (LDGSTS) instructions."""
    import shutil
    import subprocess
    from srj_b200 import _native as N
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    elf = subprocess.run([cuobjdump, "-lelf", N.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in elf
    sass = subprocess.run([cuobjdump, "-sass", N.LIB_PATH], capture_output=True, text=True).stdout
    funcs = [l for l in sass.splitlines() if "Function :" in l]
    for k in ("from_rows_kernel", "from_rows_wide_kernel", "wide_group_scan_kernel", "strings_wide_kernel", "strings_from_rows_kernel", "to_rows2_kernel", "to_rows3_kernel",
              "to_rows_w_kernel", "to_rows_kernel", "row_hash_kernel", "row_hash_plain_kernel", "row_hash_stream_kernel", "row_hash_nested_kernel",
              "part_ids_kernel", "part_rank_kernel", "partition_move_tile_kernel", "ur_to_rows_kernel", "ur_from_rows_kernel", "ur_chars_kernel", "kudo_split_kernel", "kudo_assemble_kernel"):
        assert any(k in f for f in funcs), f"kernel {k} missing from the cubin"
    assert "UBLKCP" in sass, "no TMA bulk copy in the SASS"
    assert "LDGSTS" in sass, "no cp.async in the SASS"
