"""CPU checks of the JoinPrimitives surface: the JNI shim compiles against the stub headers and defines exactly six natives
(nativeSortMergeInnerJoin and nativeFilterGatherMapsByAST stay absent); the C ABI, its Python binding and the Python mirror
agree; every argument error comes back with its code before any launch; the join kernels have no subroutine call, no stack
frame and no spill."""
import ctypes as C
import os
import re
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
JNI = os.path.join(ROOT, "spark-rapids-jni_b200", "jni")
PREFIX = "Java_com_nvidia_spark_rapids_jni_JoinPrimitives_"
NATIVES = {PREFIX + m for m in ("nativeHashInnerJoin", "nativeMakeLeftOuter", "nativeMakeFullOuter", "nativeMakeSemi", "nativeMakeAnti",
                                "nativeGetMatchedRows")}
ABSENT = {PREFIX + "nativeSortMergeInnerJoin", PREFIX + "nativeFilterGatherMapsByAST"}
ABI = {"srj_hash_join_workspace_bytes", "srj_hash_inner_join_size", "srj_hash_inner_join", "srj_join_mask_workspace_bytes", "srj_join_mark",
       "srj_join_matched_counts", "srj_join_compact", "srj_join_make_outer", "srj_join_matched_rows"}
INT32, INT64, FLOAT64, STRING, LIST, DEC64, STRUCT = 3, 4, 10, 23, 24, 26, 28
KERNELS = ("join_build_kernel", "join_count_kernel", "join_retrieve_kernel", "join_mark_kernel", "join_tile_count_kernel", "join_compact_kernel",
           "join_fill_kernel", "join_matched_rows_kernel")


def test_shim_defines_exactly_the_six_natives():
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    with tempfile.TemporaryDirectory() as td:
        obj = os.path.join(td, "j.o")
        r = subprocess.run([gxx, "-std=c++17", "-Wall", "-Werror", "-fPIC", "-DSRJ_JNI_STUBS", "-c", os.path.join(JNI, "JoinPrimitivesJni.cpp"),
                            "-o", obj], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        syms = subprocess.run(["nm", "-g", "--defined-only", obj], capture_output=True, text=True).stdout
    defined = {l.split()[-1] for l in syms.splitlines() if " T " in l and l.split()[-1].startswith("Java_")}
    assert defined == NATIVES and not defined & ABSENT


def test_header_binding_and_mirror_agree():
    from srj_b200 import _native as N
    from srj_b200 import join as J
    hdr = open(os.path.join(ROOT, "include", "srj_b200.h")).read()
    declared = set(re.findall(r"SRJ_API[^;]*?\b(srj_[a-z0-9_]+)\s*\(", hdr))
    assert {d for d in declared if "join" in d} == ABI
    assert ABI <= set(N.SYMBOLS)
    for name in ABI:
        assert hasattr(N.lib(), name)
    assert int(re.search(r"#define SRJ_MAX_JOIN_KEYS (\d+)", hdr).group(1)) == 32
    methods = [m for m in vars(J.JoinPrimitives) if not m.startswith("_")]
    assert methods == ["hashInnerJoin", "makeLeftOuter", "makeFullOuter", "makeSemi", "makeAnti", "getMatchedRows"]   # Java's order
    src = open(os.path.join(ROOT, "spark-rapids-jni_b200", "srj_b200", "join.py")).read()
    assert "oracle" not in re.sub(r'""".*?"""', "", src, flags=re.S)


def _col(t=INT32, rows=4, data=16, offsets=None, mask=None, scale=0):
    from srj_b200 import _native as N
    c = N.SrjColumn()
    c.type_id, c.size, c.data, c.offsets, c.null_mask, c.scale = t, rows, data, offsets, mask, scale
    return c


def _arr(*cols):
    from srj_b200 import _native as N
    a = (N.SrjColumn * max(1, len(cols)))()
    for i, c in enumerate(cols):
        a[i] = c
    return a


def _size(left, right, nl=None, nr=None, ws=256, pairs=True):
    from srj_b200 import _native as N
    n = C.c_int64(-7)
    rc = N.lib().srj_hash_inner_join_size(_arr(*left), len(left) if nl is None else nl, _arr(*right), len(right) if nr is None else nr, 1,
                                          C.byref(n) if pairs else None, ws, None)
    return rc, n.value


@pytest.mark.parametrize("left,right,kw,want", [
    ([], [_col()], {}, "EINVAL"), ([_col()], [], {}, "EINVAL"),                                        # zero key columns
    ([_col()], [_col()], dict(pairs=False), "EINVAL"),
    ([_col(rows=-1)], [_col()], {}, "EINVAL"), ([_col(), _col(rows=3)], [_col(), _col()], {}, "EINVAL"),  # bad row counts
    ([_col()], [_col(), _col()], {}, "EINVAL"), ([_col(INT32)], [_col(INT64)], {}, "EINVAL"),            # schema mismatch
    ([_col(DEC64, scale=-2)], [_col(DEC64, scale=-3)], {}, "EINVAL"),                                  # decimal scale
    ([_col(LIST, offsets=16)], [_col(LIST, offsets=16)], {}, "EUNSUPPORTED"), ([_col(STRUCT)], [_col(STRUCT)], {}, "EUNSUPPORTED"),
    ([_col(LIST, offsets=16)], [_col(INT32)], {}, "EUNSUPPORTED"),
    ([_col()] * 33, [_col()] * 33, {}, "EUNSUPPORTED"),
    ([_col(rows=2 ** 31)], [_col(rows=2 ** 31)], {}, "EINVAL"),                                        # > INT32_MAX rows
    ([_col(data=None)], [_col()], {}, "EINVAL"), ([_col(INT64, data=20)], [_col(INT64)], {}, "EINVAL"),  # missing / misaligned
    ([_col(STRING, offsets=None)], [_col(STRING, offsets=16)], {}, "EINVAL"), ([_col(STRING, offsets=18)], [_col(STRING, offsets=16)], {}, "EINVAL"),
    ([_col(mask=66)], [_col()], {}, "EINVAL"), ([_col()], [_col()], dict(ws=None), "EINVAL"),
])
def test_inner_join_errors_need_no_device(left, right, kw, want):
    from srj_b200 import _native as N
    assert _size(left, right, **kw)[0] == getattr(N, "SRJ_" + want)


def test_an_empty_side_is_empty_before_the_schema_checks():
    from srj_b200 import _native as N
    # mismatched column counts, types and scales, and a LIST, all with an empty side: empty, as the reference returns first
    for left, right in (([_col(rows=0)], [_col(INT64), _col()]), ([_col(DEC64, rows=0, scale=1)], [_col(DEC64, scale=2)]),
                        ([_col(LIST, rows=5)], [_col(INT32, rows=0, data=None)]), ([_col(rows=0, data=None)], [_col(rows=0, data=None)])):
        assert _size(left, right, ws=None) == (N.SRJ_OK, 0)
        assert N.lib().srj_hash_inner_join(_arr(*left), len(left), _arr(*right), len(right), 0, None, None, None, None) == N.SRJ_OK


@pytest.mark.parametrize("call,want", [
    (lambda L: L.srj_join_mark(None, 4, 10, 256, None), "EINVAL"),            # a null map with entries
    (lambda L: L.srj_join_mark(18, 4, 10, 256, None), "EINVAL"),              # misaligned map
    (lambda L: L.srj_join_mark(16, -1, 10, 256, None), "EINVAL"), (lambda L: L.srj_join_mark(16, 4, -1, 256, None), "EINVAL"),
    (lambda L: L.srj_join_mark(16, 4, 2 ** 31, 256, None), "EINVAL"), (lambda L: L.srj_join_mark(16, 4, 10, None, None), "EINVAL"),
    (lambda L: L.srj_join_compact(256, -1, 1, 16, None), "EINVAL"), (lambda L: L.srj_join_compact(256, 10, 1, None, None), "EINVAL"),
    (lambda L: L.srj_join_compact(256, 10, 1, 18, None), "EINVAL"), (lambda L: L.srj_join_compact(None, 10, 0, 16, None), "EINVAL"),
    (lambda L: L.srj_join_matched_rows(16, 4, -3, 64, None), "EINVAL"), (lambda L: L.srj_join_matched_rows(16, 4, 10, None, None), "EINVAL"),
    (lambda L: L.srj_join_matched_rows(None, 4, 10, 64, None), "EINVAL"),
    (lambda L: L.srj_join_make_outer(16, 32, 4, -1, 5, 256, 0, None, 0, 64, 128, None), "EINVAL"),       # negative size
    (lambda L: L.srj_join_make_outer(16, 32, 4, 5, -1, 256, 0, None, 0, 64, 128, None), "EINVAL"),
    (lambda L: L.srj_join_make_outer(16, 32, 4, 5, 5, 256, 6, None, 0, 64, 128, None), "EINVAL"),        # unmatched > rows
    (lambda L: L.srj_join_make_outer(16, 32, 4, 5, 5, None, 1, None, 0, 64, 128, None), "EINVAL"),
    (lambda L: L.srj_join_make_outer(16, 30, 4, 5, 5, 256, 1, None, 0, 64, 128, None), "EINVAL"),
    (lambda L: L.srj_join_make_outer(16, 32, 4, 5, 5, 256, 1, 512, -1, 64, 128, None), "EINVAL"),
])
def test_helper_errors_need_no_device(call, want):
    from srj_b200 import _native as N
    assert call(N.lib()) == getattr(N, "SRJ_" + want)


def test_zero_rows_touch_nothing():
    from srj_b200 import _native as N
    lib = N.lib()
    assert lib.srj_join_compact(None, 0, 1, None, None) == N.SRJ_OK
    assert lib.srj_join_matched_rows(None, 0, 0, None, None) == N.SRJ_OK
    assert lib.srj_join_matched_rows(16, 4, 0, None, None) == N.SRJ_OK
    assert lib.srj_join_make_outer(None, None, 0, 0, 0, None, 0, None, 0, None, None, None) == N.SRJ_OK
    assert lib.srj_join_matched_counts(None, 0, None, None) == N.SRJ_OK
    assert lib.srj_join_matched_counts(None, 1, None, None) == N.SRJ_EINVAL
    assert lib.srj_hash_join_workspace_bytes(-5, -5) == lib.srj_hash_join_workspace_bytes(0, 0)


def test_mirror_raises_the_java_exceptions():
    import torch
    from srj_b200.join import GatherMap, JoinPrimitives
    for fn in (lambda: JoinPrimitives.hashInnerJoin(None, None, True), lambda: JoinPrimitives.makeSemi(None, 3),
               lambda: JoinPrimitives.makeLeftOuter(None, None, 1, 1), lambda: JoinPrimitives.getMatchedRows(None, 1)):
        with pytest.raises(TypeError):
            fn()
    m = GatherMap(torch.zeros(3, dtype=torch.int32))
    with pytest.raises(ValueError):
        JoinPrimitives.makeFullOuter(m, GatherMap(torch.zeros(2, dtype=torch.int32)), 3, 3)


def test_library_holds_the_sm90a_join_kernels_without_calls():
    from srj_b200 import _native as N
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", N.LIB_PATH], capture_output=True, text=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)
    for k in KERNELS:
        found = [f for f in funcs if k in f.split("\n", 1)[0]]
        assert len(found) == 1, k
        assert " CALL" not in found[0], k
    assert "sm_90a" in subprocess.run([cuobjdump, "-lelf", N.LIB_PATH], capture_output=True, text=True).stdout


def test_kernels_have_no_stack_frame_or_spills():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    with tempfile.TemporaryDirectory() as td:
        r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-ccbin", "/usr/bin/g++",
                            "--expt-relaxed-constexpr", "-Xptxas", "-v", "-c",
                            os.path.join(ROOT, "spark-rapids-jni_b200", "csrc", "join.cu"), "-o", os.path.join(td, "j.o")],
                           capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    props = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(props) == len(KERNELS) and all(p == ("0", "0", "0") for p in props), props
