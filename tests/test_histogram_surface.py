"""CPU checks of the Histogram surface: the JNI shim HistogramJni.cpp compiles against the stub headers and defines exactly
the two natives of the reference's Histogram.java; the C ABI, its Python binding and the Python mirror agree; every
argument error of the C ABI comes back with its code before any device work; the histogram kernels are in the library's
sm_90a cubin with no subroutine call, stack frame or spill."""
import ctypes as C
import os
import re
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
JNI = os.path.join(ROOT, "spark-rapids-jni_b200", "jni")
NATIVES = {"Java_com_nvidia_spark_rapids_jni_Histogram_createHistogramIfValid",
           "Java_com_nvidia_spark_rapids_jni_Histogram_percentileFromHistogram"}
ABI = {"srj_percentile_workspace_bytes", "srj_percentile_from_histogram_size", "srj_percentile_from_histogram",
       "srj_histogram_workspace_bytes", "srj_histogram_create_size", "srj_histogram_create"}
KERNELS = ("pct_group_kernel", "pct_classify_kernel", "pct_rows_kernel", "sel_total_kernel", "sel_init_kernel", "sel_hist_kernel",
           "sel_pick_kernel", "sel_finish_kernel", "hc_flag_kernel", "hc_write_kernel", "pct_flat_mask_kernel", "hc_clear_mask_kernel")
INT8, INT32, INT64, FLOAT64, TS_DAYS, STRING, LIST, DEC128, STRUCT = 1, 3, 4, 10, 12, 23, 24, 27, 28
INT32_MAX = 2**31 - 1


def test_shim_defines_exactly_the_two_natives():
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    with tempfile.TemporaryDirectory() as td:
        obj = os.path.join(td, "h.o")
        r = subprocess.run([gxx, "-std=c++17", "-Wall", "-Werror", "-fPIC", "-DSRJ_JNI_STUBS", "-c", os.path.join(JNI, "HistogramJni.cpp"),
                            "-o", obj], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        syms = subprocess.run(["nm", "-g", "--defined-only", obj], capture_output=True, text=True).stdout
    assert {l.split()[-1] for l in syms.splitlines() if " T " in l and l.split()[-1].startswith("Java_")} == NATIVES


def test_header_binding_and_mirror_agree():
    from srj_b200 import _native as N
    from srj_b200.histogram import Histogram
    hdr = open(os.path.join(ROOT, "include", "srj_b200.h")).read()
    declared = set(re.findall(r"SRJ_API[^;]*?\b(srj_[a-z0-9_]+)\s*\(", hdr))
    assert {d for d in declared if "histogram" in d or "percentile" in d} == ABI
    for name in ABI:
        args = re.search(r"SRJ_API[^;]*?\b" + name + r"\s*\(([^)]*)\)", hdr).group(1)
        assert len(args.split(",")) == len(N.SYMBOLS[name][1]), name
        assert hasattr(N.lib(), name)
    assert int(re.search(r"#define SRJ_HISTOGRAM_CTA_ELEMENTS (\d+)", hdr).group(1)) == 8192
    assert [m for m in vars(Histogram) if not m.startswith("_")] == ["createHistogramIfValid", "percentileFromHistogram"]
    src = open(os.path.join(ROOT, "spark-rapids-jni_b200", "srj_b200", "histogram.py")).read()
    assert "oracle" not in re.sub(r'""".*?"""', "", src, flags=re.S)


def _col(t, rows=4, data=256, mask=None, offsets=None, kids=None):
    from srj_b200 import _native as N
    c = N.SrjColumn()
    c.type_id, c.size, c.data, c.null_mask, c.offsets = t, rows, data, mask, offsets
    if kids is not None:
        arr = (N.SrjColumn * len(kids))(*kids)
        c.children, c.num_children = arr, len(kids)
        c._keep = arr
    return c


def _hist(vt=INT32, ct=INT64, rows=4, elems=10, struct_mask=None, count_mask=None, nkids=2, st=STRUCT, vmask=None):
    kids = [_col(vt, elems, mask=vmask), _col(ct, elems, mask=count_mask), _col(INT32, elems)][:nkids]
    s = _col(st, elems, data=None, mask=struct_mask, kids=kids)
    return _col(LIST, rows, data=None, offsets=256, kids=[s])


def _pct(inp, P=1, ws=256, out=256, mask=256, lists=0, offsets=256, pct=True):
    from srj_b200 import _native as N
    lib = N.lib()
    v, n = C.c_int64(-1), C.c_int64(-1)
    pa = (C.c_double * max(P, 1))(*([0.5] * max(P, 1))) if pct else None
    a = lib.srj_percentile_from_histogram_size(C.byref(inp), P, lists, C.byref(v), C.byref(n), ws, None)
    b = lib.srj_percentile_from_histogram(C.byref(inp), pa, P, lists, out, mask, offsets, ws, None)
    return a, b


@pytest.mark.parametrize("inp,P,want", [
    (_col(INT32, 4), 1, "EINVAL"),                                          # not a LIST
    (_hist(struct_mask=256), 1, "EINVAL"),                                  # the struct child has nulls
    (_hist(nkids=3), 1, "EINVAL"), (_hist(nkids=1), 1, "EINVAL"), (_hist(st=LIST), 1, "EINVAL"),
    (_hist(count_mask=256), 1, "EINVAL"),                                   # null counts
    (_hist(ct=INT32), 1, "EINVAL"), (_hist(ct=FLOAT64), 1, "EINVAL"),       # counts not INT64
    (_hist(rows=INT32_MAX // 2 + 1), 2, "EOVERFLOW"),                       # rows * P > INT32_MAX
    (_hist(rows=2**16, vt=STRING), 2**15, "EOVERFLOW"),                     # overflow before the type
    (_hist(vt=STRING), 1, "EUNSUPPORTED"), (_hist(vt=DEC128), 1, "EUNSUPPORTED"), (_hist(vt=TS_DAYS), 1, "EUNSUPPORTED"),
    (_hist(), -1, "EINVAL"),
])
def test_percentile_errors_need_no_device(inp, P, want):
    from srj_b200 import _native as N
    code = getattr(N, "SRJ_" + want)
    assert _pct(inp, P) == (code, code)


def test_percentile_buffer_checks_need_no_device():
    from srj_b200 import _native as N
    E = N.SRJ_EINVAL
    h = _hist()
    assert _pct(h, ws=None) == (E, E)                                       # no workspace
    assert _pct(h, ws=8) == (E, E)                                          # misaligned workspace
    assert _pct(h, out=None)[1] == E and _pct(h, mask=None)[1] == E and _pct(h, pct=False)[1] == E
    assert _pct(h, lists=1, offsets=None)[1] == E
    bad = _hist()
    bad.children[0].children[1].size = 9                                    # counts and values differ in size
    assert _pct(bad) == (E, E)
    nooff = _hist()
    nooff.offsets = None
    assert _pct(nooff) == (E, E)
    empty = _hist(rows=0)
    assert _pct(empty, ws=None, out=None, mask=None) == (N.SRJ_OK, N.SRJ_OK)   # zero rows touch nothing
    lib = N.lib()
    assert lib.srj_percentile_workspace_bytes(10**6, 10**7, 5) > 16 * 10**6
    assert lib.srj_percentile_workspace_bytes(-1, -1, -1) > 0


def _create(v, f, lists=0, ws=256, out=256, mask=256, freq_out=256, offsets=256):
    from srj_b200 import _native as N
    lib = N.lib()
    n, nulls = C.c_int64(-1), C.c_int64(-1)
    a = lib.srj_histogram_create_size(C.byref(v), C.byref(f), lists, C.byref(n), C.byref(nulls), ws, None)
    b = lib.srj_histogram_create(C.byref(v), C.byref(f), lists, out, mask, freq_out, offsets, ws, None)
    return a, b


@pytest.mark.parametrize("v,f,want", [
    (_col(INT32), _col(INT64, mask=256), "EINVAL"),                         # null frequencies
    (_col(INT32), _col(INT32), "EINVAL"),                                   # frequencies not INT64
    (_col(INT32, 4), _col(INT64, 5), "EINVAL"),                             # sizes differ
    (_col(INT32, 4), _col(INT32, 5, mask=256), "EINVAL"),                   # the first failing check in the reference's order
    (_col(STRING), _col(INT64), "EUNSUPPORTED"), (_col(LIST), _col(INT64), "EUNSUPPORTED"),
    (_col(INT32, data=None), _col(INT64), "EINVAL"), (_col(INT64, data=260), _col(INT64), "EINVAL"),
    (_col(INT32, mask=258), _col(INT64), "EINVAL"),
])
def test_create_errors_need_no_device(v, f, want):
    from srj_b200 import _native as N
    code = getattr(N, "SRJ_" + want)
    assert _create(v, f) == (code, code)
    assert _create(v, f, lists=1) == (code, code)


def test_create_buffer_checks_need_no_device():
    from srj_b200 import _native as N
    E = N.SRJ_EINVAL
    v, f = _col(INT32), _col(INT64)
    assert _create(v, f, ws=None) == (E, E)
    assert _create(v, f, mask=None)[1] == E                                 # struct output: the mask is always needed
    assert _create(_col(INT32, mask=256), f, lists=1, mask=None)[1] == E    # lists: needed when the values have nulls
    assert _create(v, f, lists=1, offsets=None)[1] == E
    assert _create(_col(DEC128, data=264), f, out=260)[1] == E              # output values at the element (8 bytes at most)
    assert _create(_col(INT32, 0, data=None), _col(INT64, 0, data=None), ws=None, out=None, mask=None, offsets=None) == (N.SRJ_OK, N.SRJ_OK)
    assert N.lib().srj_histogram_workspace_bytes(1000) >= 4000


def test_library_holds_the_sm90a_histogram_kernels_without_calls():
    from srj_b200 import _native as N
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", N.LIB_PATH], capture_output=True, text=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)
    for k in KERNELS:
        found = [f for f in funcs if k in f.split("\n", 1)[0]]
        assert len(found) == (2 if k == "pct_group_kernel" else 1), k
        assert all(" CALL" not in f for f in found), k
    assert "sm_90a" in subprocess.run([cuobjdump, "-lelf", N.LIB_PATH], capture_output=True, text=True).stdout


def test_kernels_have_no_stack_frame_or_spills():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    with tempfile.TemporaryDirectory() as td:
        r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-ccbin", "/usr/bin/g++",
                            "--expt-relaxed-constexpr", "-Xptxas", "-v", "-c",
                            os.path.join(ROOT, "spark-rapids-jni_b200", "csrc", "histogram.cu"), "-o", os.path.join(td, "h.o")],
                           capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    props = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(props) == len(KERNELS) + 1 and all(p == ("0", "0", "0") for p in props), props
