"""CPU checks of the DateTimeUtils surface: the JNI shim compiles against the stub headers and defines exactly the four
natives of the reference's DateTimeUtils; the C ABI, its Python binding and the Python mirror agree; every argument error
comes back without touching a device; the shipped library holds the sm_90a kernels with no subroutine call, and
datetime.cu compiles with no stack frame or spill."""
import ctypes as C
import os
import re
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
JNI = os.path.join(ROOT, "spark-rapids-jni_b200", "jni")
PREFIX = "Java_com_nvidia_spark_rapids_jni_DateTimeUtils_"
NATIVES = {PREFIX + m for m in ("rebaseGregorianToJulian", "rebaseJulianToGregorian", "truncateWithColumnFormat", "truncateWithScalarFormat")}
ABI = {"srj_datetime_rebase", "srj_datetime_truncate"}
INT32, INT64, DAYS, MICROS, STRING = 3, 4, 12, 15, 23


def test_shim_defines_exactly_the_four_natives():
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    with tempfile.TemporaryDirectory() as td:
        obj = os.path.join(td, "d.o")
        r = subprocess.run([gxx, "-std=c++17", "-Wall", "-Werror", "-fPIC", "-DSRJ_JNI_STUBS", "-c", os.path.join(JNI, "DateTimeUtilsJni.cpp"),
                            "-o", obj], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        syms = subprocess.run(["nm", "-g", "--defined-only", obj], capture_output=True, text=True).stdout
    assert {l.split()[-1] for l in syms.splitlines() if " T " in l and l.split()[-1].startswith("Java_")} == NATIVES


def test_header_binding_and_mirror_agree():
    from srj_b200 import _native as N
    from srj_b200 import datetime as DT
    hdr = open(os.path.join(ROOT, "include", "srj_b200.h")).read()
    declared = set(re.findall(r"SRJ_API[^;]*?\b(srj_[a-z0-9_]+)\s*\(", hdr))
    assert {d for d in declared if "datetime" in d and "iceberg" not in d} == ABI
    assert ABI <= set(N.SYMBOLS)
    for name in ABI:
        assert hasattr(N.lib(), name)
    defines = {k: int(v) for k, v in re.findall(r"#define SRJ_DATETIME_([A-Z_]+) (\d+)", hdr)}
    assert defines == {"GREGORIAN_TO_JULIAN": DT.GREGORIAN_TO_JULIAN, "JULIAN_TO_GREGORIAN": DT.JULIAN_TO_GREGORIAN}
    for m in ("rebaseGregorianToJulian", "rebaseJulianToGregorian", "truncate"):
        assert callable(getattr(DT.DateTimeUtils, m))
    src = open(os.path.join(ROOT, "spark-rapids-jni_b200", "srj_b200", "datetime.py")).read()
    assert "oracle" not in re.sub(r'""".*?"""', "", src, flags=re.S)


def _col(t=MICROS, rows=4, data=16, offsets=None, mask=None):
    from srj_b200 import _native as N
    c = N.SrjColumn()
    c.type_id, c.size, c.data, c.offsets, c.null_mask = t, rows, data, offsets, mask
    return c


@pytest.mark.parametrize("direction,col,out,omask,want", [
    (2, {}, 16, None, "EINVAL"), (-1, {}, 16, None, "EINVAL"),
    (0, dict(t=INT64), 16, None, "EUNSUPPORTED"), (1, dict(t=INT32, rows=0), 16, None, "EUNSUPPORTED"),
    (0, dict(rows=-1), 16, None, "EINVAL"),
    (0, dict(data=None), 16, None, "EINVAL"), (0, dict(data=12), 16, None, "EINVAL"),     # no data; micros not 8-byte aligned
    (1, dict(t=DAYS, data=18), 16, None, "EINVAL"), (0, {}, None, None, "EINVAL"), (0, {}, 20, None, "EINVAL"),
    (0, dict(mask=64), 16, None, "EINVAL"), (0, dict(mask=64), 16, 66, "EINVAL"),
])
def test_rebase_errors_need_no_device(direction, col, out, omask, want):
    from srj_b200 import _native as N
    assert N.lib().srj_datetime_rebase(direction, C.byref(_col(**col)), out, omask, None) == getattr(N, "SRJ_" + want)


def _trunc(dt, fmt_col=None, fmt=None, flen=None, out=16, omask=64, nulls=True):
    from srj_b200 import _native as N
    n = C.c_int64(-7)
    rc = N.lib().srj_datetime_truncate(C.byref(dt) if dt is not None else None, C.byref(fmt_col) if fmt_col is not None else None, fmt,
                                       len(fmt) if flen is None and fmt is not None else (flen or 0), out, omask,
                                       C.byref(n) if nulls else None, None)
    return rc, n.value


@pytest.mark.parametrize("kw,want", [
    (dict(dt=None, fmt=b"YEAR"), "EINVAL"), (dict(dt=_col()), "EINVAL"),                             # no datetime; no format
    (dict(dt=_col(), fmt_col=_col(STRING, offsets=16), fmt=b"YEAR"), "EINVAL"),                        # both formats
    (dict(dt=_col(), fmt=b"YEAR", flen=-1), "EINVAL"), (dict(dt=_col(), fmt=b"YEAR", nulls=False), "EINVAL"),
    (dict(dt=_col(INT64), fmt=b"YEAR"), "EUNSUPPORTED"), (dict(dt=_col(MICROS), fmt_col=_col(INT32)), "EUNSUPPORTED"),
    (dict(dt=_col(rows=3), fmt_col=_col(STRING, rows=4, offsets=16)), "EINVAL"),                      # size mismatch
    (dict(dt=_col(rows=-1), fmt=b"YEAR"), "EINVAL"),
    (dict(dt=_col(data=12), fmt=b"YEAR"), "EINVAL"), (dict(dt=_col(), fmt=b"YEAR", out=None), "EINVAL"),
    (dict(dt=_col(DAYS, data=20), fmt=b"YEAR", out=18), "EINVAL"),
    (dict(dt=_col(mask=64), fmt=b"YEAR", omask=None), "EINVAL"),                                      # a mask, no output mask
    (dict(dt=_col(), fmt=b"YEARS", omask=None), "EINVAL"), (dict(dt=_col(DAYS), fmt=b"HOUR", omask=None), "EINVAL"),
    (dict(dt=_col(), fmt_col=_col(STRING, offsets=None)), "EINVAL"), (dict(dt=_col(), fmt_col=_col(STRING, offsets=18)), "EINVAL"),
    (dict(dt=_col(), fmt_col=_col(STRING, offsets=16), omask=None), "EINVAL"),
])
def test_truncate_errors_need_no_device(kw, want):
    from srj_b200 import _native as N
    assert _trunc(**kw)[0] == getattr(N, "SRJ_" + want)


def test_zero_rows_touch_nothing():
    from srj_b200 import _native as N
    lib = N.lib()
    for t in (DAYS, MICROS):
        for d in (0, 1):
            assert lib.srj_datetime_rebase(d, C.byref(_col(t, 0, data=None)), None, None, None) == N.SRJ_OK
        assert _trunc(_col(t, 0, data=None), fmt=b"bogus", out=None, omask=None) == (N.SRJ_OK, 0)
        assert _trunc(_col(t, 1, data=None), fmt_col=_col(STRING, 0, data=None), out=None, omask=None) == (N.SRJ_OK, 0)
        assert _trunc(_col(t, 0, data=None), fmt_col=_col(STRING, 0, data=None), out=None, omask=None) == (N.SRJ_OK, 0)
    assert lib.srj_datetime_rebase(0, None, None, None, None) == N.SRJ_EINVAL


def test_mirror_raises_the_java_exceptions():
    import srj_b200 as S
    from srj_b200.datetime import DateTimeUtils
    col = S.ColumnView(S.DType.TIMESTAMP_DAYS, 0)
    for fn in (lambda: DateTimeUtils.rebaseGregorianToJulian(None), lambda: DateTimeUtils.rebaseJulianToGregorian(None),
               lambda: DateTimeUtils.truncate(None, "YEAR"), lambda: DateTimeUtils.truncate(col, 3)):
        with pytest.raises(TypeError):
            fn()


def test_library_holds_the_sm90a_datetime_kernels():
    from srj_b200 import _native as N
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", N.LIB_PATH], capture_output=True, text=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)
    maps = [f for f in funcs if "dt_map_kernel" in f.split("\n", 1)[0]]
    # 4 rebase (direction x type), 4 days truncations, 10 micros truncations
    assert len(maps) == 18, [f.split("\n", 1)[0] for f in maps]
    fmts = [f for f in funcs if "dt_trunc_format_kernel" in f.split("\n", 1)[0]]
    assert len(fmts) == 2
    for f in maps + fmts:
        assert " CALL" not in f, f.split("\n", 1)[0]
    assert "sm_90a" in subprocess.run([cuobjdump, "-lelf", N.LIB_PATH], capture_output=True, text=True).stdout


def test_kernels_have_no_stack_frame_or_spills():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    with tempfile.TemporaryDirectory() as td:
        r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-ccbin", "/usr/bin/g++",
                            "--expt-relaxed-constexpr", "-Xptxas", "-v", "-c",
                            os.path.join(ROOT, "spark-rapids-jni_b200", "csrc", "datetime.cu"), "-o", os.path.join(td, "d.o")],
                           capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    props = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(props) == 20 and all(p == ("0", "0", "0") for p in props), props
