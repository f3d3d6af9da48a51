"""CPU checks of the GpuTimeZoneDB surface: the JNI shim compiles against the stub headers and defines exactly the four
natives of the reference's GpuTimeZoneDB; the C ABI, its Python binding and the Python mirror agree; every argument error
comes back without touching a device; the shipped library holds the sm_90a kernels with no subroutine call, and
timezone.cu compiles with no stack frame or spill."""
import ctypes as C
import os
import re
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
JNI = os.path.join(ROOT, "spark-rapids-jni_b200", "jni")
PREFIX = "Java_com_nvidia_spark_rapids_jni_GpuTimeZoneDB_"
NATIVES = {PREFIX + m for m in ("convertTimestampColumnToUTC", "convertUTCTimestampColumnToTimeZone", "convertTimestampColumnToUTCWithTzCv",
                                "convertOrcTimezones")}
ABI = {"srj_timezone_convert", "srj_timezone_convert_multi", "srj_orc_convert_timezones"}
INT32, INT64, UINT8, BOOL8, SECONDS, MILLIS, MICROS, NANOS, DAYS, LIST, STRUCT = 3, 4, 5, 11, 13, 14, 15, 16, 12, 24, 28


def test_shim_defines_exactly_the_four_natives():
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    with tempfile.TemporaryDirectory() as td:
        obj = os.path.join(td, "t.o")
        r = subprocess.run([gxx, "-std=c++17", "-Wall", "-Werror", "-fPIC", "-DSRJ_JNI_STUBS", "-c", os.path.join(JNI, "GpuTimeZoneDBJni.cpp"),
                            "-o", obj], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        syms = subprocess.run(["nm", "-g", "--defined-only", obj], capture_output=True, text=True).stdout
    assert {l.split()[-1] for l in syms.splitlines() if " T " in l and l.split()[-1].startswith("Java_")} == NATIVES


def test_header_binding_and_mirror_agree():
    from srj_b200 import _native as N
    from srj_b200 import timezone as TZ
    hdr = open(os.path.join(ROOT, "include", "srj_b200.h")).read()
    declared = set(re.findall(r"SRJ_API[^;]*?\b(srj_[a-z0-9_]+)\s*\(", hdr))
    assert {d for d in declared if "timezone" in d} == ABI
    assert ABI <= set(N.SYMBOLS)
    for name in ABI:
        assert hasattr(N.lib(), name)
    defines = {k: int(v) for k, v in re.findall(r"#define SRJ_TIMEZONE_([A-Z_]+) (\d+)", hdr)}
    assert defines == {"TO_UTC": TZ.TO_UTC, "FROM_UTC": TZ.FROM_UTC}
    for m in ("convertTimestampColumnToUTC", "convertUTCTimestampColumnToTimeZone", "convertTimestampColumnToUTCWithTzCv", "convertOrcTimezones"):
        assert callable(getattr(TZ.GpuTimeZoneDB, m))
    src = open(os.path.join(ROOT, "spark-rapids-jni_b200", "srj_b200", "timezone.py")).read()
    assert "oracle" not in re.sub(r'""".*?"""', "", src, flags=re.S)


def _col(t=MICROS, rows=4, data=16, offsets=None, mask=None, children=None):
    from srj_b200 import _native as N
    c = N.SrjColumn()
    c.type_id, c.size, c.data, c.offsets, c.null_mask = t, rows, data, offsets, mask
    if children:
        arr = (N.SrjColumn * len(children))(*children)
        c.children, c.num_children = arr, len(children)
        c._keep = (arr, children)
    return c


def _table(zones=2, entries=3, fields=(INT64, INT64, INT32), struct=STRUCT, rules_t=INT32, fixed_off=64, dst_off=64, dst_rows=None,
           field_data=(16, 16, 16)):
    fl = [_col(t, entries, data=d) for t, d in zip(fields, field_data)]
    st = _col(struct, entries, data=None, children=fl)
    fixed = _col(LIST, zones, data=None, offsets=fixed_off, children=[st])
    dst = _col(LIST, zones if dst_rows is None else dst_rows, data=None, offsets=dst_off, children=[_col(rules_t, 12, data=16)])
    return fixed, dst


def _convert(direction=0, inp=None, table=None, tz=0, out=16, omask=None):
    from srj_b200 import _native as N
    inp = _col() if inp is None else inp
    fixed, dst = _table() if table is None else table
    return N.lib().srj_timezone_convert(direction, C.byref(inp), C.byref(fixed) if fixed is not None else None,
                                        C.byref(dst) if dst is not None else None, tz, out, omask, None)


@pytest.mark.parametrize("kw,want", [
    (dict(direction=2), "EINVAL"), (dict(direction=-1), "EINVAL"),
    (dict(inp=_col(INT64)), "EUNSUPPORTED"), (dict(inp=_col(DAYS)), "EUNSUPPORTED"),
    (dict(table=(None, None)), "EINVAL"),
    (dict(table=_table(struct=INT64)), "EINVAL"), (dict(table=_table(fields=(INT64, INT32, INT32))), "EINVAL"),
    (dict(table=_table(rules_t=INT64)), "EINVAL"), (dict(table=_table(dst_rows=3)), "EINVAL"),
    (dict(table=_table(fixed_off=None)), "EINVAL"), (dict(table=_table(dst_off=66)), "EINVAL"),
    (dict(table=_table(field_data=(16, 20, 16))), "EINVAL"), (dict(table=_table(field_data=(None, 16, 16))), "EINVAL"),
    (dict(tz=-1), "EINVAL"), (dict(tz=2), "EINVAL"),
    (dict(inp=_col(rows=-1)), "EINVAL"), (dict(inp=_col(data=None)), "EINVAL"), (dict(inp=_col(data=12)), "EINVAL"),
    (dict(out=None), "EINVAL"), (dict(out=20), "EINVAL"),
    (dict(inp=_col(mask=64)), "EINVAL"), (dict(inp=_col(mask=64), omask=66), "EINVAL"),
])
def test_convert_errors_need_no_device(kw, want):
    from srj_b200 import _native as N
    assert _convert(**kw) == getattr(N, "SRJ_" + want)


def _multi(cols=None, table=None, out=16, omask=64, nulls=True):
    from srj_b200 import _native as N
    base = [_col(INT64), _col(INT32), _col(BOOL8), _col(UINT8), _col(INT32), _col(INT32)]
    for i, c in (cols or {}).items():
        base[i] = c
    fixed, dst = _table() if table is None else table
    n = C.c_int64(-7)
    rc = N.lib().srj_timezone_convert_multi(*[C.byref(c) if c is not None else None for c in base[:5]], C.byref(fixed), C.byref(dst),
                                            C.byref(base[5]) if base[5] is not None else None, out, omask, C.byref(n) if nulls else None, None)
    return rc, n.value


@pytest.mark.parametrize("kw,want", [
    (dict(cols={0: _col(INT32)}), "EUNSUPPORTED"), (dict(cols={1: _col(INT64)}), "EUNSUPPORTED"),
    (dict(cols={2: _col(INT32)}), "EINVAL"), (dict(cols={3: _col(1)}), "EINVAL"), (dict(cols={5: _col(INT64)}), "EINVAL"),
    (dict(cols={4: _col(INT32, rows=5)}), "EINVAL"), (dict(cols={5: None}), "EINVAL"), (dict(cols={1: None}), "EINVAL"),
    (dict(cols={0: _col(INT64, rows=-1)}), "EINVAL"), (dict(cols={2: _col(BOOL8, data=None)}), "EINVAL"),
    (dict(table=_table(struct=INT64)), "EINVAL"), (dict(out=None), "EINVAL"), (dict(out=12), "EINVAL"),
    (dict(omask=None), "EINVAL"), (dict(omask=66), "EINVAL"), (dict(nulls=False), "EINVAL"),
])
def test_multi_errors_need_no_device(kw, want):
    from srj_b200 import _native as N
    assert _multi(**kw)[0] == getattr(N, "SRJ_" + want)


def _orc(inp=None, w=(None, None), r=(None, None), out=16, omask=None):
    from srj_b200 import _native as N
    inp = _col() if inp is None else inp
    ref = lambda c: C.byref(c) if c is not None else None                          # noqa: E731
    return N.lib().srj_orc_convert_timezones(C.byref(inp), ref(w[0]), ref(w[1]), 0, ref(r[0]), ref(r[1]), 0, out, omask, None)


@pytest.mark.parametrize("kw,want", [
    (dict(inp=_col(SECONDS)), "EUNSUPPORTED"), (dict(inp=_col(INT64)), "EUNSUPPORTED"),
    (dict(w=(_col(INT64, 3), None)), "EINVAL"), (dict(r=(None, _col(INT32, 3))), "EINVAL"),
    (dict(w=(_col(INT64, 3), _col(INT32, 4))), "EINVAL"), (dict(w=(_col(INT32, 3), _col(INT32, 3))), "EINVAL"),
    (dict(r=(_col(INT64, 3), _col(INT64, 3))), "EINVAL"), (dict(r=(_col(INT64, 3, data=12), _col(INT32, 3))), "EINVAL"),
    (dict(inp=_col(data=None)), "EINVAL"), (dict(out=None), "EINVAL"), (dict(inp=_col(mask=64)), "EINVAL"),
])
def test_orc_errors_need_no_device(kw, want):
    from srj_b200 import _native as N
    assert _orc(**kw) == getattr(N, "SRJ_" + want)


def test_zero_rows_touch_nothing():
    from srj_b200 import _native as N
    lib = N.lib()
    for t in (SECONDS, MILLIS, MICROS, NANOS):
        for d in (0, 1):
            assert _convert(d, _col(t, 0, data=None), out=None) == N.SRJ_OK
    zero = {i: _col(t, 0, data=None) for i, t in enumerate((INT64, INT32, BOOL8, UINT8, INT32, INT32))}
    assert _multi(cols=zero, out=None, omask=None) == (N.SRJ_OK, 0)
    assert _orc(_col(MICROS, 0, data=None), out=None) == N.SRJ_OK
    assert lib.srj_timezone_convert(0, None, None, None, 0, None, None, None) == N.SRJ_EINVAL


def test_mirror_raises_the_java_exceptions():
    import srj_b200 as S
    from srj_b200.timezone import GpuTimeZoneDB
    col = S.ColumnView(S.DType.TIMESTAMP_MICROSECONDS, 0)
    info = S.Table(S.ColumnView(S.DType.LIST, 0), S.ColumnView(S.DType.LIST, 0))
    for fn in (lambda: GpuTimeZoneDB.convertTimestampColumnToUTC(None, info, 0), lambda: GpuTimeZoneDB.convertTimestampColumnToUTC(col, None, 0),
               lambda: GpuTimeZoneDB.convertUTCTimestampColumnToTimeZone(None, info, 0),
               lambda: GpuTimeZoneDB.convertTimestampColumnToUTCWithTzCv(col, col, None, col, col, info, col),
               lambda: GpuTimeZoneDB.convertTimestampColumnToUTCWithTzCv(col, col, col, col, col, None, col),
               lambda: GpuTimeZoneDB.convertOrcTimezones(None, None, 0, None, 0)):
        with pytest.raises(TypeError):
            fn()


def test_library_holds_the_sm90a_timezone_kernels():
    from srj_b200 import _native as N
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", N.LIB_PATH], capture_output=True, text=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)
    names = {k: [f for f in funcs if k in f.split("\n", 1)[0]] for k in ("tz_convert_kernel", "tz_multi_kernel", "orc_tz_kernel")}
    assert {k: len(v) for k, v in names.items()} == {"tz_convert_kernel": 8, "tz_multi_kernel": 1, "orc_tz_kernel": 1}   # 4 units x 2 directions
    for f in sum(names.values(), []):
        assert " CALL" not in f, f.split("\n", 1)[0]
    assert "sm_90a" in subprocess.run([cuobjdump, "-lelf", N.LIB_PATH], capture_output=True, text=True).stdout


def test_kernels_have_no_stack_frame_or_spills():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    with tempfile.TemporaryDirectory() as td:
        r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-ccbin", "/usr/bin/g++",
                            "--expt-relaxed-constexpr", "-Xptxas", "-v", "-c",
                            os.path.join(ROOT, "spark-rapids-jni_b200", "csrc", "timezone.cu"), "-o", os.path.join(td, "t.o")],
                           capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    props = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(props) == 10 and all(p == ("0", "0", "0") for p in props), props
