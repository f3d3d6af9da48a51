"""CPU checks of the Iceberg surface: the three JNI shims compile against the stub headers and define exactly the six natives
of the reference's IcebergBucket / IcebergTruncate / IcebergDateTimeUtil; the C ABI, its Python binding and the Python
mirror agree on the names; every argument error comes back without touching a device; the shipped library holds the
sm_90a kernels."""
import ctypes as C
import os
import re
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
JNI = os.path.join(ROOT, "spark-rapids-jni_b200", "jni")
PREFIX = "Java_com_nvidia_spark_rapids_jni_iceberg_"
NATIVES = {PREFIX + "IcebergBucket_computeBucket", PREFIX + "IcebergTruncate_truncate"} | \
    {PREFIX + "IcebergDateTimeUtil_" + m for m in ("yearsFromEpoch", "monthsFromEpoch", "daysFromEpoch", "hoursFromEpoch")}
SHIMS = ["IcebergBucketJni.cpp", "IcebergTruncateJni.cpp", "IcebergDateTimeUtilJni.cpp"]
ABI = {"srj_iceberg_bucket", "srj_iceberg_truncate_workspace_bytes", "srj_iceberg_truncate_sizes", "srj_iceberg_truncate",
       "srj_iceberg_datetime"}
INT8, INT32, INT64, UINT8, FLOAT64, DAYS, MICROS, STRING, LIST, DEC32, DEC64, DEC128 = 1, 3, 4, 5, 10, 12, 15, 23, 24, 25, 26, 27


def test_shims_define_exactly_the_six_natives():
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    found = set()
    with tempfile.TemporaryDirectory() as td:
        for src in SHIMS:
            obj = os.path.join(td, src + ".o")
            r = subprocess.run([gxx, "-std=c++17", "-Wall", "-Werror", "-fPIC", "-DSRJ_JNI_STUBS", "-c", os.path.join(JNI, src), "-o", obj],
                               capture_output=True, text=True)
            assert r.returncode == 0, r.stderr
            syms = subprocess.run(["nm", "-g", "--defined-only", obj], capture_output=True, text=True).stdout
            found |= {l.split()[-1] for l in syms.splitlines() if " T " in l and l.split()[-1].startswith("Java_")}
    assert found == NATIVES


def test_header_binding_and_mirror_agree():
    from srj_b200 import _native as N
    from srj_b200 import iceberg as I
    hdr = open(os.path.join(ROOT, "include", "srj_b200.h")).read()
    declared = set(re.findall(r"SRJ_API[^;]*?\b(srj_[a-z0-9_]+)\s*\(", hdr))
    assert {d for d in declared if "iceberg" in d} == ABI
    assert ABI <= set(N.SYMBOLS)
    lib = N.lib()
    for name in ABI:
        assert hasattr(lib, name)
    defines = dict(re.findall(r"#define SRJ_ICEBERG_([A-Z]+) (\d+)", hdr))
    assert {k: int(v) for k, v in defines.items()} == {"YEARS": I.YEARS, "MONTHS": I.MONTHS, "DAYS": I.DAYS, "HOURS": I.HOURS}
    assert callable(I.IcebergBucket.computeBucket) and callable(I.IcebergTruncate.truncate)
    for m in ("yearsFromEpoch", "monthsFromEpoch", "daysFromEpoch", "hoursFromEpoch"):
        assert callable(getattr(I.IcebergDateTimeUtil, m))


def test_iceberg_mirror_does_not_import_the_oracle():
    src = open(os.path.join(ROOT, "spark-rapids-jni_b200", "srj_b200", "iceberg.py")).read()
    assert "oracle" not in re.sub(r'""".*?"""', "", src, flags=re.S)


def _col(t, rows, data=None, offsets=None, child=None, mask=None):
    from srj_b200 import _native as N
    c = N.SrjColumn()
    c.type_id, c.size, c.data, c.offsets, c.null_mask = t, rows, data, offsets, mask
    if child is not None:
        arr = (N.SrjColumn * 1)()
        arr[0].type_id, arr[0].data, arr[0].null_mask = child[0], child[1], child[2] if len(child) > 2 else None
        c.children, c.num_children = arr, 1
        c._keep = arr
    return c


@pytest.mark.parametrize("col,n,want", [
    (dict(t=INT64, rows=4), 0, "EINVAL"), (dict(t=INT64, rows=4), -1, "EINVAL"), (dict(t=STRING, rows=0), 0, "EINVAL"),
    (dict(t=FLOAT64, rows=4), 16, "EUNSUPPORTED"), (dict(t=INT8, rows=4), 16, "EUNSUPPORTED"),
    (dict(t=LIST, rows=4), 16, "EUNSUPPORTED"), (dict(t=LIST, rows=4, child=(INT8, None)), 16, "EUNSUPPORTED"),
    (dict(t=INT64, rows=-1), 16, "EINVAL"),
    (dict(t=INT64, rows=4), 16, "EINVAL"),                          # no data
    (dict(t=INT64, rows=4, data=12), 16, "EINVAL"),                 # data not 8-byte aligned
    (dict(t=DEC128, rows=4, data=24), 16, "EINVAL"),                # DECIMAL128 needs 8 bytes, not 16, but a non-NULL output
    (dict(t=STRING, rows=4), 16, "EINVAL"),                         # no offsets
    (dict(t=INT32, rows=4, data=16, mask=64), 16, "EINVAL"),        # a mask but no output mask
])
def test_bucket_errors_need_no_device(col, n, want):
    from srj_b200 import _native as N
    assert N.lib().srj_iceberg_bucket(C.byref(_col(**col)), n, None, None, None) == getattr(N, "SRJ_" + want)


def test_bucket_zero_rows_touch_nothing():
    from srj_b200 import _native as N
    lib = N.lib()
    for t in (INT32, INT64, DEC32, DEC64, DEC128, DAYS, MICROS, STRING):
        assert lib.srj_iceberg_bucket(C.byref(_col(t, 0)), 16, None, None, None) == N.SRJ_OK
    assert lib.srj_iceberg_bucket(C.byref(_col(LIST, 0, child=(UINT8, None))), 16, None, None, None) == N.SRJ_OK
    assert lib.srj_iceberg_bucket(None, 16, None, None, None) == N.SRJ_EINVAL


@pytest.mark.parametrize("col,w,want", [
    (dict(t=INT32, rows=4, data=16), 0, "EINVAL"), (dict(t=DEC128, rows=0), 0, "EINVAL"),
    (dict(t=FLOAT64, rows=4, data=16), 3, "EUNSUPPORTED"), (dict(t=DAYS, rows=4, data=16), 3, "EUNSUPPORTED"),
    (dict(t=STRING, rows=4, offsets=16), 0, "EINVAL"), (dict(t=STRING, rows=0), -3, "EINVAL"),
    (dict(t=LIST, rows=4, offsets=16, child=(UINT8, 16)), 0, "EINVAL"),
    (dict(t=LIST, rows=4, offsets=16, child=(INT8, 16)), 3, "EUNSUPPORTED"),
    (dict(t=LIST, rows=4, offsets=16, child=(UINT8, 16, 64)), 3, "EINVAL"),   # a nullable child
    (dict(t=INT64, rows=4, data=20), 3, "EINVAL"),                            # misaligned input
    (dict(t=INT64, rows=4, data=16), 3, "EINVAL"),                            # no output data
    (dict(t=STRING, rows=4, offsets=16), 3, "EINVAL"),                        # no output offsets
])
def test_truncate_errors_need_no_device(col, w, want):
    from srj_b200 import _native as N
    out = _col(col["t"], col["rows"])
    assert N.lib().srj_iceberg_truncate(C.byref(_col(**col)), w, C.byref(out), None) == getattr(N, "SRJ_" + want)


def test_truncate_sizes_errors_need_no_device():
    from srj_b200 import _native as N
    lib = N.lib()
    total = C.c_int64(0)
    assert lib.srj_iceberg_truncate_sizes(C.byref(_col(INT32, 4, data=16)), 3, 16, C.byref(total), 16, None) == N.SRJ_EUNSUPPORTED
    assert lib.srj_iceberg_truncate_sizes(C.byref(_col(STRING, 4, offsets=16)), 0, 16, C.byref(total), 16, None) == N.SRJ_EINVAL
    assert lib.srj_iceberg_truncate_sizes(C.byref(_col(STRING, 4, offsets=16)), 3, None, C.byref(total), 16, None) == N.SRJ_EINVAL
    assert lib.srj_iceberg_truncate_sizes(C.byref(_col(STRING, 4, offsets=16)), 3, 16, None, 16, None) == N.SRJ_EINVAL
    assert lib.srj_iceberg_truncate_sizes(C.byref(_col(STRING, 4, offsets=16)), 3, 16, C.byref(total), None, None) == N.SRJ_EINVAL
    assert lib.srj_iceberg_truncate_sizes(C.byref(_col(STRING, 4, offsets=16)), 3, 18, C.byref(total), 16, None) == N.SRJ_EINVAL
    assert lib.srj_iceberg_truncate_workspace_bytes(0) > 0 and lib.srj_iceberg_truncate_workspace_bytes(-5) > 0
    assert lib.srj_iceberg_truncate_workspace_bytes(10**8) >= lib.srj_iceberg_truncate_workspace_bytes(10**6)


@pytest.mark.parametrize("transform,col,want", [
    (4, dict(t=MICROS, rows=4, data=16), "EINVAL"), (-1, dict(t=DAYS, rows=4, data=16), "EINVAL"),
    (3, dict(t=DAYS, rows=4, data=16), "EUNSUPPORTED"), (0, dict(t=INT32, rows=4, data=16), "EUNSUPPORTED"),
    (2, dict(t=INT64, rows=0), "EUNSUPPORTED"), (1, dict(t=STRING, rows=4), "EUNSUPPORTED"),
    (0, dict(t=MICROS, rows=4, data=12), "EINVAL"), (0, dict(t=DAYS, rows=4, data=16), "EINVAL"),   # misaligned; no output
    (3, dict(t=MICROS, rows=4, data=16, mask=64), "EINVAL"),
])
def test_datetime_errors_need_no_device(transform, col, want):
    from srj_b200 import _native as N
    assert N.lib().srj_iceberg_datetime(transform, C.byref(_col(**col)), None, None, None) == getattr(N, "SRJ_" + want)


def test_mirror_raises_the_java_exceptions_before_the_native_layer():
    import srj_b200 as S
    from srj_b200.iceberg import IcebergBucket, IcebergDateTimeUtil, IcebergTruncate
    col = S.ColumnView(S.DType.FLOAT64, 0)
    with pytest.raises(ValueError, match="numBuckets must be positive"):
        IcebergBucket.computeBucket(col, 0)
    with pytest.raises(ValueError, match="Unsupported type for truncation"):
        IcebergTruncate.truncate(col, 3)
    with pytest.raises(ValueError):
        IcebergDateTimeUtil.yearsFromEpoch(col)
    with pytest.raises(ValueError):
        IcebergDateTimeUtil.hoursFromEpoch(S.ColumnView(S.DType.TIMESTAMP_DAYS, 0))
    for fn in (lambda: IcebergBucket.computeBucket(None, 4), lambda: IcebergTruncate.truncate(None, 4),
               lambda: IcebergDateTimeUtil.daysFromEpoch(None)):
        with pytest.raises(TypeError):
            fn()


def test_library_holds_the_sm90a_iceberg_kernels():
    from srj_b200 import _native as N
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", N.LIB_PATH], capture_output=True, text=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)
    names = [f.split("\n", 1)[0] for f in funcs]
    for k in ("bucket_bytes_kernel", "truncate_sizes_kernel", "truncate_copy_kernel"):
        assert any(k in n for n in names), k
    maps = [n for n in names if "ice_map_kernel" in n]
    assert len(maps) == 14, maps              # 5 bucket, 3 truncate, 6 date-time instantiations
    # the INT32 / INT64 truncate and every bucket kernel call no division subroutine
    for f in funcs:
        name = f.split("\n", 1)[0]
        if "ice_map_kernel" in name or "bucket_bytes_kernel" in name:
            assert " CALL" not in f, name
    assert "sm_90a" in subprocess.run([cuobjdump, "-lelf", N.LIB_PATH], capture_output=True, text=True).stdout
