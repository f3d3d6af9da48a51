"""CPU checks of the ZOrder surface: the JNI shim ZOrderJni.cpp compiles against the stub headers and defines exactly the
two natives of the reference's ZOrder.java; the C ABI, its Python binding and the Python mirror agree on the names; every
argument error of the C ABI is returned without touching a device; the shipped library holds both sm_90a kernels."""
import ctypes as C
import os
import re
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
JNI = os.path.join(ROOT, "spark-rapids-jni_b200", "jni")
NATIVES = {"Java_com_nvidia_spark_rapids_jni_ZOrder_interleaveBits", "Java_com_nvidia_spark_rapids_jni_ZOrder_hilbertIndex"}
ABI = {"srj_interleave_bits_sizes", "srj_interleave_bits", "srj_hilbert_index"}
INT8, INT16, INT32, INT64, FLOAT32, STRING, LIST, DECIMAL32, DECIMAL128 = 1, 2, 3, 4, 9, 23, 24, 25, 27
INT32_MAX = 2**31 - 1


def test_shim_defines_exactly_the_two_natives():
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    with tempfile.TemporaryDirectory() as td:
        obj = os.path.join(td, "shim.o")
        r = subprocess.run([gxx, "-std=c++17", "-Wall", "-Werror", "-fPIC", "-DSRJ_JNI_STUBS", "-c", os.path.join(JNI, "ZOrderJni.cpp"),
                            "-o", obj], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        syms = subprocess.run(["nm", "-g", "--defined-only", obj], capture_output=True, text=True).stdout
    assert {l.split()[-1] for l in syms.splitlines() if " T " in l and l.split()[-1].startswith("Java_")} == NATIVES


def test_header_binding_and_mirror_agree():
    from srj_b200 import _native as N
    from srj_b200.zorder import ZOrder
    hdr = open(os.path.join(ROOT, "include", "srj_b200.h")).read()
    declared = set(re.findall(r"SRJ_API[^;]*?\b(srj_[a-z0-9_]+)\s*\(", hdr))
    assert {d for d in declared if "interleave" in d or "hilbert" in d} == ABI
    assert ABI <= set(N.SYMBOLS)
    lib = N.lib()
    for name in ABI:
        assert hasattr(lib, name)
    for m in ("interleaveBits", "hilbertIndex"):
        assert callable(getattr(ZOrder, m))


def test_zorder_mirror_does_not_import_the_oracle():
    src = open(os.path.join(ROOT, "spark-rapids-jni_b200", "srj_b200", "zorder.py")).read()
    assert "oracle" not in re.sub(r'""".*?"""', "", src, flags=re.S)


def _cols(types, rows, data=None):
    from srj_b200 import _native as N
    arr = (N.SrjColumn * max(1, len(types)))()
    for i, t in enumerate(types):
        arr[i].type_id, arr[i].size, arr[i].data = t, rows, data
    return arr


@pytest.mark.parametrize("types,rows,want", [
    ([], 10, "EINVAL"),                                      # no columns at the native level
    ([STRING], 4, "EUNSUPPORTED"), ([LIST], 4, "EUNSUPPORTED"),
    ([INT32, INT64], 4, "EINVAL"), ([INT32, FLOAT32], 4, "EINVAL"), ([DECIMAL32, INT32], 4, "EINVAL"),
    ([INT8], INT32_MAX + 1, "EINVAL"),                       # rows * N * W = INT32_MAX + 1
    ([INT16] * 2, (INT32_MAX + 1) // 4, "EINVAL"),
    ([DECIMAL128], (INT32_MAX + 1) // 16, "EINVAL"),
    ([INT32], -1, "EINVAL"),
])
def test_interleave_errors_need_no_device(types, rows, want):
    from srj_b200 import _native as N
    lib = N.lib()
    code = getattr(N, "SRJ_" + want)
    total = C.c_int64(0)
    cols = _cols(types, rows)
    assert lib.srj_interleave_bits_sizes(cols, len(types), rows, C.byref(total)) == code
    assert lib.srj_interleave_bits(cols, len(types), rows, None, None, None) == code


def test_interleave_sizes():
    from srj_b200 import _native as N
    lib = N.lib()
    total = C.c_int64(-1)
    assert lib.srj_interleave_bits_sizes(_cols([INT8], INT32_MAX), 1, INT32_MAX, C.byref(total)) == N.SRJ_OK
    assert total.value == INT32_MAX
    assert lib.srj_interleave_bits_sizes(_cols([INT32] * 4, 1000), 4, 1000, C.byref(total)) == N.SRJ_OK and total.value == 16000
    assert lib.srj_interleave_bits_sizes(_cols([INT32], 0), 1, 0, C.byref(total)) == N.SRJ_OK and total.value == 0
    # one column whose size differs from the row count
    cols = _cols([INT32, INT32], 8)
    cols[1].size = 7
    assert lib.srj_interleave_bits_sizes(cols, 2, 8, C.byref(total)) == N.SRJ_EINVAL
    assert lib.srj_interleave_bits_sizes(cols, 2, 8, None) == N.SRJ_EINVAL
    # missing data, missing outputs
    assert lib.srj_interleave_bits(_cols([INT32], 8), 1, 8, None, None, None) == N.SRJ_EINVAL
    assert lib.srj_interleave_bits(_cols([INT32], 8, data=16), 1, 8, None, None, None) == N.SRJ_EINVAL


@pytest.mark.parametrize("bits,types,want", [
    (0, [INT32], "EINVAL"), (33, [INT32], "EINVAL"), (-1, [INT32], "EINVAL"),
    (33, [], "EINVAL"), (5, [], "EINVAL"),                   # numBits out of range; no columns at the native level
    (32, [INT32] * 3, "EINVAL"), (22, [INT32] * 3, "EINVAL"), (1, [INT32] * 65, "EINVAL"),
    (4, [INT64], "EUNSUPPORTED"), (4, [INT32, INT8], "EUNSUPPORTED"), (4, [STRING], "EUNSUPPORTED"),
])
def test_hilbert_errors_need_no_device(bits, types, want):
    from srj_b200 import _native as N
    assert N.lib().srj_hilbert_index(bits, _cols(types, 4), len(types), 4, None, None) == getattr(N, "SRJ_" + want)


def test_hilbert_accepts_the_64_bit_shapes_before_the_device():
    from srj_b200 import _native as N
    lib = N.lib()
    for n in (1, 2, 4, 8, 16, 32, 64):
        b = min(32, 64 // n)
        # valid shape: the next check that fails is the missing data pointer
        assert lib.srj_hilbert_index(b, _cols([INT32] * n, 4), n, 4, None, None) == N.SRJ_EINVAL
        assert b * n <= 64
    # zero rows: nothing to do, no device touched
    assert lib.srj_hilbert_index(21, _cols([INT32] * 3, 0), 3, 0, None, None) == N.SRJ_OK


def test_library_holds_the_sm90a_zorder_kernels():
    from srj_b200 import _native as N
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", N.LIB_PATH], capture_output=True, text=True).stdout
    names = [f.split("\n", 1)[0] for f in re.split(r"\n\s*Function : ", sass)]
    inter = [n for n in names if "interleave_bits_kernel" in n]
    assert len(inter) == 5, inter                           # W = 1, 2, 4, 8, 16
    assert any("hilbert_index_kernel" in n for n in names)
    assert "sm_90a" in subprocess.run([cuobjdump, "-lelf", N.LIB_PATH], capture_output=True, text=True).stdout
