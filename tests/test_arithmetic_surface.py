"""CPU checks of the Arithmetic surface: the JNI shim ArithmeticJni.cpp compiles against the stub headers and defines exactly
the two natives of the reference's Arithmetic.java; the C ABI, its Python binding and the Python mirror agree; every
argument error of the C ABI comes back with its code before any device work; the arithmetic kernels are in the library's
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
NATIVES = {"Java_com_nvidia_spark_rapids_jni_Arithmetic_multiply", "Java_com_nvidia_spark_rapids_jni_Arithmetic_round"}
ABI = {"srj_multiply", "srj_round"}
# kernel -> instantiations: mul 4 integer types x 3 modes + 2 float types; round_float 2 types x 2 modes x 3 signs;
# round_int 4 types; round_decimal 3 types x (round, scale-up)
KERNELS = {"mul_kernel": 14, "round_float_kernel": 12, "round_int_kernel": 4, "round_decimal_kernel": 6}
INT8, INT16, INT32, INT64, UINT32, FLOAT32, FLOAT64, BOOL8, STRING, DEC32, DEC128 = 1, 2, 3, 4, 7, 9, 10, 11, 23, 25, 27


def test_shim_defines_exactly_the_two_natives():
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    with tempfile.TemporaryDirectory() as td:
        obj = os.path.join(td, "a.o")
        r = subprocess.run([gxx, "-std=c++17", "-Wall", "-Werror", "-fPIC", "-DSRJ_JNI_STUBS", "-c", os.path.join(JNI, "ArithmeticJni.cpp"),
                            "-o", obj], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        syms = subprocess.run(["nm", "-g", "--defined-only", obj], capture_output=True, text=True).stdout
    assert {l.split()[-1] for l in syms.splitlines() if " T " in l and l.split()[-1].startswith("Java_")} == NATIVES


def test_header_binding_and_mirror_agree():
    from srj_b200 import _native as N
    from srj_b200.arithmetic import Arithmetic, ExceptionWithRowIndex, RoundMode
    hdr = open(os.path.join(ROOT, "include", "srj_b200.h")).read()
    declared = set(re.findall(r"SRJ_API[^;]*?\b(srj_[a-z0-9_]+)\s*\(", hdr))
    assert {d for d in declared if d in ("srj_multiply", "srj_round") or "arith" in d} == ABI
    for name in ABI:
        args = re.search(r"SRJ_API[^;]*?\b" + name + r"\s*\(([^)]*)\)", hdr).group(1)
        assert len(args.split(",")) == len(N.SYMBOLS[name][1]), name
        assert hasattr(N.lib(), name)
    assert int(re.search(r"#define SRJ_ROUND_HALF_UP (\d+)", hdr).group(1)) == RoundMode.HALF_UP.nativeId == 0
    assert int(re.search(r"#define SRJ_ROUND_HALF_EVEN (\d+)", hdr).group(1)) == RoundMode.HALF_EVEN.nativeId == 1
    assert [m for m in vars(Arithmetic) if not m.startswith("_")] == ["multiply", "round"]
    assert ExceptionWithRowIndex(7).getRowIndex() == 7
    src = open(os.path.join(ROOT, "spark-rapids-jni_b200", "srj_b200", "arithmetic.py")).read()
    assert "oracle" not in re.sub(r'""".*?"""', "", src, flags=re.S)


def _col(t, rows=4, data=256, mask=None, scale=0):
    from srj_b200 import _native as N
    c = N.SrjColumn()
    c.type_id, c.size, c.data, c.null_mask, c.scale = t, rows, data, mask, scale
    return c


def _mul(a, b, av=None, bv=None, ansi=0, try_mode=0, out=256, mask=256):
    from srj_b200 import _native as N
    nulls, row = C.c_int64(-5), C.c_int64(-5)
    rc = N.lib().srj_multiply(C.byref(a), av, C.byref(b), bv, ansi, try_mode, out, mask, C.byref(nulls), C.byref(row), None)
    return rc, nulls.value, row.value


@pytest.mark.parametrize("a,b,av,bv,ansi,tr,want", [
    (_col(INT32), _col(INT32), 64, 64, 0, 0, "EINVAL"),                    # two scalars
    (_col(INT8), _col(INT16), None, None, 1, 0, "EINVAL"),                 # types differ (checkTypeEquals)
    (_col(BOOL8), _col(INT8), None, None, 1, 0, "EINVAL"),                 # types differ first (invalidType)
    (_col(BOOL8), _col(BOOL8), None, None, 0, 0, "EUNSUPPORTED"),
    (_col(UINT32), _col(UINT32), None, None, 0, 0, "EUNSUPPORTED"), (_col(DEC32), _col(DEC32), None, None, 0, 0, "EUNSUPPORTED"),
    (_col(STRING, 3), _col(STRING, 2), None, None, 1, 1, "EUNSUPPORTED"),  # the type before the rows and the mode
    (_col(INT8, 3), _col(INT8, 2), None, None, 1, 0, "EINVAL"),            # row counts (checkRows)
    (_col(INT8), _col(INT8), None, None, 1, 1, "EINVAL"),                  # ANSI and try (invalidMode)
    (_col(INT32, data=None), _col(INT32), None, None, 0, 0, "EINVAL"),     # missing data
    (_col(INT64, data=260), _col(INT64), None, None, 0, 0, "EINVAL"),      # misaligned data
    (_col(INT64), _col(INT64, 1, data=None), None, 64, 0, 0, "EINVAL"),    # a scalar without its value
    (_col(INT32, mask=256), _col(INT32), None, None, 0, 0, "OK_NEEDS_MASK"),
])
def test_multiply_errors_need_no_device(a, b, av, bv, ansi, tr, want):
    from srj_b200 import _native as N
    if want == "OK_NEEDS_MASK":
        assert _mul(a, b, av, bv, ansi, tr, mask=None)[0] == N.SRJ_EINVAL
        return
    code = getattr(N, "SRJ_" + want)
    rc, nulls, row = _mul(a, b, av, bv, ansi, tr)
    assert (rc, nulls, row) == (code, 0, -1)


def test_multiply_buffer_checks_need_no_device():
    from srj_b200 import _native as N
    E = N.SRJ_EINVAL
    assert _mul(_col(INT64), _col(INT64), out=None)[0] == E
    assert _mul(_col(INT64), _col(INT64), out=260)[0] == E                 # output at its element
    assert _mul(_col(INT32), _col(INT32), try_mode=1, mask=None)[0] == E   # try mode can make nulls
    assert _mul(_col(INT32), _col(INT32, 1), bv=64, mask=None)[0] == E     # a scalar can be null
    assert _mul(_col(INT32), _col(INT32), mask=258)[0] == E                # misaligned mask
    assert _mul(_col(INT32, 0, data=None), _col(INT32, 0, data=None), out=None, mask=None) == (N.SRJ_OK, 0, -1)
    assert _mul(_col(INT32, 0, data=None), _col(INT32, 7), bv=64, out=None, mask=None) == (N.SRJ_OK, 0, -1)   # scalar * empty
    lib = N.lib()
    a = _col(INT32)
    assert lib.srj_multiply(C.byref(a), None, C.byref(a), None, 0, 0, 256, 256, None, None, None) == E


def _round(inp, dp=-1, method=0, ansi=0, out=256, mask=256):
    from srj_b200 import _native as N
    row = C.c_int64(-5)
    rc = N.lib().srj_round(C.byref(inp), dp, method, ansi, out, mask, C.byref(row), None)
    return rc, row.value


@pytest.mark.parametrize("inp,method,want", [
    (_col(BOOL8), 0, "EUNSUPPORTED"), (_col(UINT32), 0, "EUNSUPPORTED"), (_col(STRING), 0, "EUNSUPPORTED"),
    (_col(BOOL8), 7, "EUNSUPPORTED"),                                       # the type before the method
    (_col(INT32), 2, "EINVAL"), (_col(FLOAT64), -1, "EINVAL"), (_col(DEC128, data=264), 9, "EINVAL"),
    (_col(INT32, data=None), 0, "EINVAL"), (_col(FLOAT64, data=260), 0, "EINVAL"),
    (_col(INT32, mask=256), 0, "OK_NEEDS_MASK"),
])
def test_round_errors_need_no_device(inp, method, want):
    from srj_b200 import _native as N
    if want == "OK_NEEDS_MASK":
        assert _round(inp, method=method, mask=None)[0] == N.SRJ_EINVAL
        return
    assert _round(inp, method=method) == (getattr(N, "SRJ_" + want), -1)


def test_round_buffer_checks_need_no_device():
    from srj_b200 import _native as N
    E = N.SRJ_EINVAL
    assert _round(_col(INT64), out=None)[0] == E
    assert _round(_col(INT32), out=258)[0] == E
    assert _round(_col(INT32), mask=258)[0] == E                           # a given mask is written: 4-byte aligned
    # an empty input returns before any check, the method's and the type's included (the reference's empty_like)
    for t, method in ((STRING, 0), (INT32, 5), (BOOL8, 9)):
        assert _round(_col(t, 0, data=None), method=method, out=None, mask=None) == (N.SRJ_OK, -1)
    lib = N.lib()
    assert lib.srj_round(None, 0, 0, 0, None, None, None, None) == E


def test_library_holds_the_sm90a_arithmetic_kernels_without_calls():
    from srj_b200 import _native as N
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", N.LIB_PATH], capture_output=True, text=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)
    for k, count in KERNELS.items():
        found = [f for f in funcs if re.search(r"\b_ZN3srj[^ ]*" + str(len(k)) + k, f.split("\n", 1)[0])]
        assert len(found) == count, (k, len(found))
        assert all(" CALL" not in f for f in found), k
    assert "sm_90a" in subprocess.run([cuobjdump, "-lelf", N.LIB_PATH], capture_output=True, text=True).stdout


def test_kernels_have_no_stack_frame_or_spills():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    with tempfile.TemporaryDirectory() as td:
        r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-ccbin", "/usr/bin/g++",
                            "--expt-relaxed-constexpr", "-Xptxas", "-v", "-c",
                            os.path.join(ROOT, "spark-rapids-jni_b200", "csrc", "arithmetic.cu"), "-o", os.path.join(td, "a.o")],
                           capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    props = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(props) == sum(KERNELS.values()) and all(p == ("0", "0", "0") for p in props), props
