"""CPU checks of the DecimalUtils surface: the JNI shim compiles against the stub headers and defines exactly the five
arithmetic natives of the reference's DecimalUtils (floatingPointToDecimal, the sixth, is absent); the C ABI, its Python
binding and the Python mirror agree; every argument error comes back without touching a device; the shipped library
holds the sm_90a kernels, with no division subroutine call, stack frame or spill."""
import ctypes as C
import os
import re
import shutil
import subprocess
import tempfile

import pytest

from oracle import decimal as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
JNI = os.path.join(ROOT, "spark-rapids-jni_b200", "jni")
PREFIX = "Java_com_nvidia_spark_rapids_jni_DecimalUtils_"
NATIVES = {PREFIX + m for m in ("multiply128", "divide128", "remainder128", "add128", "subtract128")}
DEC128, INT64 = 27, 4


def test_shim_defines_exactly_the_five_natives():
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    with tempfile.TemporaryDirectory() as td:
        obj = os.path.join(td, "d.o")
        r = subprocess.run([gxx, "-std=c++17", "-Wall", "-Werror", "-fPIC", "-DSRJ_JNI_STUBS", "-c", os.path.join(JNI, "DecimalUtilsJni.cpp"),
                            "-o", obj], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        syms = subprocess.run(["nm", "-g", "--defined-only", obj], capture_output=True, text=True).stdout
    found = {l.split()[-1] for l in syms.splitlines() if " T " in l and l.split()[-1].startswith("Java_")}
    assert found == NATIVES
    assert PREFIX + "floatingPointToDecimal" not in found


def test_header_binding_and_mirror_agree():
    from srj_b200 import _native as N
    from srj_b200 import decimal as D
    hdr = open(os.path.join(ROOT, "include", "srj_b200.h")).read()
    declared = set(re.findall(r"SRJ_API[^;]*?\b(srj_[a-z0-9_]+)\s*\(", hdr))
    assert {d for d in declared if "decimal" in d} == {"srj_decimal128_binary"}
    assert hasattr(N.lib(), "srj_decimal128_binary") and "srj_decimal128_binary" in N.SYMBOLS
    defines = {k: int(v) for k, v in re.findall(r"#define SRJ_DECIMAL_([A-Z_]+) (\d+)", hdr)}
    want = {"MULTIPLY": O.MULTIPLY, "DIVIDE": O.DIVIDE, "INTEGER_DIVIDE": O.INTEGER_DIVIDE, "REMAINDER": O.REMAINDER, "ADD": O.ADD,
            "SUBTRACT": O.SUBTRACT}
    assert defines == want
    assert (D.MULTIPLY, D.DIVIDE, D.INTEGER_DIVIDE, D.REMAINDER, D.ADD, D.SUBTRACT) == tuple(want[k] for k in want)
    for m in ("multiply128", "divide128", "integerDivide128", "remainder128", "add128", "subtract128"):
        assert callable(getattr(D.DecimalUtils, m))
    src = open(os.path.join(ROOT, "spark-rapids-jni_b200", "srj_b200", "decimal.py")).read()
    assert "oracle" not in re.sub(r'""".*?"""', "", src, flags=re.S)


def _col(t=DEC128, rows=4, scale=0, data=16, mask=None):
    from srj_b200 import _native as N
    c = N.SrjColumn()
    c.type_id, c.scale, c.size, c.data, c.null_mask = t, scale, rows, data, mask
    return c


def _call(op, a, b, so=0, ovf=16, out=16, mask=None, nulls=True):
    from srj_b200 import _native as N
    n = C.c_int64(-1)
    return N.lib().srj_decimal128_binary(op, C.byref(a) if a is not None else None, C.byref(b) if b is not None else None, so, 1, ovf, out,
                                         mask, C.byref(n) if nulls else None, None)


@pytest.mark.parametrize("op,a,b,so,kw,want", [
    (6, {}, {}, 0, {}, "EINVAL"), (-1, {}, {}, 0, {}, "EINVAL"),
    (0, dict(t=INT64), {}, 0, {}, "EUNSUPPORTED"), (1, {}, dict(t=INT64), 0, {}, "EUNSUPPORTED"),
    (0, dict(rows=4), dict(rows=5), 0, {}, "EINVAL"), (0, dict(rows=-1), dict(rows=-1), 0, {}, "EINVAL"),
    (0, {}, {}, 39, {}, "EINVAL"),                                   # multiply: "divisor too big"
    (0, dict(scale=-20), dict(scale=-20), -1, {}, "EINVAL"),         # 39 again, from the inputs' scales
    (1, {}, {}, 39, {}, "EINVAL"), (2, {}, {}, -115, {}, "EINVAL"),  # divide outside [-114, 38]
    (3, {}, {}, 39, {}, "EINVAL"),                                   # remainder: a divisor rounding by 10^39
    (3, dict(scale=77), {}, 0, {}, "EINVAL"),                        # remainder: the dividend scaled by 10^77
    (4, dict(scale=77), {}, 0, {}, "EINVAL"),                        # add: |a_scale - b_scale| = 77 (Java lets it through)
    (5, {}, {}, 39, {}, "EINVAL"), (4, {}, {}, -77, {}, "EINVAL"),
    (0, dict(data=None), {}, 0, {}, "EINVAL"), (0, dict(data=12), {}, 0, {}, "EINVAL"),   # no data; not 8-byte aligned
    (0, {}, {}, 0, dict(ovf=None), "EINVAL"), (0, {}, {}, 0, dict(out=None), "EINVAL"), (0, {}, {}, 0, dict(out=12), "EINVAL"),
    (0, dict(mask=64), {}, 0, {}, "EINVAL"),                         # a mask but no output mask
    (0, {}, dict(mask=64), 0, dict(mask=64, nulls=False), "EINVAL"),  # a mask but no null count
])
def test_errors_need_no_device(op, a, b, so, kw, want):
    from srj_b200 import _native as N
    assert _call(op, _col(**a), _col(**b), so, **kw) == getattr(N, "SRJ_" + want)


def test_valid_scale_edges_and_zero_rows_touch_nothing():
    from srj_b200 import _native as N
    assert _call(0, None, _col()) == N.SRJ_EINVAL
    for op, sa, sb, so in ((0, 0, 0, 38), (1, 0, 0, 38), (1, 0, 0, -114), (3, 0, 0, 38), (3, 76, 0, 0), (4, 76, 0, 0), (4, 0, 0, 38),
                           (4, 0, 0, -76), (0, 0, 0, -1000)):
        assert _call(op, _col(rows=0, scale=sa), _col(rows=0, scale=sb), so, ovf=None, out=None, nulls=False) == N.SRJ_OK, (op, sa, sb, so)
        O.check_scales(op, sa, sb, so)
    # multiply's product scale is bounded only from above: far below, every row overflows (the kernel clamps e0 at -40)
    for so in (-(2**31) + 1, -(2**31), -2**31 + 77):
        assert _call(0, _col(rows=0, scale=2**31 - 1), _col(rows=0, scale=2**31 - 1), so, ovf=None, out=None, nulls=False) == N.SRJ_OK
        O.check_scales(0, 0, 0, so)
    for op, sa, sb, so in ((0, 0, 0, 39), (2, 0, 0, 39), (3, 77, 0, 0), (4, 77, 0, 0), (5, 0, 0, -77)):
        with pytest.raises(ValueError):
            O.check_scales(op, sa, sb, so)


def test_mirror_raises_the_java_exceptions():
    import srj_b200 as S
    from srj_b200.decimal import DecimalUtils
    a = S.ColumnView(S.DType(S.DType.DECIMAL128, 0), 0)
    b = S.ColumnView(S.DType(S.DType.DECIMAL128, -78), 0)
    for fn in (DecimalUtils.add128, DecimalUtils.subtract128):
        with pytest.raises(ValueError, match="256-bit"):
            fn(a, b, 0)
    for fn in (lambda: DecimalUtils.multiply128(None, a, 0), lambda: DecimalUtils.divide128(a, None, 0),
               lambda: DecimalUtils.integerDivide128(None, None), lambda: DecimalUtils.remainder128(None, a, 0)):
        with pytest.raises(TypeError):
            fn()


def test_library_holds_the_sm90a_decimal_kernels():
    from srj_b200 import _native as N
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", N.LIB_PATH], capture_output=True, text=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)
    maps = [f for f in funcs if "dec_map_kernel" in f.split("\n", 1)[0]]
    # one per op and per-call path: multiply (cast or not) 2, divide and integral divide 3 each, remainder 4, add and
    # subtract 3 each
    assert len(maps) == 18, [f.split("\n", 1)[0] for f in maps]
    for f in maps + [f for f in funcs if "dec_mask_and_kernel" in f.split("\n", 1)[0]]:
        assert " CALL" not in f, f.split("\n", 1)[0]
    assert "sm_90a" in subprocess.run([cuobjdump, "-lelf", N.LIB_PATH], capture_output=True, text=True).stdout


def test_kernels_have_no_stack_frame_or_spills():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    with tempfile.TemporaryDirectory() as td:
        r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-ccbin", "/usr/bin/g++",
                            "--expt-relaxed-constexpr", "-Xptxas", "-v", "-c",
                            os.path.join(ROOT, "spark-rapids-jni_b200", "csrc", "decimal.cu"), "-o", os.path.join(td, "d.o")],
                           capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    props = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert props and all(p == ("0", "0", "0") for p in props), props
