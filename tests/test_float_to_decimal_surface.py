"""CPU checks of the floatingPointToDecimal surface: the JNI shim DecimalUtilsCastJni.cpp compiles against the stub headers
and defines exactly that native, and with DecimalUtilsJni.cpp all six natives of the reference's DecimalUtils.java; the
C ABI, its Python binding and the Python mirror agree; every argument error comes back with its code before any device
work, and zero rows touch nothing; the f2d kernels are in the library's sm_90a cubin with no subroutine call, stack frame
or spill; the 128-by-128 quotient dec::udiv128 they divide with matches exact integers."""
import ctypes as C
import os
import re
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
JNI = os.path.join(ROOT, "spark-rapids-jni_b200", "jni")
CSRC = os.path.join(ROOT, "spark-rapids-jni_b200", "csrc")
PREFIX = "Java_com_nvidia_spark_rapids_jni_DecimalUtils_"
# DecimalUtils.java:215-225
ALL_NATIVES = {PREFIX + m for m in ("multiply128", "divide128", "remainder128", "add128", "subtract128", "floatingPointToDecimal")}
KERNELS = 6                                     # f2d_kernel: FLOAT32 / FLOAT64 x DECIMAL32 / 64 / 128
INT32, FLOAT32, FLOAT64, STRING, DEC32, DEC64, DEC128 = 3, 9, 10, 23, 25, 26, 27


def _natives(src):
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    with tempfile.TemporaryDirectory() as td:
        obj = os.path.join(td, "d.o")
        r = subprocess.run([gxx, "-std=c++17", "-Wall", "-Werror", "-fPIC", "-DSRJ_JNI_STUBS", "-c", os.path.join(JNI, src), "-o", obj],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        syms = subprocess.run(["nm", "-g", "--defined-only", obj], capture_output=True, text=True).stdout
    return {l.split()[-1] for l in syms.splitlines() if " T " in l and l.split()[-1].startswith("Java_")}


def test_shim_defines_exactly_the_one_native_and_completes_the_class():
    cast = _natives("DecimalUtilsCastJni.cpp")
    assert cast == {PREFIX + "floatingPointToDecimal"}
    arith = _natives("DecimalUtilsJni.cpp")
    assert not cast & arith and cast | arith == ALL_NATIVES


def test_header_binding_and_mirror_agree():
    from srj_b200 import _native as N
    from srj_b200 import decimal as D
    hdr = open(os.path.join(ROOT, "include", "srj_b200.h")).read()
    args = re.search(r"SRJ_API int srj_float_to_fixed_point\s*\(([^)]*)\)", hdr).group(1)
    assert len(args.split(",")) == len(N.SYMBOLS["srj_float_to_fixed_point"][1]) == 9
    assert hasattr(N.lib(), "srj_float_to_fixed_point")
    assert callable(D.DecimalUtils.floatingPointToDecimal)
    r = D.CastFloatToDecimalResult(None, -1)
    assert r.result is None and r.failureRowId == -1
    with pytest.raises(TypeError):
        D.DecimalUtils.floatingPointToDecimal(None, D.DType(DEC64, -2), 18)
    src = open(os.path.join(ROOT, "spark-rapids-jni_b200", "srj_b200", "decimal.py")).read()
    assert "oracle" not in re.sub(r'""".*?"""', "", src, flags=re.S)


def _col(t=FLOAT64, rows=4, data=256, mask=None):
    from srj_b200 import _native as N
    c = N.SrjColumn()
    c.type_id, c.size, c.data, c.null_mask = t, rows, data, mask
    return c


def _cast(inp, out_type=DEC64, precision=18, scale=-2, out=256, mask=256, counts=True):
    from srj_b200 import _native as N
    nulls, row = C.c_int64(-5), C.c_int64(-5)
    rc = N.lib().srj_float_to_fixed_point(C.byref(inp) if inp is not None else None, out_type, precision, scale, out, mask,
                                          C.byref(nulls) if counts else None, C.byref(row) if counts else None, None)
    return rc, nulls.value, row.value


@pytest.mark.parametrize("inp,out_type,precision,scale,want", [
    (_col(INT32), DEC64, 18, -2, "EUNSUPPORTED"), (_col(STRING), DEC64, 18, -2, "EUNSUPPORTED"),
    (_col(FLOAT64), INT32, 9, 0, "EUNSUPPORTED"), (_col(FLOAT32), FLOAT64, 9, 0, "EUNSUPPORTED"),
    (_col(INT32), DEC64, 99, 99, "EUNSUPPORTED"),                          # the types before the domain
    (_col(FLOAT64), DEC32, 10, 0, "EINVAL"), (_col(FLOAT64), DEC32, 0, 0, "EINVAL"), (_col(FLOAT64), DEC64, 19, 0, "EINVAL"),
    (_col(FLOAT64), DEC128, 39, 0, "EINVAL"), (_col(FLOAT32), DEC128, -1, 0, "EINVAL"),
    (_col(FLOAT64), DEC32, 9, -10, "EINVAL"), (_col(FLOAT64), DEC64, 5, -6, "EINVAL"),   # Spark scale above the precision
    (_col(FLOAT64), DEC128, 38, 39, "EINVAL"), (_col(FLOAT64), DEC64, 18, 39, "EINVAL"),  # Spark scale below -38
    (_col(FLOAT64, rows=-1), DEC64, 18, -2, "EINVAL"),
    (_col(FLOAT64, data=None), DEC64, 18, -2, "EINVAL"), (_col(FLOAT64, data=260), DEC64, 18, -2, "EINVAL"),
    (_col(FLOAT32, data=258), DEC32, 9, -2, "EINVAL"),
])
def test_argument_errors_need_no_device(inp, out_type, precision, scale, want):
    from srj_b200 import _native as N
    assert _cast(inp, out_type, precision, scale) == (getattr(N, "SRJ_" + want), 0, -1)


@pytest.mark.parametrize("out_type,precision,scale", [(DEC32, 1, -1), (DEC32, 9, -9), (DEC32, 9, 38), (DEC64, 18, -18),
                                                      (DEC64, 1, 38), (DEC128, 38, -38), (DEC128, 38, 38)])
def test_the_domain_edges_are_accepted(out_type, precision, scale):
    from srj_b200 import _native as N
    assert _cast(_col(FLOAT64, rows=0, data=None), out_type, precision, scale, out=None, mask=None) == (N.SRJ_OK, 0, -1)


def test_buffer_checks_need_no_device():
    from srj_b200 import _native as N
    E = N.SRJ_EINVAL
    assert _cast(_col(), out=None)[0] == E
    assert _cast(_col(), out=260)[0] == E                                   # DECIMAL64 output at 8 bytes
    assert _cast(_col(), out_type=DEC128, precision=38, out=260)[0] == E    # DECIMAL128 needs 8 bytes
    assert _cast(_col(FLOAT32), out_type=DEC32, precision=9, out=258)[0] == E
    assert _cast(_col(), mask=None)[0] == E                                 # the mask is always written
    assert _cast(_col(), mask=258)[0] == E
    assert _cast(_col(), counts=False)[0] == E                              # no null-count or failure-row pointer
    assert _cast(None)[0] == E
    # zero rows touch nothing: no buffer is needed or written
    assert _cast(_col(rows=0, data=None), out=None, mask=None) == (N.SRJ_OK, 0, -1)


def test_library_holds_the_sm90a_kernels_without_calls():
    from srj_b200 import _native as N
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", N.LIB_PATH], capture_output=True, text=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)
    found = [f for f in funcs if re.search(r"\b_ZN3srj[^ ]*10f2d_kernel", f.split("\n", 1)[0])]
    assert len(found) == KERNELS
    assert all(" CALL" not in f for f in found)


def test_kernels_have_no_stack_frame_or_spills():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    with tempfile.TemporaryDirectory() as td:
        r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-ccbin", "/usr/bin/g++",
                            "--expt-relaxed-constexpr", "-Xptxas", "-v", "-c", os.path.join(CSRC, "float_to_decimal.cu"),
                            "-o", os.path.join(td, "f.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    props = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(props) == KERNELS and all(p == ("0", "0", "0") for p in props), props


def test_udiv128_matches_exact_integers():
    """dec::udiv128 compiled as plain C++: quotients of random and edge dividends by powers of ten, their values mod 2^64
    and 2^128, small and large divisors, and 0 (all ones)."""
    import random
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    src = r'''
#include <cstdio>
#include "decimal_arith.cuh"
using namespace srj::dec;
int main() {
  unsigned long long a, b, c, d;
  while (std::scanf("%llx %llx %llx %llx", &a, &b, &c, &d) == 4) {
    const u128 n = (static_cast<u128>(a) << 64) | b, dv = (static_cast<u128>(c) << 64) | d;
    const u128 q = udiv128(n, make_div(dv));
    std::printf("%016llx%016llx\n", static_cast<unsigned long long>(q >> 64), static_cast<unsigned long long>(q));
  }
}
'''
    M = (1 << 128) - 1
    rng = random.Random(5)
    divisors = [10 ** k & M for k in range(0, 128)] + [10 ** k & ((1 << 64) - 1) for k in range(0, 64)] + [1, 3, 7, (1 << 64) + 1, M]
    dividends = [0, 1, M, M - 1, 1 << 127, (1 << 64) - 1, 1 << 64] + [rng.getrandbits(rng.choice([32, 64, 100, 128])) for _ in range(200)]
    pairs = [(n, d) for d in divisors for n in dividends]
    with tempfile.TemporaryDirectory() as td:
        exe = os.path.join(td, "u")
        r = subprocess.run([gxx, "-std=c++17", "-O1", "-I", CSRC, "-x", "c++", "-", "-o", exe], input=src, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        inp = "".join(f"{n >> 64:x} {n & (2**64 - 1):x} {d >> 64:x} {d & (2**64 - 1):x}\n" for n, d in pairs)
        out = subprocess.run([exe], input=inp, capture_output=True, text=True).stdout.split()
    assert len(out) == len(pairs)
    for (n, d), q in zip(pairs, out):
        assert int(q, 16) == (n // d if d else M), (n, d)
