"""CPU checks of the radix casts' surface: the two JNI shims compile against the stub headers and define exactly their
natives; the C ABI, its Python binding and the mirror agree; argument errors come back with their codes before any
device work; the radix kernels are in the library's sm_90a cubin with no subroutine call, stack frame or spill."""
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
KERNELS = 21   # conv parse (sizes, overflow) and write, int sizes and write for 8 types, hex offsets and chars
INT8, INT32, INT64, UINT8, FLOAT64, STRING, LIST = 1, 3, 4, 5, 10, 23, 24
ABI = {"srj_conv_workspace_bytes": 1, "srj_conv_sizes": 13, "srj_conv": 11, "srj_conv_overflow": 9,
       "srj_long_to_binary_workspace_bytes": 1, "srj_long_to_binary_sizes": 5, "srj_long_to_binary": 3,
       "srj_integers_to_string_workspace_bytes": 1, "srj_integers_to_string_sizes": 6, "srj_integers_to_string": 4,
       "srj_bytes_to_hex_sizes": 4, "srj_bytes_to_hex": 3}


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


def test_shims_define_exactly_their_natives():
    p = "Java_com_nvidia_spark_rapids_jni_"
    assert _natives("NumberConverterJni.cpp") == {p + "NumberConverter_convert", p + "NumberConverter_isConvertOverflow"}
    assert _natives("CastStringsRadixJni.cpp") == {p + "CastStrings_" + m for m in ("fromLongToBinary", "fromIntegersWithBase", "bytesToHex")}


def test_header_binding_and_mirror_agree():
    from srj_b200 import _native as N
    from srj_b200 import radix as RX
    from srj_b200.bloom import Scalar
    from srj_b200.cast import CastStrings
    hdr = open(os.path.join(ROOT, "include", "srj_b200.h")).read()
    for name, nargs in ABI.items():
        args = re.search(r"SRJ_API \w+ " + name + r"\s*\(([^)]*)\)", hdr).group(1)
        assert len(args.split(",")) == len(N.SYMBOLS[name][1]) == nargs, name
        assert hasattr(N.lib(), name)
    methods = {m for m in vars(RX.NumberConverter) if not m.startswith("_")}
    assert methods == {k + o for k in ("convert", "isConvertOverflow") for o in ("CvCvCv", "CvCvS", "CvSCv", "CvSS", "SCvCv", "SCvS", "SSCv")}
    assert all(callable(getattr(CastStrings, m)) for m in ("fromLongToBinary", "fromIntegersWithBase", "bytesToHex"))
    assert callable(Scalar.fromString)
    with pytest.raises(TypeError):
        RX.NumberConverter.convertCvSS(None, 10, 16)
    with pytest.raises(TypeError):
        CastStrings.bytesToHex(None)
    for f in ("radix.py", "cast.py"):
        src = open(os.path.join(ROOT, "spark-rapids-jni_b200", "srj_b200", f)).read()
        assert "oracle" not in re.sub(r'""".*?"""', "", src, flags=re.S)


def _col(t=STRING, rows=4, data=256, offsets=256, mask=None, children=None):
    from srj_b200 import _native as N
    c = N.SrjColumn()
    c.type_id, c.size, c.data, c.offsets, c.null_mask = t, rows, data, offsets, mask
    if children is not None:
        arr = (N.SrjColumn * len(children))(*children)
        c.children, c.num_children = arr, len(children)
        c._keep = arr
    return c


def _conv(inp, s=None, slen=0, fb=None, f=10, tb=None, t=16):
    from srj_b200 import _native as N
    nulls, total = C.c_int64(-5), C.c_int64(-5)
    ref = lambda c: C.byref(c) if c is not None else None
    rc = N.lib().srj_conv_sizes(ref(inp), s, slen, ref(fb), f, ref(tb), t, 256, 256, C.byref(nulls), C.byref(total), 256, None)
    flag = C.c_int32(-5)
    rc2 = N.lib().srj_conv_overflow(ref(inp), s, slen, ref(fb), f, ref(tb), t, C.byref(flag), None)
    return rc, rc2


def test_conv_argument_errors_need_no_device():
    from srj_b200 import _native as N
    E, U = N.SRJ_EINVAL, N.SRJ_EUNSUPPORTED
    assert _conv(_col(), fb=_col(INT32, rows=5)) == (E, E)                          # mismatched row counts
    assert _conv(_col(), tb=_col(INT32, rows=3)) == (E, E)
    assert _conv(None, s=256, slen=2, fb=_col(INT32, rows=3), tb=_col(INT32, rows=4)) == (E, E)
    assert _conv(_col(INT32)) == (U, U)                                               # wrong types
    assert _conv(_col(), fb=_col(INT64)) == (U, U)
    assert _conv(_col(), tb=_col(FLOAT64)) == (U, U)
    assert _conv(None, s=256, slen=2) == (E, E)                                       # scalar input, two scalar bases
    assert _conv(None, s=256, slen=-1, fb=_col(INT32)) == (E, E)                      # a null scalar
    assert _conv(None, s=None, slen=3, fb=_col(INT32)) == (E, E)
    assert _conv(_col(offsets=None)) == (E, E)


def _int_sizes(inp, base=10):
    from srj_b200 import _native as N
    total = C.c_int64(-5)
    return N.lib().srj_integers_to_string_sizes(C.byref(inp), base, 256, C.byref(total), 256, None)


def test_integer_and_hex_argument_errors_need_no_device():
    from srj_b200 import _native as N
    E, U = N.SRJ_EINVAL, N.SRJ_EUNSUPPORTED
    assert _int_sizes(_col(INT32), 8) == E and _int_sizes(_col(FLOAT64), 8) == E      # base 8: the base before the type
    assert "Bases supported 10, 16; Actual: 8" in N.lib().srj_last_error().decode()
    assert _int_sizes(_col(FLOAT64)) == U and _int_sizes(_col(STRING)) == U
    assert _int_sizes(_col(INT32, data=None)) == E and _int_sizes(_col(INT64, data=260)) == E
    total = C.c_int64(0)
    assert N.lib().srj_long_to_binary_sizes(C.byref(_col(INT32)), 256, C.byref(total), 256, None) == U
    assert N.lib().srj_long_to_binary_sizes(C.byref(_col(INT64, rows=-1)), 256, C.byref(total), 256, None) == E
    hx = lambda c: N.lib().srj_bytes_to_hex_sizes(C.byref(c), 256, C.byref(total), None)
    assert hx(_col(LIST, children=[_col(INT8)])) == U                                # a LIST whose child is not UINT8
    assert hx(_col(LIST)) == U and hx(_col(INT32)) == U
    assert hx(_col(STRING, offsets=None)) == E
    out = _col(STRING, mask=None)
    assert N.lib().srj_bytes_to_hex(C.byref(_col(mask=256)), C.byref(out), None) == E   # a masked input needs an output mask


def test_library_holds_the_sm90a_kernels_without_calls():
    from srj_b200 import _native as N
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", N.LIB_PATH], capture_output=True, text=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)
    found = [f for f in funcs if re.search(r"radix_cu", f.split("\n", 1)[0])]
    assert len(found) == KERNELS
    assert all(" CALL" not in f for f in found)


def test_kernels_have_no_stack_frame_or_spills():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    with tempfile.TemporaryDirectory() as td:
        r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-ccbin", "/usr/bin/g++",
                            "--expt-relaxed-constexpr", "-Xptxas", "-v", "-c", os.path.join(CSRC, "radix.cu"),
                            "-o", os.path.join(td, "r.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    props = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(props) == KERNELS and all(p == ("0", "0", "0") for p in props), props
