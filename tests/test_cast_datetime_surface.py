"""CPU checks of the CastStrings surface: the JNI shim compiles against the stub headers and defines exactly the two natives,
the header, the ctypes binding and the Python mirror agree, the cast kernels compile with no CALL, stack frame or spill,
and sharing the zone evaluation left every timezone.cu kernel's SASS unchanged."""
import os
import re
import shutil
import subprocess
import sys
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
JNI = os.path.join(ROOT, "spark-rapids-jni_b200", "jni")
PREFIX = "Java_com_nvidia_spark_rapids_jni_CastStrings_"
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def test_shim_defines_exactly_the_two_natives():
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    with tempfile.TemporaryDirectory() as td:
        obj = os.path.join(td, "c.o")
        r = subprocess.run([gxx, "-std=c++17", "-Wall", "-Werror", "-fPIC", "-DSRJ_JNI_STUBS", "-c", os.path.join(JNI, "CastStringsJni.cpp"),
                            "-o", obj], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        syms = subprocess.run(["nm", "--defined-only", obj], capture_output=True, text=True).stdout
    defined = sorted(s.split()[-1] for s in syms.splitlines() if s.split()[-1].startswith("Java_"))
    assert defined == [PREFIX + "parseDateStringsToDate", PREFIX + "parseTimestampStringsToIntermediate"]


def test_header_binding_and_mirror_agree():
    sys.path.insert(0, os.path.join(ROOT, "spark-rapids-jni_b200"))
    from srj_b200 import _native as N
    hdr = open(os.path.join(ROOT, "include", "srj_b200.h")).read()
    for name, nargs in (("srj_cast_parse_timestamps", 18), ("srj_cast_parse_dates", 5)):
        m = re.search(r"SRJ_API int %s\((.*?)\);" % name, hdr, re.S)
        assert m, name
        assert len(m.group(1).split(",")) == nargs == len(N.SYMBOLS[name][1]), name
    assert "#define SRJ_SPARK_VANILLA 0" in hdr and "#define SRJ_SPARK_DATABRICKS 1" in hdr
    from srj_b200.cast import Version
    assert (Version.VANILLA_SPARK, Version.DATABRICKS) == (0, 1)
    src = open(os.path.join(ROOT, "spark-rapids-jni_b200", "srj_b200", "cast.py")).read()
    assert "srj_cast_parse_timestamps" in src and "srj_cast_parse_dates" in src


def _compile(src, td, extra=()):
    obj = os.path.join(td, "k.o")
    r = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-ccbin", "/usr/bin/g++",
                        "--expt-relaxed-constexpr", "-Xptxas", "-v", "-I", os.path.join(ROOT, "include"), *extra, "-c",
                        os.path.join(ROOT, "spark-rapids-jni_b200", "csrc", src), "-o", obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return obj, r.stderr


def test_cast_kernels_have_no_call_stack_frame_or_spill():
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    with tempfile.TemporaryDirectory() as td:
        obj, log = _compile("cast_datetime.cu", td)
        sass = subprocess.run([os.path.join(os.path.dirname(NVCC), "cuobjdump"), "-sass", obj], capture_output=True, text=True).stdout
    props = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert len(props) == 2 and all(p == ("0", "0", "0") for p in props), props
    funcs = re.split(r"\n\s*Function : ", sass)[1:]
    assert len(funcs) == 2
    assert sum("parse_ts_kernel" in f.split("\n", 1)[0] for f in funcs) == 1
    assert sum("parse_date_kernel" in f.split("\n", 1)[0] for f in funcs) == 1
    for f in funcs:
        assert " CALL" not in f and "STL" not in f and "LDL" not in f, f.split("\n", 1)[0]


def _anon(text):
    """Kernel names without the anonymous-namespace hashes, which nvcc derives from the translation unit, not the kernel."""
    return re.sub(r"_GLOBAL__N__(?:[0-9a-f]+_)?(\d+_\w+?_cu)_[0-9a-f]{8}", r"_GLOBAL__N__\1_", text)


def _kernel_hashes(obj):
    import hashlib
    out = subprocess.run([os.path.join(os.path.dirname(NVCC), "cuobjdump"), "-sass", obj], capture_output=True, text=True, check=True).stdout
    out = _anon(out)
    hashes = {}
    for part in re.split(r"\n\s*Function : ", out)[1:]:
        name, body = part.split("\n", 1)
        hashes[name.strip()] = hashlib.sha256(body.split("\n\t\t..........", 1)[0].encode()).hexdigest()
    return hashes


def test_timezone_kernels_keep_their_sass_whatever_the_unit_hash():
    """Sharing the zone evaluation with the cast (tz_eval.cuh) leaves every timezone.cu kernel's SASS as it was."""
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from golden import timezone_sass as TS
    if TS.NVCC_RELEASE not in subprocess.run([NVCC, "--version"], capture_output=True, text=True).stdout:
        pytest.skip("the recorded SASS is of another nvcc release")
    with tempfile.TemporaryDirectory() as td:
        obj, _ = _compile("timezone.cu", td)
        assert _kernel_hashes(obj) == {_anon(k): v for k, v in TS.KERNELS.items()}
