"""CPU checks of the BloomFilter surface: the JNI shim BloomFilterJni.cpp compiles against the stub headers and defines
exactly the five natives of the reference's BloomFilter.java:112-118; the C ABI, its Python binding and the Python mirror
expose the same capabilities; the C ABI's argument checks need no device; the shipped library holds the sm_90a bloom
kernels, and the put / probe kernels call no division subroutine."""
import ctypes as C
import os
import re
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
JNI = os.path.join(ROOT, "spark-rapids-jni_b200", "jni")
NATIVES = {f"Java_com_nvidia_spark_rapids_jni_BloomFilter_{m}" for m in ("creategpu", "put", "merge", "probe", "probebuffer")}
ABI = {"srj_bloom_filter_sizes", "srj_bloom_filter_init", "srj_bloom_filter_put", "srj_bloom_filter_probe",
       "srj_bloom_filter_merge_workspace_bytes", "srj_bloom_filter_merge"}
INT64, INT32 = 4, 3


def test_shim_defines_exactly_the_five_natives():
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    with tempfile.TemporaryDirectory() as td:
        obj = os.path.join(td, "shim.o")
        r = subprocess.run([gxx, "-std=c++17", "-Wall", "-Werror", "-fPIC", "-DSRJ_JNI_STUBS", "-c", os.path.join(JNI, "BloomFilterJni.cpp"),
                            "-o", obj], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        syms = subprocess.run(["nm", "-g", "--defined-only", obj], capture_output=True, text=True).stdout
    assert {l.split()[-1] for l in syms.splitlines() if " T " in l and l.split()[-1].startswith("Java_")} == NATIVES


def test_header_binding_and_mirror_agree():
    from srj_b200 import _native as N
    from srj_b200.bloom import BloomFilter
    hdr = open(os.path.join(ROOT, "include", "srj_b200.h")).read()
    declared = set(re.findall(r"SRJ_API[^;]*?\b(srj_[a-z0-9_]+)\s*\(", hdr))
    assert {d for d in declared if d.startswith("srj_bloom")} == ABI
    assert ABI <= set(N.SYMBOLS)
    lib = N.lib()
    for name in ABI:
        assert hasattr(lib, name)
    assert (BloomFilter.VERSION_1, BloomFilter.VERSION_2, BloomFilter.DEFAULT_SEED) == (1, 2, 0)
    for m in ("create", "put", "merge", "probe", "probebuffer"):
        assert callable(getattr(BloomFilter, m))


def test_bloom_mirror_does_not_import_the_oracle():
    src = open(os.path.join(ROOT, "spark-rapids-jni_b200", "srj_b200", "bloom.py")).read()
    assert "oracle" not in re.sub(r'""".*?"""', "", src, flags=re.S)


@pytest.mark.parametrize("args", [(3, 3, 64), (1, 0, 64), (2, -1, 64), (1, 3, 0), (2, 3, -5), (1, 3, (2**31 - 1) * 64 + 1),
                                  (2, 3, 2**62)])
def test_sizes_rejects_bad_parameters(args):
    from srj_b200 import _native as N
    longs, total = C.c_int32(0), C.c_int64(0)
    assert N.lib().srj_bloom_filter_sizes(*args, C.byref(longs), C.byref(total)) == N.SRJ_EINVAL


def test_sizes():
    from srj_b200 import _native as N
    lib = N.lib()
    longs, total = C.c_int32(0), C.c_int64(0)
    for version, bits, want_longs in [(1, 1, 1), (1, 64, 1), (1, 65, 2), (2, 29_193_763, 456_153), (2, 2**33, 2**27)]:
        assert lib.srj_bloom_filter_sizes(version, 5, bits, C.byref(longs), C.byref(total)) == N.SRJ_OK
        assert longs.value == want_longs and total.value == (12 if version == 1 else 16) + 8 * want_longs
    # the largest bit count Spark's BitArray allows still needs a buffer over INT32_MAX bytes
    assert lib.srj_bloom_filter_sizes(2, 5, (2**31 - 1) * 64, C.byref(longs), C.byref(total)) == N.SRJ_EINVAL


def test_c_abi_argument_checks_need_no_device():
    from srj_b200 import _native as N
    lib = N.lib()
    col = N.SrjColumn()
    col.type_id, col.size = INT32, 0
    assert lib.srj_bloom_filter_put(None, 0, C.byref(col), None) == N.SRJ_EUNSUPPORTED
    assert lib.srj_bloom_filter_probe(None, 0, C.byref(col), None, None, None) == N.SRJ_EUNSUPPORTED
    col.type_id = INT64
    assert lib.srj_bloom_filter_put(None, 0, C.byref(col), None) == N.SRJ_EINVAL           # truncated filter
    assert lib.srj_bloom_filter_probe(None, 11, C.byref(col), None, None, None) == N.SRJ_EINVAL
    assert lib.srj_bloom_filter_init(3, 3, 1, 0, None, None) == N.SRJ_EINVAL
    assert lib.srj_bloom_filter_init(1, 0, 1, 0, None, None) == N.SRJ_EINVAL
    assert lib.srj_bloom_filter_init(1, 3, 0, 0, None, None) == N.SRJ_EINVAL
    assert lib.srj_bloom_filter_merge(None, 0, 0, None, None, None) == N.SRJ_EINVAL
    assert lib.srj_bloom_filter_merge(None, 8, 1, None, None, None) == N.SRJ_EINVAL
    assert lib.srj_bloom_filter_merge_workspace_bytes() >= 4


@pytest.mark.parametrize("args", [(3, 3, 64, 0), (1, 0, 64, 0), (2, 3, 0, 0), (2, 3, (2**31 - 1) * 64 + 1, 0)])
def test_mirror_create_raises_value_error_before_touching_the_device(args):
    from srj_b200.bloom import BloomFilter
    with pytest.raises(ValueError):
        BloomFilter.create(*args)


def test_library_holds_the_sm90a_bloom_kernels_without_division_calls():
    from srj_b200 import _native as N
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", N.LIB_PATH], capture_output=True, text=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)
    names = [f.split("\n", 1)[0] for f in funcs]
    for k in ("bloom_put_kernel", "bloom_probe_kernel", "bloom_merge_or_kernel", "bloom_merge_check_kernel", "bloom_init_kernel"):
        assert any(k in n for n in names), f"kernel {k} missing from the cubin"
    hot = [f for f in funcs if "bloom_put_kernel" in f.split("\n", 1)[0] or "bloom_probe_kernel" in f.split("\n", 1)[0]]
    assert len(hot) == 8                                          # V1 / V2 x vector / scalar keys, put and probe
    for f in hot:
        assert "CALL" not in f, "a division subroutine is left in " + f.split("\n", 1)[0]
    put = [f for f in hot if "bloom_put_kernel" in f.split("\n", 1)[0]]
    assert all("REDG.E.OR" in f and "ATOMG" not in f for f in put)    # atomicOr with the result unused
    assert "sm_90a" in subprocess.run([cuobjdump, "-lelf", N.LIB_PATH], capture_output=True, text=True).stdout
