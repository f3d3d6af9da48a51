"""CPU checks of the SHA-2 / hostCrc32 surface: the JNI shim HashSha2Jni.cpp compiles against the stub headers and defines
exactly the five natives HashJni.cpp lacks (together: all nine of the reference's Hash.java:176-190), the C ABI, its
Python binding and the Python mirror expose the same capabilities, and the shipped library holds the sm_90a SHA kernels."""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
JNI = os.path.join(ROOT, "spark-rapids-jni_b200", "jni")

SHA2_NATIVES = ["Java_com_nvidia_spark_rapids_jni_Hash_sha224NullsPreserved", "Java_com_nvidia_spark_rapids_jni_Hash_sha256NullsPreserved",
                "Java_com_nvidia_spark_rapids_jni_Hash_sha384NullsPreserved", "Java_com_nvidia_spark_rapids_jni_Hash_sha512NullsPreserved",
                "Java_com_nvidia_spark_rapids_jni_Hash_hostCrc32"]
# Hash.java:176-190 of the reference: every native of the class
HASH_NATIVES = {"getMaxStackDepth", "murmurHash32", "xxhash64", "hiveHash", "sha224NullsPreserved", "sha256NullsPreserved",
                "sha384NullsPreserved", "sha512NullsPreserved", "hostCrc32"}


def _natives(src):
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    with tempfile.TemporaryDirectory() as td:
        obj = os.path.join(td, "shim.o")
        r = subprocess.run([gxx, "-std=c++17", "-Wall", "-Werror", "-fPIC", "-DSRJ_JNI_STUBS", "-c", os.path.join(JNI, src), "-o", obj],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        syms = subprocess.run(["nm", "-g", "--defined-only", obj], capture_output=True, text=True).stdout
    return {l.split()[-1] for l in syms.splitlines() if " T " in l and l.split()[-1].startswith("Java_")}


def test_sha2_shim_defines_exactly_the_five_natives():
    assert _natives("HashSha2Jni.cpp") == set(SHA2_NATIVES)


def test_hash_shims_together_define_every_native_of_hash_java():
    prefix = "Java_com_nvidia_spark_rapids_jni_Hash_"
    both = _natives("HashJni.cpp") | _natives("HashSha2Jni.cpp")
    assert {s[len(prefix):] for s in both} == HASH_NATIVES


def test_header_binding_and_mirror_agree():
    from srj_b200 import _native as N
    import srj_b200 as S
    hdr = open(os.path.join(ROOT, "include", "srj_b200.h")).read()
    new = {"srj_sha2_workspace_bytes", "srj_sha2_sizes", "srj_sha2_hash", "srj_host_crc32"}
    declared = set(re.findall(r"SRJ_API[^;]*?\b(srj_[a-z0-9_]+)\s*\(", hdr))
    assert new <= declared and new <= set(N.SYMBOLS)
    lib = N.lib()
    for name in new:
        assert hasattr(lib, name)
    for m in ("sha224NullsPreserved", "sha256NullsPreserved", "sha384NullsPreserved", "sha512NullsPreserved", "hostCrc32"):
        assert callable(getattr(S.Hash, m))


def test_mirror_rejects_non_string_columns_before_touching_the_device():
    import srj_b200 as S
    with pytest.raises(ValueError):
        S.Hash.sha256NullsPreserved(None)
    with pytest.raises(ValueError):
        S.Hash.sha512NullsPreserved(S.ColumnVector(S.DType.INT32, 0, None))


def test_c_abi_argument_checks_need_no_device():
    import ctypes as C
    from srj_b200 import _native as N
    lib = N.lib()
    col = N.SrjColumn()
    col.type_id, col.size = 3, 0                                   # INT32
    total = C.c_int64(0)
    assert lib.srj_sha2_sizes(256, C.byref(col), None, C.byref(total), None, None) == N.SRJ_EUNSUPPORTED
    col.type_id = 23                                               # STRING
    assert lib.srj_sha2_sizes(257, C.byref(col), None, C.byref(total), None, None) == N.SRJ_EINVAL
    assert lib.srj_sha2_hash(160, C.byref(col), C.byref(col), None) == N.SRJ_EINVAL


def test_library_holds_the_sm90a_sha2_kernels():
    from srj_b200 import _native as N
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", N.LIB_PATH], capture_output=True, text=True).stdout
    funcs = [l for l in sass.splitlines() if "Function :" in l]
    for k in ("sha256_kernel", "sha512_kernel", "sha2_offsets_kernel", "sha2_word_popc_kernel"):
        assert any(k in f for f in funcs), f"kernel {k} missing from the cubin"
    assert "sm_90a" in subprocess.run([cuobjdump, "-lelf", N.LIB_PATH], capture_output=True, text=True).stdout
