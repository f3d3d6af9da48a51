"""Builds libsrj_b200.so (hand-written sm_90a CUDA + the C ABI) in-tree with nvcc.

    python spark-rapids-jni_b200/build.py [--force] [--verbose]

The .so lands next to the python package (spark-rapids-jni_b200/srj_b200/libsrj_b200.so) so it
travels with the repo snapshot to the GPU box; it is git-ignored.
"""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "srj_b200", "libsrj_b200.so")
SOURCES = ["capi.cu", "from_rows.cu", "from_rows_wide.cu", "to_rows.cu", "to_rows_var.cu", "strings.cu", "hash.cu", "hash_nested.cu", "sharding.cu", "partition.cu", "unsafe_row.cu", "kudo.cu", "host_api.cu", "sha2.cu", "bloom_filter.cu", "zorder.cu", "iceberg.cu", "decimal.cu", "datetime.cu", "join.cu", "timezone.cu", "cast_datetime.cu", "histogram.cu", "arithmetic.cu", "float_to_decimal.cu", "radix.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "--shared", "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "-ccbin", "/usr/bin/g++",
    "--expt-relaxed-constexpr", "-Xptxas", "-v" if os.environ.get("SRJ_PTXAS_V") else "-O3",
]


def needs_build() -> bool:
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "srj_b200.h"),
                                                                 os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return OUT
    objs = []
    procs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    for src in SOURCES:
        obj = os.path.join(HERE, "build", src.replace(".cu", ".o"))
        cmd = [NVCC] + [f for f in FLAGS if f != "--shared"] + ["-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            print(" ".join(cmd))
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or verbose or os.environ.get("SRJ_PTXAS_V"):
            sys.stderr.write(f"--- {src}\n{out}\n")
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed")
    cmd = [NVCC, "--shared", "-gencode", "arch=compute_90a,code=sm_90a", "-ccbin", "/usr/bin/g++", "-Xlinker", "--no-undefined", "-o", OUT] + objs
    subprocess.check_call(cmd)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
