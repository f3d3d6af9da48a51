"""JoinPrimitives on one GPU: the hash inner join and the gather-map helpers, timed with CUDA events after a warm-up.

    python bench_join.py [--steps K] [--warmup W] [--only NAME ...] [--dump-outputs DIR]

Workloads (the shapes of a Spark fact-to-dimension join and its outer / semi / anti forms):
  fact_dim     100 M INT64 probe keys against 10 M unique build keys, half of the probes hit; the 256 MB table is beyond L2
  small_build  the same probe against 1 M build keys: a 32 MB table that fits in the 50 MB L2
  multi_key    INT32 (10 % nulls) + INT64 keys, 20 M probes against 2 M unique build rows, nulls unequal and equal
  string_key   16 M probe strings of 4 to 40 bytes against 2 M build strings
  dup          1 M probe rows against 10 M build rows, 100 build rows per key: about 100 M output pairs (write bound)
  full_outer / semi / anti on 100 M-entry maps over 100 M-row tables
Each prints one JSON line: the time, and a lower-bound HBM traffic model computed from the shapes (a streamed key read,
one random 32-byte sector per probe, a key gather per hash-equal candidate, 8 bytes written per pair).  The card's name
and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [ROOT, os.path.join(ROOT, "spark-rapids-jni_b200")]

import srj_b200 as S                                   # noqa: E402
from srj_b200.join import GatherMap, JoinPrimitives    # noqa: E402

HBM = 3.35e12


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:        # noqa: BLE001
        return f"unknown ({e})"


def col(t, values, valid=None):
    mask = None
    if valid is not None:
        bits = torch.zeros(((len(valid) + 31) // 32) * 32, dtype=torch.bool, device="cuda")
        bits[:len(valid)] = valid
        w = (bits.view(-1, 32).to(torch.int64) << torch.arange(32, device="cuda")).sum(1)
        mask = (w - ((w >> 31) & 1) * (1 << 32)).to(torch.int32)         # the uint32 words as int32
    return S.ColumnVector(S.DType(t), values.numel(), values.contiguous().view(torch.uint8), mask)


def strings(n, lo, hi, pool, gen):
    ids = torch.randint(0, pool, (n,), device="cuda", generator=gen)
    lens = lo + ids % (hi - lo + 1)
    offs = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    offs[1:] = torch.cumsum(lens, 0)
    pos = torch.arange(int(offs[-1]), device="cuda") - torch.repeat_interleave(offs[:-1], lens)
    rid = torch.repeat_interleave(ids, lens)
    chars = torch.where(pos < 4, (rid >> (8 * pos.clamp(max=3))) & 255, (rid * 2654435761 + pos * 40503) % 251).to(torch.uint8)  # id in bytes 0-3
    return S.ColumnVector(S.DType(23), n, chars, None, offs.to(torch.int32)), int(offs[-1])


def timed(fn, steps, warmup):
    for _ in range(warmup):
        out = fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(steps):
        out = fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / steps, out


def workloads(gen):
    def fact_dim(nb):
        build = torch.randperm(nb, device="cuda", generator=gen).to(torch.int64) * 2
        probe = torch.randint(0, 2 * nb, (100_000_000,), device="cuda", generator=gen)   # half are even: a hit
        l, r = S.Table([col(4, probe)]), S.Table([col(4, build)])
        pairs = 50_000_000
        model = probe.numel() * (8 + 32) + pairs * (8 + 8) + nb * (8 + 2 * 32)
        return (lambda: JoinPrimitives.hashInnerJoin(l, r, False)), model
    yield "fact_dim", lambda: fact_dim(10_000_000)
    yield "small_build", lambda: fact_dim(1_000_000)

    def multi_key(eq):
        nb, npr = 2_000_000, 20_000_000
        bk = torch.randperm(nb, device="cuda", generator=gen)
        pk = torch.randint(0, 2 * nb, (npr,), device="cuda", generator=gen)
        # 10 % nulls in the INT32 column only, so that the INT64 column keeps each probe to at most one match in both modes
        bv, pv = torch.rand(nb, device="cuda", generator=gen) >= 0.1, torch.rand(npr, device="cuda", generator=gen) >= 0.1
        l = S.Table([col(3, pk.to(torch.int32), pv), col(4, pk * 3)])
        r = S.Table([col(3, bk.to(torch.int32), bv), col(4, bk * 3)])
        return (lambda: JoinPrimitives.hashInnerJoin(l, r, eq)), npr * (12 + 32 + 12) + nb * (12 + 64)
    yield "multi_key_nulls_unequal", lambda: multi_key(False)
    yield "multi_key_nulls_equal", lambda: multi_key(True)

    def string_key():
        lc, lb = strings(16_000_000, 4, 40, 4_000_000, gen)
        rc, rb = strings(2_000_000, 4, 40, 2_000_000, gen)
        l, r = S.Table([lc]), S.Table([rc])
        return (lambda: JoinPrimitives.hashInnerJoin(l, r, False)), lb + 8 * 16_000_000 + 16_000_000 * 32 + rb + 8 * 2_000_000
    yield "string_key", string_key

    def dup():
        build = torch.arange(10_000_000, device="cuda", dtype=torch.int64) // 100
        probe = torch.randint(0, 100_000, (1_000_000,), device="cuda", generator=gen)
        l, r = S.Table([col(4, probe)]), S.Table([col(4, build)])
        return (lambda: JoinPrimitives.hashInnerJoin(l, r, False)), 100_000_000 * 8 * 2 + 100_000_000 * 8
    yield "dup", dup

    def helper(kind):
        n = 100_000_000
        lm = GatherMap(torch.randint(0, n, (n,), device="cuda", generator=gen, dtype=torch.int32))
        rm = GatherMap(torch.randint(0, n, (n,), device="cuda", generator=gen, dtype=torch.int32))
        if kind == "full_outer":
            return (lambda: JoinPrimitives.makeFullOuter(lm, rm, n, n)), n * 4 * 2 * 3 + n // 8 * 4
        if kind == "semi":
            return (lambda: JoinPrimitives.makeSemi(lm, n)), n * 4 + n * 4 * 0.64 + n // 8 * 2
        return (lambda: JoinPrimitives.makeAnti(lm, n)), n * 4 + n * 4 * 0.37 + n // 8 * 2
    for k in ("full_outer", "semi", "anti"):
        yield k, (lambda k=k: helper(k))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--only", nargs="*")
    ap.add_argument("--dump-outputs", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_join.py needs a GPU")
    name = card()
    gen = torch.Generator("cuda").manual_seed(1234)
    for wl, make in workloads(gen):
        if a.only and wl not in a.only:
            continue
        fn, model = make()
        ms, out = timed(fn, a.steps, a.warmup)
        maps = out if isinstance(out, list) else [out]
        rec = {"workload": wl, "ms": round(ms, 3), "model_bytes": int(model), "model_floor_ms": round(model / HBM * 1e3, 3),
               "pairs": maps[0].getRowCount(), "card": name}
        print(json.dumps(rec), flush=True)
        if a.dump_outputs:
            os.makedirs(a.dump_outputs, exist_ok=True)
            for i, m in enumerate(maps):
                np.save(os.path.join(a.dump_outputs, f"{wl}_{i}.npy"), m.data.cpu().numpy())
        del fn, out, maps
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
