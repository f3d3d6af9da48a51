#!/usr/bin/env python
"""bench_iceberg.py -- benchmark of Iceberg's partition transforms (bucket, truncate, hour) on one GPU.

    python bench_iceberg.py [--workload bucket_long|bucket_string|bucket_decimal|truncate_long|truncate_string|hours]
                            [--steps K] [--warmup W] [--dump-outputs DIR]

Workloads:
  bucket_long      bucket[16] of 100M INT64, 10% nulls
  bucket_string    bucket[1024] of 16M mixed UTF-8 strings of 4-40 bytes, 10% nulls
  bucket_decimal   bucket[16] of 50M DECIMAL128(38, 2)
  truncate_long    truncate[1000] of 100M INT64
  truncate_string  truncate[4] of 16M mixed UTF-8 strings of 4-40 bytes (sizes, scan, read-back, prefix copy)
  hours            hour of 100M TIMESTAMP_MICROSECONDS
A step is the C-ABI call(s) of one transform (truncate_string: srj_iceberg_truncate_sizes, which synchronises once, then
srj_iceberg_truncate), inputs resident in HBM, outputs preallocated, CUDA events around each step.  Prints one JSON line:
rows/s, the HBM model (algorithmic bytes moved) and its share of the H100 SXM data-sheet bandwidth, the card and its
power limit read in the same run, the SM clock sampled during the run, and a one-core numpy-oracle baseline on a sample.
--dump-outputs DIR writes a seeded sample of the output plus whole-output checksums (float .npy files).  Shares its
measurement helpers with bench.py.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, os.path.join(ROOT, "spark-rapids-jni_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402

from bench import ClockSampler, byte_sum, sample_rows, write_dump  # noqa: E402
from bench_sha2 import card_info  # noqa: E402

HBM_PEAK = 3.35e12          # H100 SXM data sheet, HBM3 (a card allowed 700 W)
INT64, MICROS, STRING, DECIMAL128 = 4, 15, 23, 27
WORKLOADS = {
    "bucket_long": dict(name="bucket[16], 100M INT64, 10% nulls", kind="bucket", type_id=INT64, rows=100_000_000, n=16, nulls=0.10),
    "bucket_string": dict(name="bucket[1024], 16M UTF-8 strings of 4-40 bytes, 10% nulls", kind="bucket", type_id=STRING,
                          rows=16_000_000, n=1024, nulls=0.10),
    "bucket_decimal": dict(name="bucket[16], 50M DECIMAL128(38, 2)", kind="bucket", type_id=DECIMAL128, rows=50_000_000, n=16,
                           nulls=None),
    "truncate_long": dict(name="truncate[1000], 100M INT64", kind="truncate", type_id=INT64, rows=100_000_000, n=1000, nulls=None),
    "truncate_string": dict(name="truncate[4], 16M UTF-8 strings of 4-40 bytes", kind="truncate", type_id=STRING, rows=16_000_000,
                            n=4, nulls=None),
    "hours": dict(name="hour, 100M TIMESTAMP_MICROSECONDS", kind="hours", type_id=MICROS, rows=100_000_000, n=0, nulls=None),
}
UTF8_CHARS = ["a", "b", "Z", "0", " ", "é", "ж", "€", "中", "😀"]


def _mask(torch, g, n, frac):
    valid = torch.rand(n + (-n % 32), device="cuda", generator=g) >= frac
    w = (valid.view(-1, 32).to(torch.int64) << torch.arange(32, device="cuda", dtype=torch.int64)).sum(1)
    return torch.where(w >= 2**31, w - 2**32, w).to(torch.int32)


def make_input(torch, S, wl, g):
    n, t = wl["rows"], wl["type_id"]
    mask = _mask(torch, g, n, wl["nulls"]) if wl["nulls"] else None
    if t == STRING:
        rng = np.random.default_rng(42)
        pool = torch.from_numpy(np.frombuffer("".join(rng.choice(UTF8_CHARS, 1 << 20)).encode(), np.uint8).copy()).cuda()
        lens = torch.randint(4, 41, (n,), device="cuda", generator=g, dtype=torch.int64)
        offs = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
        offs[1:] = torch.cumsum(lens, 0)
        total = int(offs[-1])
        reps = (total + pool.numel() - 1) // pool.numel()
        chars = pool.repeat(reps)[:total].contiguous()
        return S.ColumnVector(S.DType.STRING, n, chars, mask, offs.to(torch.int32))
    width = {INT64: 8, MICROS: 8, DECIMAL128: 16}[t]
    data = torch.randint(0, 256, (n * width,), dtype=torch.uint8, device="cuda", generator=g).view(torch.int64)
    if t == DECIMAL128:                  # DECIMAL(38, 2): |unscaled| < 10^38, here spread over every byte length
        d = data.view(-1, 2)
        d[:, 1] >>= torch.randint(0, 64, (n,), device="cuda", generator=g)
        d[:, 0] = torch.where(d[:, 1] == 0, d[:, 0] >> 32, d[:, 0])
    if t == MICROS:                      # timestamps within +-290 000 years of the epoch
        data >>= 4
    return S.ColumnVector(S.DType(t, -2 if t == DECIMAL128 else 0), n, data.view(torch.uint8), mask)


def host_slice(col, s, e):
    """(data, mask, offsets) of rows [s, e) on the host (s a multiple of 32)"""
    mask = None if col.mask is None else col.mask[s // 32:(e + 31) // 32].cpu().numpy().view(np.uint32)
    if col.dtype.type_id == STRING:
        offs = col.offsets[s:e + 1].cpu().numpy().astype(np.int64)
        data = col.data[int(offs[0]):int(offs[-1])].cpu().numpy()
        return data, mask, (offs - offs[0]).astype(np.int32)
    w = col.dtype.size_in_bytes()
    return col.data[s * w:e * w].cpu().numpy(), mask, None


def oracle(wl, data, mask, offs, rows):
    from oracle import iceberg as O
    if wl["kind"] == "bucket":
        return O.bucket(wl["type_id"], data, mask, rows, wl["n"], offs)
    if wl["kind"] == "hours":
        return O.datetime_transform("hours", MICROS, data, rows)
    if wl["type_id"] == STRING:
        return O.truncate_bytes(STRING, data, offs, mask, rows, wl["n"])
    return O.truncate_integral(wl["type_id"], data, mask, rows, wl["n"])


def cpu_baseline(wl, col, n_sample):
    """oracle/iceberg.py (numpy, one core) on a sample of the same work"""
    args = host_slice(col, 0, n_sample)
    fn = lambda: oracle(wl, *args, n_sample)       # noqa: E731
    fn()
    times = []
    while sum(times) < 5.0 and len(times) < 5:
        t0 = time.perf_counter()
        fn()
        times.append(time.perf_counter() - t0)
    best = min(times)
    return {"value": n_sample / best, "unit": "rows/s", "cores": 1, "kind": "numpy oracle (oracle/iceberg.py)",
            "sample": f"{n_sample} rows, best of {len(times)} passes"}


def run(args, wl_key):
    import torch
    import srj_b200 as S
    from srj_b200 import _native as N
    torch.cuda.set_device(0)
    wl = WORKLOADS[wl_key]
    lib = N.lib()
    stream = torch.cuda.current_stream()
    st = int(stream.cuda_stream)
    g = torch.Generator(device="cuda").manual_seed(42)
    n, t = wl["rows"], wl["type_id"]
    col = make_input(torch, S, wl, g)
    cin = col._c()
    mask_bytes = 4 * ((n + 31) // 32) if col.mask is not None else 0
    out_mask = torch.empty((n + 31) // 32, dtype=torch.int32, device="cuda") if col.mask is not None else None
    mptr = out_mask.data_ptr() if out_mask is not None else None
    in_bytes = col.data.numel() + (4 * (n + 1) if col.offsets is not None else 0) + mask_bytes
    res = {}
    if wl["kind"] == "bucket" or wl["kind"] == "hours":
        out = torch.empty(n, dtype=torch.int32, device="cuda")
        if wl["kind"] == "bucket":
            def step():
                N.check(lib.srj_iceberg_bucket(C.byref(cin), wl["n"], out.data_ptr(), mptr, st))
        else:
            def step():
                N.check(lib.srj_iceberg_datetime(3, C.byref(cin), out.data_ptr(), mptr, st))
        bytes_alg = in_bytes + 4 * n + 2 * mask_bytes        # the mask is read again and copied
        res["out"] = out
    elif t != STRING:
        out = torch.empty(n * 8, dtype=torch.uint8, device="cuda")
        cout = S.ColumnVector(S.DType(t), n, out, out_mask)._c()

        def step():
            N.check(lib.srj_iceberg_truncate(C.byref(cin), wl["n"], C.byref(cout), st))
        bytes_alg = in_bytes + 8 * n + 2 * mask_bytes
        res["out"] = out
    else:
        offs = torch.empty(n + 1, dtype=torch.int32, device="cuda")
        ws = torch.empty(lib.srj_iceberg_truncate_workspace_bytes(n), dtype=torch.uint8, device="cuda")
        total = C.c_int64(0)
        N.check(lib.srj_iceberg_truncate_sizes(C.byref(cin), wl["n"], offs.data_ptr(), C.byref(total), ws.data_ptr(), st))
        out = torch.empty(total.value, dtype=torch.uint8, device="cuda")
        cout = S.ColumnVector(S.DType.STRING, n, out, out_mask, offs)._c()

        def step():
            N.check(lib.srj_iceberg_truncate_sizes(C.byref(cin), wl["n"], offs.data_ptr(), C.byref(total), ws.data_ptr(), st))
            N.check(lib.srj_iceberg_truncate(C.byref(cin), wl["n"], C.byref(cout), st))
        # sizes: offsets in (+ the bytes of rows longer than the width: about 4 words of each), sizes out; scan: 2 passes
        # over the offsets; copy: both offsets in, prefix bytes in and out
        bytes_alg = 4 * (n + 1) * 6 + 16 * n + 2 * total.value
        res["offsets"], res["out"] = offs, out

    # correctness gate against the oracle before timing, on the first rows and on a 32-row-aligned slice in the middle
    step()
    torch.cuda.synchronize()
    n_check = min(n, 250_000)
    for s in (0, (n // 2) & ~31):
        e = min(n, s + n_check)
        want = oracle(wl, *host_slice(col, s, e), e - s)
        if wl["kind"] == "truncate" and t == STRING:
            o = offs[s:e + 1].cpu().numpy().astype(np.int64)
            assert np.array_equal(o - o[0], want[0]), "bench_iceberg: offsets differ from the oracle"
            assert np.array_equal(out[int(o[0]):int(o[-1])].cpu().numpy(), want[1]), "bench_iceberg: bytes differ from the oracle"
        elif wl["kind"] == "truncate":
            assert np.array_equal(out[s * 8:e * 8].cpu().numpy(), want), "bench_iceberg: values differ from the oracle"
        else:
            assert np.array_equal(out[s:e].cpu().numpy(), want), "bench_iceberg: values differ from the oracle"

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    sampler = ClockSampler(0)
    sampler.start()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
    for a, b in evs:
        a.record(stream)
        step()
        b.record(stream)
    torch.cuda.synchronize()
    clocks = sampler.stop()
    ms = float(np.mean([a.elapsed_time(b) for a, b in evs]))
    ms_min = float(np.min([a.elapsed_time(b) for a, b in evs]))
    if args.dump_outputs:
        arrays = {}
        for name, tsr in res.items():
            b = tsr.view(torch.uint8)
            idx_np = sample_rows(b.numel())
            arrays[f"{name}_sample_rows"] = idx_np.astype(np.float64)
            arrays[f"{name}_sample_bytes"] = b[torch.from_numpy(idx_np).cuda()].cpu().numpy().astype(np.float64)
            arrays[f"{name}_byte_sum"] = np.array([byte_sum(torch, b)])
        write_dump(args.dump_outputs, arrays)
    card = card_info()
    sec = ms * 1e-3
    hbm_ms = bytes_alg / HBM_PEAK * 1e3
    print(json.dumps({
        "metric": f"rows_per_s_{wl_key}", "value": n / sec, "unit": "rows/s", "n_gpus": 1, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": ms, "ms_per_step_min": ms_min, "higher_is_better": True, "data": "synthetic",
        "config": {"workload": wl["name"], "rows": n},
        "algorithmic_bytes_per_sec": bytes_alg / sec, "hbm_peak_frac": round(bytes_alg / sec / HBM_PEAK, 4),
        "models": {"note": "models, not measurements", "hbm": {"bytes": bytes_alg, "bound_ms": hbm_ms, "achieved_frac": round(hbm_ms / ms, 4)}},
        "card": card, "cpu_baseline": cpu_baseline(wl, col, min(n, 1_000_000)), "clocks": clocks}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="bucket_long", choices=sorted(WORKLOADS))
    ap.add_argument("--gpus", type=int, default=1, choices=[1])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write a seeded sample of the output plus checksums as DIR/<name>.npy")
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be at least 1")
    run(args, args.workload)


if __name__ == "__main__":
    main()
