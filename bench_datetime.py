#!/usr/bin/env python
"""bench_datetime.py -- benchmark of DateTimeUtils' rebase and truncation on one GPU.

    python bench_datetime.py [--workload rebase_days|rebase_micros|trunc_month|trunc_column]
                             [--direction g2j|j2g] [--steps K] [--warmup W] [--dump-outputs DIR]

Workloads:
  rebase_days    rebase of 100M TIMESTAMP_DAYS spread over years 1000-2100, 10% nulls (--direction)
  rebase_micros  the same for 100M TIMESTAMP_MICROSECONDS
  trunc_month    truncate(ts, "MONTH") of 100M TIMESTAMP_MICROSECONDS over years 1000-2100, 10% nulls
  trunc_column   truncate(ts, fmt) of 16M TIMESTAMP_MICROSECONDS with a STRING format column cycling through the 15 formats
                 in mixed case, 5% of the rows an invalid format (one stream synchronisation: the null count read-back)
A step is one C-ABI call, inputs resident in HBM, outputs preallocated, CUDA events around each step.  Prints one JSON
line: rows/s, the HBM model (algorithmic bytes moved) and its share of the H100 SXM data-sheet bandwidth, the card and its
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
from bench_iceberg import _mask  # noqa: E402
from bench_sha2 import card_info  # noqa: E402

HBM_PEAK = 3.35e12          # H100 SXM data sheet, HBM3 (a card allowed 700 W)
DAYS, MICROS = 12, 15
DAY_LO, DAY_HI = -354285, 47482          # 1000-01-01 .. 2100-01-01
US = 86_400_000_000
FORMATS = ["YEAR", "YYYY", "YY", "QUARTER", "MONTH", "MM", "MON", "WEEK", "DAY", "DD", "HOUR", "MINUTE", "SECOND", "MILLISECOND",
           "MICROSECOND"]
WORKLOADS = {
    "rebase_days": dict(name="rebase, 100M TIMESTAMP_DAYS (years 1000-2100), 10% nulls", type_id=DAYS, rows=100_000_000, nulls=0.10),
    "rebase_micros": dict(name="rebase, 100M TIMESTAMP_MICROSECONDS (years 1000-2100), 10% nulls", type_id=MICROS, rows=100_000_000,
                          nulls=0.10),
    "trunc_month": dict(name="truncate MONTH, 100M TIMESTAMP_MICROSECONDS, 10% nulls", type_id=MICROS, rows=100_000_000, nulls=0.10),
    "trunc_column": dict(name="truncate, 16M TIMESTAMP_MICROSECONDS, a format column of 15 formats in mixed case, 5% invalid",
                         type_id=MICROS, rows=16_000_000, nulls=None),
}


def make_formats(n):
    """(chars uint8, offsets int32, format strings of the pool, pool index per row): the 15 names in upper, lower and
    alternating case, and invalid names on 5% of the rows"""
    pool = [f for n_ in FORMATS for f in (n_, n_.lower(), "".join(c.lower() if j % 2 else c for j, c in enumerate(n_)))]
    bad = ["YEARS", "hours", "", "Sec"]
    rng = np.random.default_rng(5)
    idx = rng.integers(0, len(pool), n)
    inv = rng.random(n) < 0.05
    idx[inv] = len(pool) + rng.integers(0, len(bad), int(inv.sum()))
    pool = pool + bad
    bs = [p.encode() for p in pool]
    mat = np.zeros((len(pool), 12), np.uint8)
    for i, b in enumerate(bs):
        mat[i, :len(b)] = np.frombuffer(b, np.uint8)
    lens = np.array([len(b) for b in bs], np.int64)[idx]
    offs = np.zeros(n + 1, np.int32)
    offs[1:] = np.cumsum(lens)
    return mat[idx][np.arange(12)[None, :] < lens[:, None]], offs, pool, idx


def oracle(wl_key, direction, data, mask, rows, fmts=None):
    from oracle import datetime as O
    t = WORKLOADS[wl_key]["type_id"]
    if wl_key.startswith("rebase"):
        return O.rebase(direction, t, data)
    valid = None if mask is None else np.unpackbits(mask.view(np.uint8), bitorder="little")[:rows].astype(bool)
    if wl_key == "trunc_month":
        return O.truncate_scalar(t, data, valid, "MONTH")[0]
    return O.truncate_column(t, data, valid, fmts)[0]


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
    w = 4 if t == DAYS else 8
    direction = 0 if args.direction == "g2j" else 1
    days = torch.randint(DAY_LO, DAY_HI, (n,), device="cuda", generator=g, dtype=torch.int64)
    if t == DAYS:
        data = days.to(torch.int32)
    else:
        data = days * US + torch.randint(0, US, (n,), device="cuda", generator=g, dtype=torch.int64)
    mask = _mask(torch, g, n, wl["nulls"]) if wl["nulls"] else None
    col = S.ColumnVector(S.DType(t), n, data.view(torch.uint8), mask)
    cin = col._c()
    mask_bytes = 4 * ((n + 31) // 32)
    out = torch.empty(n * w, dtype=torch.uint8, device="cuda")
    out_mask = torch.empty((n + 31) // 32, dtype=torch.int32, device="cuda")
    nulls = C.c_int64(0)
    fmts = None
    if wl_key.startswith("rebase"):
        def step():
            N.check(lib.srj_datetime_rebase(direction, C.byref(cin), out.data_ptr(), out_mask.data_ptr(), st))
        bytes_alg = 2 * n * w + 2 * mask_bytes                                  # values in and out, the mask copied
    elif wl_key == "trunc_month":
        def step():
            N.check(lib.srj_datetime_truncate(C.byref(cin), None, b"MONTH", 5, out.data_ptr(), out_mask.data_ptr(), C.byref(nulls), st))
        bytes_alg = 2 * n * w + 3 * mask_bytes                                  # + the mask read by the kernel
    else:
        chars, offs, pool, idx = make_formats(n)
        fcol = S.ColumnVector.from_numpy(S.DType.STRING, chars, None, offs)
        cfmt = fcol._c()
        fmts = pool, idx

        def step():
            N.check(lib.srj_datetime_truncate(C.byref(cin), C.byref(cfmt), None, 0, out.data_ptr(), out_mask.data_ptr(), C.byref(nulls), st))
        bytes_alg = 2 * n * w + 4 * (n + 1) + len(chars) + mask_bytes           # values, offsets, format bytes, mask out

    # correctness gate against the oracle before timing, on the first rows and on a 32-row-aligned slice in the middle
    step()
    torch.cuda.synchronize()
    n_check = min(n, 250_000)
    for s in (0, (n // 2) & ~31):
        e = min(n, s + n_check)
        h = data[s:e].cpu().numpy()
        hm = None if mask is None else mask[s // 32:(e + 31) // 32].cpu().numpy().view(np.uint32)
        f = None if fmts is None else [fmts[0][i] for i in fmts[1][s:e]]
        want = oracle(wl_key, direction, h, hm, e - s, f)
        got = out[s * w:e * w].cpu().numpy().view(np.int32 if t == DAYS else np.int64)
        assert np.array_equal(got, want), "bench_datetime: values differ from the oracle"

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
        for name, tsr in (("out", out), ("out_mask", out_mask)):
            b = tsr.view(torch.uint8)
            idx_np = sample_rows(b.numel())
            arrays[f"{name}_sample_rows"] = idx_np.astype(np.float64)
            arrays[f"{name}_sample_bytes"] = b[torch.from_numpy(idx_np).cuda()].cpu().numpy().astype(np.float64)
            arrays[f"{name}_byte_sum"] = np.array([byte_sum(torch, b)])
        write_dump(args.dump_outputs, arrays)
    card = card_info()
    sec = ms * 1e-3
    hbm_ms = bytes_alg / HBM_PEAK * 1e3

    # one-core numpy oracle on a sample of the same work
    n_sample = min(n, 1_000_000)
    h = data[:n_sample].cpu().numpy()
    hm = None if mask is None else mask[:(n_sample + 31) // 32].cpu().numpy().view(np.uint32)
    f = None if fmts is None else [fmts[0][i] for i in fmts[1][:n_sample]]
    times = []
    while sum(times) < 5.0 and len(times) < 5:
        t0 = time.perf_counter()
        oracle(wl_key, direction, h, hm, n_sample, f)
        times.append(time.perf_counter() - t0)
    cpu = {"value": n_sample / min(times), "unit": "rows/s", "cores": 1, "kind": "numpy oracle (oracle/datetime.py)",
           "sample": f"{n_sample} rows, best of {len(times)} passes"}
    config = {"workload": wl["name"], "rows": n}
    if wl_key.startswith("rebase"):
        config["direction"] = args.direction
    print(json.dumps({
        "metric": f"rows_per_s_{wl_key}", "value": n / sec, "unit": "rows/s", "n_gpus": 1, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": ms, "ms_per_step_min": ms_min, "higher_is_better": True, "data": "synthetic",
        "config": config, "algorithmic_bytes_per_sec": bytes_alg / sec, "hbm_peak_frac": round(bytes_alg / sec / HBM_PEAK, 4),
        "models": {"note": "models, not measurements", "hbm": {"bytes": bytes_alg, "bound_ms": hbm_ms, "achieved_frac": round(hbm_ms / ms, 4)}},
        "card": card, "cpu_baseline": cpu, "clocks": clocks}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="rebase_days", choices=sorted(WORKLOADS))
    ap.add_argument("--direction", default="g2j", choices=["g2j", "j2g"])
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
