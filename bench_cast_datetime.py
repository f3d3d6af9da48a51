#!/usr/bin/env python
"""bench_cast_datetime.py -- benchmark of CastStrings' string-to-timestamp and string-to-date parses on one GPU.

    python bench_cast_datetime.py [--workload NAME|all] [--steps K] [--warmup W]

Workloads (100M rows each, or as many as int32 offsets allow: width * rows < 2^31; strings resident in HBM, outputs
preallocated, no nulls).  Each draws its rows from a pool of 4096 strings; the rows of a workload are padded with trailing
spaces to its longest string, so offsets are i * width:
  ts_plain      yyyy-mm-dd hh:mm:ss.ffffff, years 1900-2100, the default zone
  ts_offset     the same with +hh:mm
  ts_region     the same with one of the 32 fixture zone names (6 to 19 bytes)
  ts_dirty      ts_plain with 1-3 leading spaces or tabs, and 10 % of rows damaged to invalid
  to_timestamp  ts_region parsed, then converted to UTC with one zone per row (parse + convertTimestampColumnToUTCWithTzCv)
  date          yyyy-mm-dd
A step is the C-ABI calls of one cast, timed with CUDA events.  Each workload is checked against oracle/cast_datetime.py on
a sample first.  The traffic model is the chars and offsets read plus 22 B/row written (parse), 4 B/row and the mask (date);
to_timestamp adds the convert's 22 B/row read and 8 B/row and mask written.  Prints one JSON line per workload with its
share of the H100 SXM data-sheet bandwidth, the card and its power limit read in the same run.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import random
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, os.path.join(ROOT, "spark-rapids-jni_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402

from bench import ClockSampler  # noqa: E402
from bench_sha2 import card_info  # noqa: E402

HBM_PEAK = 3.35e12          # H100 SXM data sheet, HBM3 (a card allowed 700 W)
ROWS = 100_000_000
POOL = 4096
NOW = 1_760_000_000
WORKLOADS = ["ts_plain", "ts_offset", "ts_region", "ts_dirty", "to_timestamp", "date"]


def pool(key, zones):
    rng = random.Random(7)
    out = []
    for _ in range(POOL):
        y, mo, d = rng.randint(1900, 2100), rng.randint(1, 12), rng.randint(1, 28)
        h, mi, s, us = rng.randint(0, 23), rng.randint(0, 59), rng.randint(0, 59), rng.randint(0, 999999)
        if key == "date":
            out.append(b"%04d-%02d-%02d" % (y, mo, d))
            continue
        t = b"%04d-%02d-%02d %02d:%02d:%02d.%06d" % (y, mo, d, h, mi, s, us)
        if key == "ts_offset":
            t += b"%+03d:%02d" % (rng.randint(-12, 14), rng.choice((0, 30, 45)))
        elif key in ("ts_region", "to_timestamp"):
            t += b" " + rng.choice(zones).encode()
        elif key == "ts_dirty":
            t = b"".join(rng.choice((b" ", b"\t")) for _ in range(rng.randint(1, 3))) + t
            if rng.random() < 0.1:
                i = rng.randrange(len(t))
                t = t[:i] + b"x" + t[i + 1:]
        out.append(t)
    return out


def run(args, key):
    import torch
    import srj_b200 as S
    from golden import timezone_golden as G
    from oracle import cast_datetime as OC
    from oracle import timezone as OT
    from srj_b200 import _native as N
    from srj_b200.timezone import TimeZoneTable
    torch.cuda.set_device(0)
    lib = N.lib()
    stream = torch.cuda.current_stream()
    st = int(stream.cuda_stream)
    strs = pool(key, G.ZONES)
    width = max(len(s) for s in strs)
    n = min(ROWS, (2**31 - 1) // width // 32 * 32)      # a STRING column holds at most 2^31 - 1 chars
    mat = torch.from_numpy(np.frombuffer(b"".join(s.ljust(width) for s in strs), np.uint8).reshape(POOL, width).copy()).cuda()
    g = torch.Generator(device="cuda").manual_seed(42)
    pick = torch.randint(0, POOL, (n,), device="cuda", generator=g)
    chars = mat[pick].reshape(-1)
    offsets = torch.arange(0, (n + 1) * width, width, device="cuda", dtype=torch.int64).to(torch.int32)
    col = S.ColumnVector(S.DType(S.DType.STRING), n, chars, None, offsets)
    cin = col._c()
    tzt = TimeZoneTable(G.ZONES, G.ENTRIES, G.RULES)
    otz = OT.Table(*tzt.arrays())
    info = tzt.to_device()
    cfix, cdst = info.getColumn(0)._c(), info.getColumn(1)._c()
    cmap = tzt.name_to_index_map()
    cm = cmap._c()
    names = sorted((k.encode(), v) for k, v in tzt.name_to_index().items())
    la = tzt.index("America/Los_Angeles")
    nulls = C.c_int64(0)
    if key == "date":
        out = torch.empty(n, dtype=torch.int32, device="cuda")
        mask = torch.empty((n + 31) // 32, dtype=torch.int32, device="cuda")

        def step():
            N.check(lib.srj_cast_parse_dates(C.byref(cin), out.data_ptr(), mask.data_ptr(), C.byref(nulls), st))

        def check(rows):
            got = out[rows].cpu().numpy()
            for r, v in zip(rows.tolist(), got):
                w = OC.parse_date(strs[int(pick[r])].ljust(width))
                assert w is not None and w == v, f"bench_cast_datetime {key}: row {r} differs from the oracle"
        bytes_alg = n * width + 4 * (n + 1) + 4 * n + n // 8
    else:
        outs = [torch.empty(n * w, dtype=torch.uint8, device="cuda") for w in (1, 8, 4, 1, 4, 4)]
        res = torch.empty(n, dtype=torch.int64, device="cuda")
        rmask = torch.empty((n + 31) // 32, dtype=torch.int32, device="cuda")
        kids = [S.ColumnVector(S.DType(t), n, o)._c() for t, o in
                zip((S.DType.UINT8, S.DType.INT64, S.DType.INT32, S.DType.UINT8, S.DType.INT32, S.DType.INT32), outs)]

        def parse():
            N.check(lib.srj_cast_parse_timestamps(C.byref(cin), C.byref(cm), C.byref(cfix), C.byref(cdst), la, 20000, NOW, 0, 3, 5, 0,
                                                  *[o.data_ptr() for o in outs], st))

        if key == "to_timestamp":
            def step():
                parse()
                N.check(lib.srj_timezone_convert_multi(C.byref(kids[1]), C.byref(kids[2]), C.byref(kids[0]), C.byref(kids[3]), C.byref(kids[4]),
                                                       C.byref(cfix), C.byref(cdst), C.byref(kids[5]), res.data_ptr(), rmask.data_ptr(),
                                                       C.byref(nulls), st))
            bytes_alg = n * width + 4 * (n + 1) + 22 * n + 22 * n + 8 * n + n // 8
        else:
            step = parse
            bytes_alg = n * width + 4 * (n + 1) + 22 * n

        def check(rows):
            h = [o.view(d)[rows].cpu().numpy() for o, d in zip(outs, (torch.uint8, torch.int64, torch.int32, torch.uint8, torch.int32, torch.int32))]
            for k, r in enumerate(rows.tolist()):
                w = OC.parse_timestamp(strs[int(pick[r])].ljust(width), la, 20000, names, otz, NOW, False, False)
                assert tuple(int(c[k]) for c in h) == w, f"bench_cast_datetime {key}: row {r} differs from the oracle"
    step()
    torch.cuda.synchronize()
    check(torch.from_numpy(np.unique(np.concatenate([np.random.default_rng(1).integers(0, n, 2000), np.arange(n - 100, n)]))).cuda())
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
    hbm_ms = bytes_alg / HBM_PEAK * 1e3
    print(json.dumps({
        "metric": f"rows_per_s_{key}", "value": n / (ms * 1e-3), "unit": "rows/s", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": ms, "ms_per_step_min": ms_min, "higher_is_better": True, "data": "synthetic",
        "config": {"workload": key, "rows": n, "width": width},
        "hbm_peak_frac": round(bytes_alg / (ms * 1e-3) / HBM_PEAK, 4),
        "models": {"note": "models, not measurements", "hbm": {"bytes": bytes_alg, "bound_ms": hbm_ms, "achieved_frac": round(hbm_ms / ms, 4)}},
        "card": card_info(), "clocks": clocks}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="all", choices=WORKLOADS + ["all"])
    ap.add_argument("--gpus", type=int, default=1, choices=[1])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be at least 1")
    for key in (WORKLOADS if args.workload == "all" else [args.workload]):
        run(args, key)


if __name__ == "__main__":
    main()
