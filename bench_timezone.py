#!/usr/bin/env python
"""bench_timezone.py -- benchmark of GpuTimeZoneDB's conversions on one GPU.

    python bench_timezone.py [--workload NAME|all] [--steps K] [--warmup W]

Workloads (100M rows each, inputs resident in HBM, outputs preallocated, no nulls):
  to_utc_1900_2100 / from_utc_1900_2100  America/Los_Angeles, TIMESTAMP_MICROSECONDS over years 1900-2100 (its transition
                                         table up to 2037, its DST rules after)
  to_utc_2000_2030 / from_utc_2000_2030  the same over 2000-2030
  fixed                                  to UTC in Etc/GMT+5 (one fixed entry)
  with_tz_cv                             one zone per row over the 32 fixture zones, 5% fixed offsets, 2% invalid rows
                                         (seconds, micros, 3 byte columns' worth of inputs; one stream synchronisation)
  orc                                    ORC writer Asia/Shanghai -> reader Asia/Kolkata
A step is one C-ABI call, timed with CUDA events.  Each workload is checked against the numpy oracle on a sample first.
Prints one JSON line per workload: rows/s, the HBM model (bytes in and out) and its share of the H100 SXM data-sheet
bandwidth, the card and its power limit read in the same run, and the SM clock sampled during the run.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, os.path.join(ROOT, "spark-rapids-jni_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402

from bench import ClockSampler  # noqa: E402
from bench_sha2 import card_info  # noqa: E402

HBM_PEAK = 3.35e12          # H100 SXM data sheet, HBM3 (a card allowed 700 W)
MICROS = 15
Y1900, Y2000, Y2030, Y2100 = -2208988800, 946684800, 1893456000, 4102444800
WORKLOADS = {
    "to_utc_1900_2100": dict(kind="convert", direction=0, zone="America/Los_Angeles", span=(Y1900, Y2100)),
    "from_utc_1900_2100": dict(kind="convert", direction=1, zone="America/Los_Angeles", span=(Y1900, Y2100)),
    "to_utc_2000_2030": dict(kind="convert", direction=0, zone="America/Los_Angeles", span=(Y2000, Y2030)),
    "from_utc_2000_2030": dict(kind="convert", direction=1, zone="America/Los_Angeles", span=(Y2000, Y2030)),
    "fixed": dict(kind="convert", direction=0, zone="Etc/GMT+5", span=(Y1900, Y2100)),
    "with_tz_cv": dict(kind="multi", span=(Y1900, Y2100)),
    "orc": dict(kind="orc", writer="Asia/Shanghai", reader="Asia/Kolkata", span=(Y1900, Y2100)),
}
ROWS = 100_000_000


def run(args, key):
    import torch
    import srj_b200 as S
    from golden import timezone_golden as G
    from oracle import timezone as OT
    from srj_b200 import _native as N
    from srj_b200.timezone import TimeZoneTable
    torch.cuda.set_device(0)
    wl = WORKLOADS[key]
    lib = N.lib()
    stream = torch.cuda.current_stream()
    st = int(stream.cuda_stream)
    g = torch.Generator(device="cuda").manual_seed(42)
    n = ROWS
    lo, hi = wl["span"]
    data = torch.randint(lo * 10**6, hi * 10**6, (n,), device="cuda", generator=g, dtype=torch.int64)
    tzt = TimeZoneTable(G.ZONES, G.ENTRIES, G.RULES)
    otz = OT.Table(*tzt.arrays())
    info = tzt.to_device()
    cfix, cdst = info.getColumn(0)._c(), info.getColumn(1)._c()
    out = torch.empty(n, dtype=torch.int64, device="cuda")
    out_mask = torch.empty((n + 31) // 32, dtype=torch.int32, device="cuda")
    col = S.ColumnVector(S.DType(MICROS), n, data.view(torch.uint8))
    cin = col._c()
    if wl["kind"] == "convert":
        zone = tzt.index(wl["zone"])

        def step():
            N.check(lib.srj_timezone_convert(wl["direction"], C.byref(cin), C.byref(cfix), C.byref(cdst), zone, out.data_ptr(), None, st))

        def want(idx):
            return OT.convert(wl["direction"], MICROS, data[idx].cpu().numpy(), otz, zone)
        bytes_alg = 16 * n
    elif wl["kind"] == "multi":
        sec = torch.div(data, 10**6, rounding_mode="floor")
        us = (data - sec * 10**6).to(torch.int32)
        r = torch.rand(n, device="cuda", generator=g)
        invalid = (r < 0.02).to(torch.uint8)
        ttype = ((r >= 0.02) & (r < 0.07)).to(torch.uint8)
        toff = torch.randint(-43200, 43200, (n,), device="cuda", generator=g, dtype=torch.int32)
        idx = torch.randint(0, len(G.ZONES), (n,), device="cuda", generator=g, dtype=torch.int32)
        host_cols = []
        cs = []
        for tid, tsr in ((S.DType.INT64, sec), (S.DType.INT32, us), (S.DType.UINT8, invalid), (S.DType.UINT8, ttype), (S.DType.INT32, toff),
                         (S.DType.INT32, idx)):
            host_cols.append(tsr)
            cs.append(S.ColumnVector(S.DType(tid), n, tsr.contiguous().view(torch.uint8))._c())
        nulls = C.c_int64(0)

        def step():
            N.check(lib.srj_timezone_convert_multi(*[C.byref(c) for c in cs[:5]], C.byref(cfix), C.byref(cdst), C.byref(cs[5]), out.data_ptr(),
                                                   out_mask.data_ptr(), C.byref(nulls), st))

        def want(i):
            h = [t[i].cpu().numpy() for t in host_cols]
            return OT.convert_multi(h[0], h[1], h[2].astype(bool), h[3], h[4], otz, h[5])[0]
        bytes_alg = n * (8 + 4 + 1 + 1 + 4 + 4 + 8) + n // 8                     # inputs, the value, the mask
    else:
        def table(name):
            raw, tr, of = G.ORC[name]
            if not tr:
                return None, raw
            return (torch.tensor(tr, dtype=torch.int64, device="cuda"), torch.tensor(of, dtype=torch.int32, device="cuda")), raw
        (wt, wraw), (rt, rraw) = table(wl["writer"]), table(wl["reader"])
        cw = [S.ColumnVector(S.DType(dt), len(x), x.view(torch.uint8))._c() for dt, x in zip((S.DType.INT64, S.DType.INT32), wt)] if wt else None
        cr = [S.ColumnVector(S.DType(dt), len(x), x.view(torch.uint8))._c() for dt, x in zip((S.DType.INT64, S.DType.INT32), rt)] if rt else None

        def step():
            N.check(lib.srj_orc_convert_timezones(C.byref(cin), C.byref(cw[0]) if cw else None, C.byref(cw[1]) if cw else None, wraw,
                                                  C.byref(cr[0]) if cr else None, C.byref(cr[1]) if cr else None, rraw, out.data_ptr(), None, st))

        def want(i):
            return OT.convert_orc(data[i].cpu().numpy(), *(x.cpu().numpy() for x in wt) if wt else (None, None), wraw,
                                  *(x.cpu().numpy() for x in rt) if rt else (None, None), rraw)
        bytes_alg = 16 * n

    step()
    torch.cuda.synchronize()
    idx = torch.from_numpy(np.unique(np.concatenate([np.random.default_rng(1).integers(0, n, 500_000), np.arange(n - 1000, n)]))).cuda()
    assert np.array_equal(out[idx].cpu().numpy(), want(idx)), f"bench_timezone {key}: values differ from the oracle"
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
        "ms_per_step": ms, "ms_per_step_min": ms_min, "higher_is_better": True, "data": "synthetic", "config": {"workload": key, "rows": n, **wl},
        "hbm_peak_frac": round(bytes_alg / (ms * 1e-3) / HBM_PEAK, 4),
        "models": {"note": "models, not measurements", "hbm": {"bytes": bytes_alg, "bound_ms": hbm_ms, "achieved_frac": round(hbm_ms / ms, 4)}},
        "card": card_info(), "clocks": clocks}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="all", choices=sorted(WORKLOADS) + ["all"])
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
