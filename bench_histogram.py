#!/usr/bin/env python
"""bench_histogram.py -- benchmark of Histogram (Spark's percentile / median over cudf histograms) on one GPU.

    python bench_histogram.py [--only NAME] [--steps K] [--warmup W] [--dump-outputs DIR]

Workloads (one step = the C-ABI calls of one Histogram call, inputs resident in HBM, outputs preallocated):
  median_small        percentileFromHistogram: 10M histograms of 5..15 INT64 elements, p = 0.5, flat output (the warp tier)
  percentiles_medium  1M histograms of 50..150 FLOAT64 elements, 5 percentages, list output (the warp tier)
  near_k              2,000 histograms of K - 64 .. K + 64 INT32 elements, half on each side of K = 8192, p = 0.5 (the CTA
                      tier below K, the radix select above it)
  large               8 histograms of 10M FLOAT64 elements, p = 0.5 (the radix select: 8 passes)
  create              createHistogramIfValid: 100M INT64 values with INT64 frequencies, 1% of them 0, list output
A percentile step is srj_percentile_from_histogram_size (one synchronisation) then srj_percentile_from_histogram; a
create step is srj_histogram_create_size then srj_histogram_create.  CUDA events bracket each step.  Each line reports
ms per step, the bytes the step must move (computed from the shapes: offsets, values, counts and masks read; results,
masks and offsets written) over that time, and its share of the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s), with
the card's name and power limit read in the same run.  --dump-outputs DIR writes the outputs of the last step.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, os.path.join(ROOT, "spark-rapids-jni_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402

from bench_sha2 import card_info  # noqa: E402

HBM_PEAK = 3.35e12
K = 8192
INT32, INT64, FLOAT64 = 3, 4, 10
WORKLOADS = {
    "median_small": dict(kind="pct", rows=10_000_000, lo=5, hi=15, type_id=INT64, pct=[0.5], lists=False),
    "percentiles_medium": dict(kind="pct", rows=1_000_000, lo=50, hi=150, type_id=FLOAT64, pct=[0.1, 0.25, 0.5, 0.75, 0.9], lists=True),
    "near_k": dict(kind="pct", rows=2_000, lo=K - 64, hi=K + 64, type_id=INT32, pct=[0.5], lists=False),
    "large": dict(kind="pct", rows=8, lo=10_000_000, hi=10_000_000, type_id=FLOAT64, pct=[0.5], lists=False),
    "create": dict(kind="create", rows=100_000_000, type_id=INT64),
}
WIDTH = {INT32: 4, INT64: 8, FLOAT64: 8}


def _pct_inputs(torch, S, w, gen):
    rows = w["rows"]
    lens = torch.randint(w["lo"], w["hi"] + 1, (rows,), generator=gen, device="cuda", dtype=torch.int64)
    offsets = torch.zeros(rows + 1, dtype=torch.int64, device="cuda")
    offsets[1:] = torch.cumsum(lens, 0)
    n = int(offsets[-1])
    if w["type_id"] == FLOAT64:
        vals = torch.randn(n, generator=gen, device="cuda", dtype=torch.float64) * 1000
    else:
        dt = torch.int32 if w["type_id"] == INT32 else torch.int64
        vals = torch.randint(-10**6, 10**6, (n,), generator=gen, device="cuda", dtype=dt)
    counts = torch.randint(1, 100, (n,), generator=gen, device="cuda", dtype=torch.int64)
    v = S.ColumnView(w["type_id"], n, vals.view(torch.uint8))
    c = S.ColumnView(INT64, n, counts.view(torch.uint8))
    return S.ColumnView.makeListView(offsets.to(torch.int32), S.ColumnView.makeStructView(v, c)), n


def run_pct(torch, S, N, w, steps, warmup, gen):
    view, n = _pct_inputs(torch, S, w, gen)
    rows, P, lists = w["rows"], len(w["pct"]), int(w["lists"])
    lib = N.lib()
    cin = view._c()
    pct = np.array(w["pct"], np.float64)
    ws = torch.empty(lib.srj_percentile_workspace_bytes(rows, n, P), dtype=torch.uint8, device="cuda")
    out = torch.empty(rows * P, dtype=torch.float64, device="cuda")
    mask = torch.empty((rows + 31) // 32, dtype=torch.int32, device="cuda")
    offs = torch.empty(rows + 1, dtype=torch.int32, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    valid, nv = C.c_int64(0), C.c_int64(0)

    def step():
        N.check(lib.srj_percentile_from_histogram_size(C.byref(cin), P, lists, C.byref(valid), C.byref(nv), ws.data_ptr(), stream))
        N.check(lib.srj_percentile_from_histogram(C.byref(cin), pct.ctypes.data_as(C.c_void_p), P, lists, out.data_ptr(), mask.data_ptr(),
                                                  offs.data_ptr(), ws.data_ptr(), stream))
    ms = _time(torch, step, steps, warmup)
    width = WIDTH[w["type_id"]]
    moved = (rows + 1) * 4 + n * (width + 8) + nv.value * 8 + (rows + 31) // 32 * 4 + (rows + 1) * 4 * lists
    outs = {"values": out[: nv.value].cpu().numpy(), "mask": mask.cpu().numpy().view(np.uint32).astype(np.float64)}
    return ms, moved, {"histograms": rows, "elements": n, "percentages": P}, outs


def run_create(torch, S, N, w, steps, warmup, gen):
    rows = w["rows"]
    vals = torch.randint(-10**9, 10**9, (rows,), generator=gen, device="cuda", dtype=torch.int64)
    freqs = torch.randint(1, 50, (rows,), generator=gen, device="cuda", dtype=torch.int64)
    freqs[torch.rand(rows, generator=gen, device="cuda") < 0.01] = 0
    v = S.ColumnView(INT64, rows, vals.view(torch.uint8))._c()
    f = S.ColumnView(INT64, rows, freqs.view(torch.uint8))._c()
    lib = N.lib()
    ws = torch.empty(lib.srj_histogram_workspace_bytes(rows), dtype=torch.uint8, device="cuda")
    out_v = torch.empty(rows, dtype=torch.int64, device="cuda")
    out_f = torch.empty(rows, dtype=torch.int64, device="cuda")
    offs = torch.empty(rows + 1, dtype=torch.int32, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    kept, nulls = C.c_int64(0), C.c_int64(0)

    def step():
        N.check(lib.srj_histogram_create_size(C.byref(v), C.byref(f), 1, C.byref(kept), C.byref(nulls), ws.data_ptr(), stream))
        N.check(lib.srj_histogram_create(C.byref(v), C.byref(f), 1, out_v.data_ptr(), None, out_f.data_ptr(), offs.data_ptr(), ws.data_ptr(),
                                         stream))
    ms = _time(torch, step, steps, warmup)
    # size pass: frequencies read, flags written; fill: flags scanned (read + write), values and frequencies read,
    # kept values / frequencies and offsets written
    moved = rows * 8 + rows * 4 + 2 * rows * 4 + rows * 16 + kept.value * 16 + (rows + 1) * 4
    outs = {"offsets": offs[-1:].cpu().numpy().astype(np.float64), "freq_sum": np.array([float(out_f[: kept.value].sum())])}
    return ms, moved, {"rows": rows, "kept": kept.value}, outs


def _time(torch, step, steps, warmup):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    times = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        step()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", choices=sorted(WORKLOADS))
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--dump-outputs")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_histogram: no CUDA device")
    import srj_b200 as S
    from srj_b200 import _native as N
    card = card_info()
    for name in ([args.only] if args.only else list(WORKLOADS)):
        w = WORKLOADS[name]
        gen = torch.Generator(device="cuda").manual_seed(1234)
        run = run_pct if w["kind"] == "pct" else run_create
        ms, moved, shape, outs = run(torch, S, N, w, args.steps, args.warmup, gen)
        rate = moved / (ms * 1e-3)
        print(json.dumps({"workload": name, **shape, "ms": round(ms, 4), "bytes": moved, "bytes_per_s": rate,
                          "hbm_floor_share": rate / HBM_PEAK, "card": card["name"], "power_limit_w": card["power_limit_w"]}), flush=True)
        if args.dump_outputs:
            os.makedirs(args.dump_outputs, exist_ok=True)
            for k, a in outs.items():
                np.save(os.path.join(args.dump_outputs, f"{name}_{k}.npy"), np.asarray(a, np.float64))
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
