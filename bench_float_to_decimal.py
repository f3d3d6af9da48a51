#!/usr/bin/env python
"""bench_float_to_decimal.py -- benchmark of DecimalUtils.floatingPointToDecimal (CAST(float / double AS DECIMAL)) on one GPU.

    python bench_float_to_decimal.py [--workload all|f64_dec64_2|f32_dec32_2|f64_dec128_10|f64_dec128_30|f64_dec64_ovf_1pct]
                                     [--rows N] [--steps K] [--warmup W] [--dump-outputs DIR]

Workloads (100M rows each unless --rows says otherwise):
  f64_dec64_2         prices k / 100 within +-10^6 to DECIMAL64(18, 2)
  f32_dec32_2         FLOAT32 within +-10^6, 10% nulls, to DECIMAL32(9, 2)
  f64_dec128_10       log-uniform magnitudes 10^-6 .. 10^20 to DECIMAL128(38, 10)
  f64_dec128_30       magnitudes 10^-6 .. 10^6 to DECIMAL128(38, 30): every row takes the 18-digit step of the shifting
  f64_dec64_ovf_1pct  prices within +-10^6 to DECIMAL64(10, 2), 1% of the rows above the bound (null, failure row read)
A step is one C-ABI call (srj_float_to_fixed_point: the kernel, then the one read-back of the null count and the failure
row), inputs resident in HBM, outputs preallocated, CUDA events around each step.  Prints one JSON line per workload:
rows/s, the HBM model (algorithmic bytes: input, input mask, output and output mask) and its share of the H100 SXM
data-sheet bandwidth, the card and its power limit read in the same run, and the SM clock sampled during the run.
Before timing, the output is checked against the C oracle (oracle/float_to_decimal.c) on two slices.  --dump-outputs DIR
writes DIR/<workload>.npz with the whole input, its mask, the output values and validity, the failure row and the cast's
(type, precision, scale): use a small --rows with it.
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

from bench import ClockSampler  # noqa: E402
from bench_sha2 import card_info  # noqa: E402

HBM_PEAK = 3.35e12          # H100 SXM data sheet, HBM3 (a card allowed 700 W)
FLOAT32, FLOAT64, DEC32, DEC64, DEC128 = 9, 10, 25, 26, 27
WORKLOADS = {
    "f64_dec64_2": dict(name="FLOAT64 prices to DECIMAL64(18, 2)", src=FLOAT64, out=DEC64, precision=18, scale=-2, gen="prices"),
    "f32_dec32_2": dict(name="FLOAT32 with 10% nulls to DECIMAL32(9, 2)", src=FLOAT32, out=DEC32, precision=9, scale=-2, gen="uniform",
                        nulls=0.10),
    "f64_dec128_10": dict(name="FLOAT64 log-uniform 1e-6..1e20 to DECIMAL128(38, 10)", src=FLOAT64, out=DEC128, precision=38, scale=-10,
                          gen="log20"),
    "f64_dec128_30": dict(name="FLOAT64 log-uniform 1e-6..1e6 to DECIMAL128(38, 30)", src=FLOAT64, out=DEC128, precision=38, scale=-30,
                          gen="log6"),
    "f64_dec64_ovf_1pct": dict(name="FLOAT64 prices to DECIMAL64(10, 2), 1% over the bound", src=FLOAT64, out=DEC64, precision=10,
                               scale=-2, gen="prices", overflow=0.01),
}
WIDTH = {FLOAT32: 4, FLOAT64: 8, DEC32: 4, DEC64: 8, DEC128: 16}


def _mask(torch, g, n, frac):
    valid = torch.rand(n + (-n % 32), device="cuda", generator=g) >= frac
    w = (valid.view(-1, 32).to(torch.int64) << torch.arange(32, device="cuda", dtype=torch.int64)).sum(1)
    return torch.where(w >= 2**31, w - 2**32, w).to(torch.int32)


def make_input(torch, g, wl, n):
    sign = torch.where(torch.rand(n, device="cuda", generator=g) < 0.5, -1.0, 1.0).to(torch.float64)
    if wl["gen"] == "prices":
        x = torch.randint(-10**8, 10**8, (n,), device="cuda", generator=g, dtype=torch.int64).to(torch.float64) / 100.0
    elif wl["gen"] == "uniform":
        x = (torch.rand(n, device="cuda", generator=g, dtype=torch.float64) * 2 - 1) * 1e6
    else:
        hi = 20.0 if wl["gen"] == "log20" else 6.0
        x = sign * torch.pow(10.0, torch.rand(n, device="cuda", generator=g, dtype=torch.float64) * (hi + 6.0) - 6.0)
    if wl.get("overflow"):
        hit = torch.rand(n, device="cuda", generator=g) < wl["overflow"]
        x[hit] = sign[hit] * 1e9
    return x.to(torch.float32) if wl["src"] == FLOAT32 else x


def run(args, wl_key):
    import torch
    import srj_b200 as S
    from srj_b200 import _native as NT
    from oracle import float_to_decimal as D
    torch.cuda.set_device(0)
    wl = WORKLOADS[wl_key]
    lib = NT.lib()
    stream = torch.cuda.current_stream()
    st = int(stream.cuda_stream)
    g = torch.Generator(device="cuda").manual_seed(42)
    n = args.rows
    x = make_input(torch, g, wl, n)
    in_mask = _mask(torch, g, n, wl["nulls"]) if wl.get("nulls") else None
    col = S.ColumnVector(S.DType(wl["src"]), n, x.view(torch.uint8), in_mask)
    ci = col._c()
    ow = WIDTH[wl["out"]]
    out = torch.empty(n * ow, dtype=torch.uint8, device="cuda")
    out_mask = torch.empty((n + 31) // 32, dtype=torch.int32, device="cuda")
    nulls, row = C.c_int64(0), C.c_int64(-1)
    mask_bytes = 4 * ((n + 31) // 32)

    def step():
        NT.check(lib.srj_float_to_fixed_point(C.byref(ci), wl["out"], wl["precision"], wl["scale"], out.data_ptr(), out_mask.data_ptr(),
                                              C.byref(nulls), C.byref(row), st))
    bytes_alg = n * WIDTH[wl["src"]] + (mask_bytes if in_mask is not None else 0) + n * ow + mask_bytes

    def host_valid(m, s, e):
        return np.unpackbits(m[s // 32:(e + 31) // 32].cpu().numpy().view(np.uint8), bitorder="little")[:e - s].astype(bool)

    def outputs(s, e):
        vals = out[s * ow:e * ow].cpu().numpy()
        vals = vals.view(np.int32) if ow == 4 else vals.view(np.int64) if ow == 8 else vals.reshape(-1, 16)
        return vals, host_valid(out_mask, s, e)

    def oracle(s, e):
        m = in_mask[s // 32:(e + 31) // 32].cpu().numpy().view(np.uint32) if in_mask is not None else None
        return D.floating_point_to_decimal_c(x[s:e].cpu().numpy(), m, wl["out"], wl["precision"], wl["scale"])

    # correctness gate against the oracle before timing, on the first rows and on a 32-row-aligned slice in the middle
    step()
    torch.cuda.synchronize()
    n_check = min(n, 1_000_000)
    for s in (0, (n // 2) & ~31):
        e = min(n, s + n_check)
        want, wok, wfirst = oracle(s, e)
        got, ok = outputs(s, e)
        assert np.array_equal(ok, wok) and np.array_equal(got, want), f"bench_float_to_decimal {wl_key}: output differs from the oracle"
        if s == 0 and wfirst >= 0:
            assert row.value == wfirst, f"bench_float_to_decimal {wl_key}: failure row differs from the oracle"

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    sampler = ClockSampler(0)
    sampler.start()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
    for ev_a, ev_b in evs:
        ev_a.record(stream)
        step()
        ev_b.record(stream)
    torch.cuda.synchronize()
    clocks = sampler.stop()
    ms = float(np.mean([a.elapsed_time(b) for a, b in evs]))
    ms_min = float(np.min([a.elapsed_time(b) for a, b in evs]))
    if args.dump_outputs:
        os.makedirs(args.dump_outputs, exist_ok=True)
        vals, ok = outputs(0, n)
        np.savez(os.path.join(args.dump_outputs, f"{wl_key}.npz"), input=x.cpu().numpy(),
                 in_mask=in_mask.cpu().numpy().view(np.uint32) if in_mask is not None else np.zeros(0, np.uint32),
                 values=vals, valid=ok, failure_row=np.array(row.value),
                 config=np.array([wl["out"], wl["precision"], wl["scale"]]))
    card = card_info()
    sec = ms * 1e-3
    hbm_ms = bytes_alg / HBM_PEAK * 1e3
    print(json.dumps({
        "metric": f"rows_per_s_{wl_key}", "value": n / sec, "unit": "rows/s", "n_gpus": 1, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": ms, "ms_per_step_min": ms_min, "higher_is_better": True, "data": "synthetic",
        "config": {"workload": wl["name"], "rows": n, "null_count": nulls.value, "failure_row": row.value},
        "algorithmic_bytes_per_sec": bytes_alg / sec, "hbm_peak_frac": round(bytes_alg / sec / HBM_PEAK, 4),
        "models": {"note": "models, not measurements", "hbm": {"bytes": bytes_alg, "bound_ms": hbm_ms, "achieved_frac": round(hbm_ms / ms, 4)}},
        "card": card, "clocks": clocks}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="all", choices=["all"] + sorted(WORKLOADS))
    ap.add_argument("--gpus", type=int, default=1, choices=[1])
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write each workload's input and output as DIR/<workload>.npz")
    args = ap.parse_args()
    if args.steps < 1 or args.rows < 1:
        ap.error("--steps and --rows must be at least 1")
    for key in (sorted(WORKLOADS) if args.workload == "all" else [args.workload]):
        run(args, key)


if __name__ == "__main__":
    main()
