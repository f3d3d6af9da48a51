#!/usr/bin/env python
"""bench_arithmetic.py -- benchmark of Arithmetic.multiply and Arithmetic.round on one GPU.

    python bench_arithmetic.py [--workload mul_i64|mul_i32_scalar|mul_try_1pct|round_f64_2|round_i64_ansi_m3|round_dec128_m2]
                               [--steps K] [--warmup W] [--dump-outputs DIR]

Workloads (100M rows each):
  mul_i64            INT64 * INT64 columns, ANSI mode, no overflow (the error-row read-back every step)
  mul_i32_scalar     INT32 column * INT32 scalar, default mode, 10% nulls (output mask and null count)
  mul_try_1pct       INT64 * INT64 columns, try mode, 1% of the rows overflow to null
  round_f64_2        round(FLOAT64, 2) HALF_UP, 10% nulls
  round_i64_ansi_m3  round(INT64, -3) HALF_UP in ANSI mode, no overflow (the error-row read-back every step)
  round_dec128_m2    round(DECIMAL128(38, 4), -2) HALF_EVEN: a 10^6 division per row
A step is one C-ABI call (srj_multiply or srj_round), inputs resident in HBM, outputs preallocated, CUDA events around
each step.  Prints one JSON line: rows/s, the HBM model (algorithmic bytes: operands, output and masks) and its share of
the H100 SXM data-sheet bandwidth, the card and its power limit read in the same run, and the SM clock sampled during the
run.  Before timing, the output is checked against oracle/arithmetic.py on two slices.  --dump-outputs DIR writes a
seeded sample of the output plus whole-output checksums (float .npy files).  Shares its measurement helpers with bench.py.
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

from bench import ClockSampler, byte_sum, sample_rows, write_dump  # noqa: E402
from bench_sha2 import card_info  # noqa: E402

HBM_PEAK = 3.35e12          # H100 SXM data sheet, HBM3 (a card allowed 700 W)
INT32, INT64, FLOAT64, DECIMAL128 = 3, 4, 10, 27
N = 100_000_000
WORKLOADS = {
    "mul_i64": dict(name="INT64 * INT64, ANSI, no overflow", op="mul", type_id=INT64, ansi=1, try_mode=0, nulls=None, scalar=False),
    "mul_i32_scalar": dict(name="INT32 * INT32 scalar, 10% nulls", op="mul", type_id=INT32, ansi=0, try_mode=0, nulls=0.10, scalar=True),
    "mul_try_1pct": dict(name="INT64 * INT64, try mode, 1% overflow", op="mul", type_id=INT64, ansi=0, try_mode=1, nulls=None,
                         scalar=False, overflow=0.01),
    "round_f64_2": dict(name="round(FLOAT64, 2) HALF_UP, 10% nulls", op="round", type_id=FLOAT64, dp=2, mode=0, ansi=0, nulls=0.10),
    "round_i64_ansi_m3": dict(name="round(INT64, -3) HALF_UP, ANSI, no overflow", op="round", type_id=INT64, dp=-3, mode=0, ansi=1,
                              nulls=None),
    "round_dec128_m2": dict(name="round(DECIMAL128(38, 4), -2) HALF_EVEN", op="round", type_id=DECIMAL128, scale=-4, dp=-2, mode=1,
                            ansi=0, nulls=None),
}
NP = {INT32: np.int32, INT64: np.int64, FLOAT64: np.float64, DECIMAL128: np.uint64}


def _mask(torch, g, n, frac):
    valid = torch.rand(n + (-n % 32), device="cuda", generator=g) >= frac
    w = (valid.view(-1, 32).to(torch.int64) << torch.arange(32, device="cuda", dtype=torch.int64)).sum(1)
    return torch.where(w >= 2**31, w - 2**32, w).to(torch.int32)


def make_column(torch, S, g, t, n, nulls, scale=0, bits=None):
    mask = _mask(torch, g, n, nulls) if nulls else None
    if t == FLOAT64:
        data = (torch.randn(n, device="cuda", generator=g, dtype=torch.float64) * 1e4).view(torch.uint8)
    elif t == DECIMAL128:                  # |unscaled| < 2^100: DECIMAL(38, 4) values of every size up to 30 digits
        d = torch.randint(-2**62, 2**62, (n, 2), device="cuda", generator=g, dtype=torch.int64)
        d[:, 1] >>= torch.randint(26, 64, (n,), device="cuda", generator=g)
        data = d.view(torch.uint8).reshape(-1)
    else:
        lim = 2 ** (bits or 30)
        data = torch.randint(-lim, lim, (n,), device="cuda", generator=g, dtype=torch.int64)
        data = (data if t == INT64 else data.to(torch.int32)).view(torch.uint8)
    return S.ColumnVector(S.DType(t, scale), n, data, mask)


def host(col, s, e):
    w = col.dtype.size_in_bytes()
    data = col.data[s * w:e * w].cpu().numpy().view(NP[col.dtype.type_id])
    valid = None
    if col.mask is not None:
        valid = np.unpackbits(col.mask[s // 32:(e + 31) // 32].cpu().numpy().view(np.uint8), bitorder="little")[:e - s].astype(bool)
    return data, valid


def run(args, wl_key):
    import torch
    import srj_b200 as S
    from srj_b200 import _native as NT
    from srj_b200.bloom import Scalar
    from oracle import arithmetic as A
    torch.cuda.set_device(0)
    wl = WORKLOADS[wl_key]
    lib = NT.lib()
    stream = torch.cuda.current_stream()
    st = int(stream.cuda_stream)
    g = torch.Generator(device="cuda").manual_seed(42)
    n, t = N, wl["type_id"]
    width = 16 if t == DECIMAL128 else 8 if t in (INT64, FLOAT64) else 4
    mask_bytes = 4 * ((n + 31) // 32)
    out = torch.empty(n * width, dtype=torch.uint8, device="cuda")
    out_mask = torch.empty((n + 31) // 32, dtype=torch.int32, device="cuda")
    nulls, row = C.c_int64(0), C.c_int64(-1)
    if wl["op"] == "mul":
        a = make_column(torch, S, g, t, n, wl["nulls"], bits=31 if wl.get("overflow") else 30)
        if wl["scalar"]:
            sc = Scalar.fromInt(3)
            ca, cb, bv = a._c(), NT.SrjColumn(), sc.valid.data_ptr()
            cb.type_id, cb.size, cb.data = t, 1, sc.data.data_ptr()
        else:
            b = make_column(torch, S, g, t, n, None, bits=2)
            if wl.get("overflow"):             # 1% of the rows get a factor that overflows INT64 with |a| >= 2^30
                hit = torch.rand(n, device="cuda", generator=g) < wl["overflow"]
                bb = b.data.view(torch.int64)
                bb[hit] = 2**40
                a.data.view(torch.int64)[hit] |= 2**30
            ca, cb, bv = a._c(), b._c(), None
        can_null = wl["scalar"] or wl["nulls"] or wl["try_mode"]

        def step():
            NT.check(lib.srj_multiply(C.byref(ca), None, C.byref(cb), bv, wl["ansi"], wl["try_mode"], out.data_ptr(),
                                      out_mask.data_ptr() if can_null else None, C.byref(nulls), C.byref(row), st))
        ops = 1 if wl["scalar"] else 2
        bytes_alg = ops * n * width + n * width + (mask_bytes if wl["nulls"] else 0) + (mask_bytes if can_null else 0)

        def check(s, e):
            xa, va = host(a, s, e)
            if wl["scalar"]:
                want, wv, err = A.multiply(xa, va, np.array([3], np.int32), True, wl["ansi"], wl["try_mode"], b_scalar=True)
            else:
                xb, vb = host(b, s, e)
                want, wv, err = A.multiply(xa, va, xb, vb, wl["ansi"], wl["try_mode"])
            assert err == -1 and row.value == -1, "bench_arithmetic: unexpected overflow"
            got = out[s * width:e * width].cpu().numpy().view(NP[t])
            assert np.array_equal(got, want), "bench_arithmetic: values differ from the oracle"
            if can_null:
                gv = np.unpackbits(out_mask[s // 32:(e + 31) // 32].cpu().numpy().view(np.uint8), bitorder="little")[:e - s].astype(bool)
                assert np.array_equal(gv, wv), "bench_arithmetic: mask differs from the oracle"
    else:
        bits = 62 if t == INT64 else None
        a = make_column(torch, S, g, t, n, wl["nulls"], scale=wl.get("scale", 0), bits=bits)
        ca = a._c()

        def step():
            NT.check(lib.srj_round(C.byref(ca), wl["dp"], wl["mode"], wl["ansi"], out.data_ptr(),
                                   out_mask.data_ptr() if a.mask is not None else None, C.byref(row), st))
        bytes_alg = 2 * n * width + (2 * mask_bytes if a.mask is not None else 0)    # the mask is read and copied

        def check(s, e):
            xa, va = host(a, s, e)
            if t == DECIMAL128:
                want, err = A.round_decimal128(xa, wl["scale"], wl["dp"], wl["mode"]), -1
            else:
                want, err = A.round_(xa, va, wl["dp"], wl["mode"], bool(wl["ansi"]))
            assert err == -1 and row.value == -1, "bench_arithmetic: unexpected overflow"
            got = out[s * width:e * width].cpu().numpy().view(NP[t])
            assert np.array_equal(got.reshape(-1).view(np.uint8), np.asarray(want).reshape(-1).view(np.uint8)), \
                "bench_arithmetic: values differ from the oracle"

    # correctness gate against the oracle before timing, on the first rows and on a 32-row-aligned slice in the middle
    step()
    torch.cuda.synchronize()
    n_check = 50_000 if t == DECIMAL128 else 250_000
    for s in (0, (n // 2) & ~31):
        check(s, s + n_check)

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
    ms = float(np.mean([x.elapsed_time(y) for x, y in evs]))
    ms_min = float(np.min([x.elapsed_time(y) for x, y in evs]))
    if args.dump_outputs:
        arrays = {}
        for name, tsr in (("out", out), ("mask", out_mask)):
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
        "config": {"workload": wl["name"], "rows": n, "null_count": nulls.value},
        "algorithmic_bytes_per_sec": bytes_alg / sec, "hbm_peak_frac": round(bytes_alg / sec / HBM_PEAK, 4),
        "models": {"note": "models, not measurements", "hbm": {"bytes": bytes_alg, "bound_ms": hbm_ms, "achieved_frac": round(hbm_ms / ms, 4)}},
        "card": card, "clocks": clocks}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="mul_i64", choices=sorted(WORKLOADS))
    ap.add_argument("--gpus", type=int, default=1, choices=[1])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write a seeded sample of the output plus checksums as DIR/<name>.npy")
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be at least 1")
    run(args, args.workload)


if __name__ == "__main__":
    main()
