#!/usr/bin/env python
"""bench_radix.py -- benchmark of the radix casts (Spark's conv(), bin() and hex()) on one GPU.

    python bench_radix.py [--workload all|conv_10_16|conv_16_m10|conv_row_bases|conv_overflow|bin_i64|hex_i64|dec_i32|bytes_to_hex]
                          [--scale F] [--steps K] [--warmup W]

Workloads (row counts times --scale):
  conv_10_16      NumberConverter.convert, bases 10 -> 16, 50M decimal strings of non-negative INT64
  conv_16_m10     convert, bases 16 -> -10, 50M hex strings, half of them with '-'
  conv_row_bases  convert with per-row bases: the conv_10_16 strings, fromBase uniform in 2..36, toBase +-2..36, 1% of
                  the base rows null or out of range
  conv_overflow   isConvertOverflow on the conv_10_16 input with one more row at 2^64
  bin_i64         CastStrings.fromLongToBinary, 100M INT64 below 2^20 (the chars stay under 2^31), 10% nulls
  hex_i64         fromIntegersWithBase(16), 100M INT64 over the whole range
  dec_i32         fromIntegersWithBase(10), 100M INT32 over the whole range
  bytes_to_hex    bytesToHex, 16M strings of 4-40 bytes
A step is the op's C-ABI calls with preallocated outputs: the sizes call (kernel, scan and the one read-back of the
total) and the write call, or the one overflow call, with CUDA events around each step.  The inputs are built on the
device, the strings by the casts themselves.  Each workload's output is checked against oracle/radix.py on two slices
before it is timed.  Prints one JSON line per workload: rows/s, the algorithmic bytes (inputs read and outputs written;
conv's 8-byte kept value per row is not counted) and their share of the H100 SXM data-sheet bandwidth, the card and its
power limit read in the same run, and the SM clock sampled during it.
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
WORKLOADS = ["conv_10_16", "conv_16_m10", "conv_row_bases", "conv_overflow", "bin_i64", "hex_i64", "dec_i32", "bytes_to_hex"]
CHECK_ROWS = 20_000


def _mask(torch, g, n, frac):
    valid = torch.rand(n + (-n % 32), device="cuda", generator=g) >= frac
    w = (valid.view(-1, 32).to(torch.int64) << torch.arange(32, device="cuda", dtype=torch.int64)).sum(1)
    return torch.where(w >= 2**31, w - 2**32, w).to(torch.int32)


def _valid(mask, s, e):
    if mask is None:
        return [True] * (e - s)
    bits = np.unpackbits(mask.cpu().numpy().view(np.uint8), bitorder="little")
    return bits[s:e].astype(bool).tolist()


def _rows(col, s, e):
    """rows s .. e of a STRING / LIST<UINT8> column as bytes, None for a null row"""
    offs = col.offsets[s:e + 1].cpu().numpy().astype(np.int64)
    data = (col.child.data if col.child is not None else col.data)[offs[0]:offs[-1]].cpu().numpy().tobytes()
    valid = _valid(col.mask, s, e)
    return [data[a - offs[0]:b - offs[0]] if v else None for a, b, v in zip(offs[:-1], offs[1:], valid)]


def _out_rows(offsets, chars, mask, s, e):
    offs = offsets[s:e + 1].cpu().numpy().astype(np.int64)
    data = chars[offs[0]:offs[-1]].cpu().numpy().tobytes()
    valid = _valid(mask, s, e)
    return [data[a - offs[0]:b - offs[0]] if v else None for a, b, v in zip(offs[:-1], offs[1:], valid)]


def _ints(torch, g, n, lo, hi, dtype):
    return torch.randint(lo, hi, (n,), device="cuda", generator=g, dtype=torch.int64).to(dtype)


def _nbytes(t):
    return 0 if t is None else t.numel() * t.element_size()


def run(args, key):
    import torch
    import srj_b200 as S
    from srj_b200 import _native as NT
    from srj_b200.cast import CastStrings
    from srj_b200.radix import NumberConverter
    from oracle import radix as R
    torch.cuda.set_device(0)
    lib = NT.lib()
    stream = torch.cuda.current_stream()
    st = int(stream.cuda_stream)
    g = torch.Generator(device="cuda").manual_seed(42)

    def int_col(t, v, mask=None):
        return S.ColumnVector(S.DType(t), v.numel(), v.view(torch.uint8), mask)

    def decimal_strings(n):
        return CastStrings.fromIntegersWithBase(int_col(S.DType.INT64, _ints(torch, g, n, 0, 2**63 - 1, torch.int64)), 10)

    if key.startswith("conv"):
        n = int(50_000_000 * args.scale)
        fb_col = tb_col = None
        if key == "conv_16_m10":
            signed = CastStrings.fromIntegersWithBase(int_col(S.DType.INT64, _ints(torch, g, n, -(2**63), 2**63 - 1, torch.int64)), 10)
            inp, fb, tb = NumberConverter.convertCvSS(signed, 10, -16), 16, -10
        else:
            inp, fb, tb = decimal_strings(n), 10, 16
        if key == "conv_row_bases":
            fbv = _ints(torch, g, n, 2, 37, torch.int32)
            tbv = _ints(torch, g, n, 2, 37, torch.int32) * torch.where(torch.rand(n, device="cuda", generator=g) < 0.5, -1, 1).to(torch.int32)
            bad = torch.rand(n, device="cuda", generator=g) < 0.005
            fbv[bad] = 37
            fb_col, tb_col = int_col(S.DType.INT32, fbv), int_col(S.DType.INT32, tbv, _mask(torch, g, n, 0.005))
        if key == "conv_overflow":
            big = torch.tensor(list(b"18446744073709551616"), dtype=torch.uint8, device="cuda")
            end = inp.offsets[-1:]
            inp = S.ColumnVector(S.DType(S.DType.STRING), n + 1, torch.cat([inp.data, big]), None,
                                 torch.cat([inp.offsets, end + big.numel()]))
            n += 1
        ci = inp._c()
        cf, ct = (fb_col._c() if fb_col is not None else None), (tb_col._c() if tb_col is not None else None)
        args3 = [C.byref(ci), None, 0, C.byref(cf) if cf is not None else None, fb, C.byref(ct) if ct is not None else None, tb]
        if key == "conv_overflow":
            flag = C.c_int32(0)

            def step():
                NT.check(lib.srj_conv_overflow(*args3, C.byref(flag), st))
            step()
            assert flag.value == 1 and NumberConverter.isConvertOverflowCvSS(inp, 10, 16), "bench_radix conv_overflow: no overflow found"
            s0 = (n // 2) & ~31
            assert not R.conv_overflow(_rows(inp, s0, s0 + CHECK_ROWS), 10, 16)
            assert R.conv_overflow(_rows(inp, n - CHECK_ROWS, n), 10, 16), "bench_radix conv_overflow: oracle finds no overflow"
            out_bytes, config = 0, {"overflow": True}
        else:
            offsets = torch.empty(n + 1, dtype=torch.int32, device="cuda")
            mask = torch.empty((n + 31) // 32, dtype=torch.int32, device="cuda")
            ws = torch.empty(lib.srj_conv_workspace_bytes(n), dtype=torch.uint8, device="cuda")
            nulls, total = C.c_int64(0), C.c_int64(0)
            NT.check(lib.srj_conv_sizes(*args3, offsets.data_ptr(), mask.data_ptr(), C.byref(nulls), C.byref(total), ws.data_ptr(), st))
            chars = torch.empty(max(total.value, 1), dtype=torch.uint8, device="cuda")

            def step():
                NT.check(lib.srj_conv_sizes(*args3, offsets.data_ptr(), mask.data_ptr(), C.byref(nulls), C.byref(total), ws.data_ptr(), st))
                NT.check(lib.srj_conv(*args3, offsets.data_ptr(), chars.data_ptr(), ws.data_ptr(), st))
            step()
            torch.cuda.synchronize()
            for s in (0, (n // 2) & ~31):
                e = min(n, s + CHECK_ROWS)
                fbs = fb_col.data.view(torch.int32)[s:e].cpu().tolist() if fb_col is not None else fb
                tbs = tb_col.data.view(torch.int32)[s:e].cpu().tolist() if tb_col is not None else tb
                if tb_col is not None:
                    tbs = [t if v else None for t, v in zip(tbs, _valid(tb_col.mask, s, e))]
                want = R.conv(_rows(inp, s, e), fbs, tbs)
                assert _out_rows(offsets, chars, mask if nulls.value else None, s, e) == want, f"bench_radix {key}: output differs from the oracle"
            out_bytes, config = 4 * (n + 1) + total.value + _nbytes(mask), {"null_count": nulls.value, "chars": total.value}
        in_bytes = _nbytes(inp.offsets) + int(inp.offsets[-1] - inp.offsets[0]) + sum(_nbytes(c.data) + _nbytes(c.mask)
                                                                                       for c in (fb_col, tb_col) if c is not None)
    else:
        if key == "bytes_to_hex":
            n = int(16_000_000 * args.scale)
            lens = _ints(torch, g, n, 4, 41, torch.int32)
            offs = torch.zeros(n + 1, dtype=torch.int32, device="cuda")
            offs[1:] = torch.cumsum(lens, 0, dtype=torch.int32)
            data = _ints(torch, g, int(offs[-1]), 0, 256, torch.uint8)
            col = S.ColumnVector(S.DType(S.DType.STRING), n, data, None, offs)
            sizes = lambda o, t: lib.srj_bytes_to_hex_sizes(C.byref(ci), o, t, st)
            write = lambda out: lib.srj_bytes_to_hex(C.byref(ci), C.byref(out), st)
            oracle = lambda s, e: [r.hex().upper().encode() for r in _rows(col, s, e)]
            in_bytes = _nbytes(offs) + _nbytes(data)
        else:
            n = int(100_000_000 * args.scale)
            if key == "bin_i64":
                col = int_col(S.DType.INT64, _ints(torch, g, n, 0, 2**20, torch.int64), _mask(torch, g, n, 0.10))
                base, bits = 2, 64
                ws_fn = lib.srj_long_to_binary_workspace_bytes
                sizes = lambda o, t: lib.srj_long_to_binary_sizes(C.byref(ci), o, t, ws.data_ptr(), st)
                write = lambda out: lib.srj_long_to_binary(C.byref(ci), C.byref(out), st)
            else:
                base, bits, t, dt = (16, 64, S.DType.INT64, torch.int64) if key == "hex_i64" else (10, 32, S.DType.INT32, torch.int32)
                col = int_col(t, _ints(torch, g, n, -(2**(bits - 1)), 2**(bits - 1) - 1, dt))
                ws_fn = lib.srj_integers_to_string_workspace_bytes
                sizes = lambda o, tt: lib.srj_integers_to_string_sizes(C.byref(ci), base, o, tt, ws.data_ptr(), st)
                write = lambda out: lib.srj_integers_to_string(C.byref(ci), base, C.byref(out), st)
            ws = torch.empty(ws_fn(n), dtype=torch.uint8, device="cuda")
            npt = np.int64 if bits == 64 else np.int32

            def oracle(s, e):
                vals = col.data.cpu().numpy().view(npt)[s:e].tolist()
                valid = _valid(col.mask, s, e)
                if base == 2:
                    return R.long_to_binary(vals, valid)
                return R.integers_to_string(vals, valid, bits, True, base)
            in_bytes = _nbytes(col.data) + _nbytes(col.mask)
        ci = col._c()
        offsets = torch.empty(n + 1, dtype=torch.int32, device="cuda")
        total = C.c_int64(0)
        NT.check(sizes(offsets.data_ptr(), C.byref(total)))
        chars = torch.empty(max(total.value, 1), dtype=torch.uint8, device="cuda")
        mask = torch.empty((n + 31) // 32, dtype=torch.int32, device="cuda") if col.mask is not None else None
        out = S.ColumnVector(S.DType(S.DType.STRING), n, chars, mask, offsets)._c()

        def step():
            NT.check(sizes(offsets.data_ptr(), C.byref(total)))
            NT.check(write(out))
        step()
        torch.cuda.synchronize()
        for s in (0, (n // 2) & ~31):
            e = min(n, s + CHECK_ROWS)
            want = oracle(s, e)
            got = _out_rows(offsets, chars, mask, s, e)
            assert got == want, f"bench_radix {key}: output differs from the oracle"
        out_bytes, config = _nbytes(offsets) + total.value + _nbytes(mask), {"chars": total.value}

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
    bytes_alg = in_bytes + out_bytes
    sec = ms * 1e-3
    hbm_ms = bytes_alg / HBM_PEAK * 1e3
    print(json.dumps({
        "metric": f"rows_per_s_{key}", "value": n / sec, "unit": "rows/s", "n_gpus": 1, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": ms, "ms_per_step_min": ms_min, "higher_is_better": True, "data": "synthetic",
        "config": dict(workload=key, rows=n, **config),
        "algorithmic_bytes_per_sec": bytes_alg / sec, "hbm_peak_frac": round(bytes_alg / sec / HBM_PEAK, 4),
        "models": {"note": "models, not measurements", "hbm": {"bytes": bytes_alg, "bound_ms": hbm_ms, "achieved_frac": round(hbm_ms / ms, 4)}},
        "card": card_info(), "clocks": clocks}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="all", choices=["all"] + WORKLOADS)
    ap.add_argument("--gpus", type=int, default=1, choices=[1])
    ap.add_argument("--scale", type=float, default=1.0, help="multiplies every workload's row count")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if args.steps < 1 or args.scale <= 0:
        ap.error("--steps must be at least 1 and --scale positive")
    for key in (WORKLOADS if args.workload == "all" else [args.workload]):
        run(args, key)


if __name__ == "__main__":
    main()
