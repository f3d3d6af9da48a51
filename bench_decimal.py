#!/usr/bin/env python
"""bench_decimal.py -- benchmark of DecimalUtils' DECIMAL128 arithmetic on one GPU.

    python bench_decimal.py [--workload mul|mul_exact|div|intdiv|rem|add] [--steps K] [--warmup W]

Workloads (100M rows, 10% nulls on the left operand; cudf scales in brackets):
  mul        decimal(38,10) x decimal(38,10) -> scale 6 [-10, -10 -> -6], interim cast, ~28-digit values: every row rounds
  mul_exact  store_sales-like decimal(7,2) operands held as DECIMAL128 -> scale 4 [-2, -2 -> -4]: no division
  div        decimal(38,10) / decimal(38,10) -> scale 6 [-10, -10 -> -6]: a per-row 128-bit divisor
  intdiv     integral divide of the same operands (INT64 out)
  rem        remainder of the same operands [-> -10]
  add        scales 10 and 2 -> scale 10 [-10, -2 -> -10]: one operand scaled by 10^8, no division
A step is one srj_decimal128_binary call (the mask AND, the one null-count read-back, the row kernel), inputs resident in
HBM, outputs preallocated, CUDA events around each step.  Prints one JSON line: rows/s, the HBM model (algorithmic bytes
over the H100 SXM data-sheet 3.35 TB/s), the issue model (SASS instructions a row runs on the workload's path, from nvdisasm, issued at
one warp-instruction per clock per SM sub-partition), the card and its power limit read in the same run, the SM clock
sampled during the run, and a one-core baseline of oracle/decimal.py on a sample.  Shares its helpers with bench.py.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import re
import shutil
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, os.path.join(ROOT, "spark-rapids-jni_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402

from bench import ClockSampler  # noqa: E402
from bench_sha2 import card_info  # noqa: E402

HBM_PEAK = 3.35e12          # H100 SXM data sheet, HBM3 (a card allowed 700 W)
SMS, SUBPARTITIONS = 132, 4  # H100 SXM
MUL, DIV, INTDIV, REM, ADD = 0, 1, 2, 3, 4
DIVISION = ("reciprocal_word", "make_div", "div_3by2", "shl_in", "udivrem", "sdivrem", "round_half_up")
WORKLOADS = {
    # kernel: the instantiation this call's path runs (divide: x = -6 and 0, the multiply-then-divide path; remainder:
    # ds = ns = 0; add: ka = 0, kb = 8, kt = 0).  ran: the share of a decimal_arith.cuh function's inlined copies that the
    # workload's rows execute inside that kernel, where it is not all of them: the multiply chooses its roundings and its
    # scale-up per row (mul: the interim rounding and the scale-up by 10^4, not the final rounding; mul_exact: neither);
    # add runs one of its two scale-ups (b's), the remainder one of its three multiplies (the quotient times the divisor)
    "mul": dict(op=MUL, scales=(-10, -10, -6), digits=28, kernel="MulOpILb1EE", ran={f: 0.5 for f in DIVISION}),
    "mul_exact": dict(op=MUL, scales=(-2, -2, -4), digits=7, kernel="MulOpILb1EE", ran={f: 0.0 for f in DIVISION + ("mul",)}),
    "div": dict(op=DIV, scales=(-10, -10, -6), digits=28, kernel="DivOpILb0ELi2EE", ran={}),
    "intdiv": dict(op=INTDIV, scales=(-10, -10, 0), digits=28, kernel="DivOpILb1ELi2EE", ran={}),
    "rem": dict(op=REM, scales=(-10, -10, -10), digits=28, kernel="RemOpILb0ELb0EE", ran={"mul": 1 / 3}),
    "add": dict(op=ADD, scales=(-10, -2, -10), digits=28, kernel="AddOpILb0ELi0EE", ran={"mul": 0.5}),
}
ROWS, NULLS, ROWS_PER_THREAD = 100_000_000, 0.10, 4


def _mask(torch, g, n, frac):
    valid = torch.rand(n + (-n % 32), device="cuda", generator=g) >= frac
    w = (valid.view(-1, 32).to(torch.int64) << torch.arange(32, device="cuda", dtype=torch.int64)).sum(1)
    return torch.where(w >= 2**31, w - 2**32, w).to(torch.int32)


def _operand(torch, g, n, digits):
    """|v| < 10^digits, both signs, as little-endian int64 pairs"""
    bound = 10 ** digits
    if digits <= 18:
        lo = torch.randint(-bound + 1, bound, (n,), dtype=torch.int64, device="cuda", generator=g)
        return torch.stack([lo, lo >> 63], 1).contiguous()
    hi_bits = (bound.bit_length() - 1) - 64             # |hi| < 2^hi_bits keeps |v| < 2^(64 + hi_bits) <= 10^digits
    v = torch.randint(-2**63, 2**63 - 1, (n, 2), dtype=torch.int64, device="cuda", generator=g)
    v[:, 1] >>= 64 - hi_bits
    v[:, 1] |= (v[:, 1] == 0).to(torch.int64)           # most rows keep all their digits
    return v


def _arith_functions():
    """line -> function name of csrc/decimal_arith.cuh (a function spans from its signature to the next one)"""
    path = os.path.join(ROOT, "spark-rapids-jni_b200", "csrc", "decimal_arith.cuh")
    owner, cur = {}, None
    for i, line in enumerate(open(path), 1):
        m = re.match(r"__host__ __device__ __forceinline__ [\w:]+ (\w+)\(", line)
        if m:
            cur = m.group(1)
        owner[i] = cur
    return owner


def issue_model(wl, tmp):
    """SASS instructions a row executes on this workload's path, itemised by the decimal_arith.cuh function the
    instruction comes from (nvdisasm's line table of the built library; the row code is unrolled over ROWS_PER_THREAD
    rows), weighted by the share of each function's copies the rows run.  Branches inside a function, and helpers shared
    by run and skipped code (neg, add, ge), are counted in full, so this is an upper bound for the path."""
    from srj_b200 import _native as N
    cuda = os.path.dirname(os.path.dirname(shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"))
    try:
        subprocess.run([os.path.join(cuda, "bin", "cuobjdump"), "-xelf", "all", N.LIB_PATH], cwd=tmp, capture_output=True, timeout=300,
                       check=True)
        sass = ""
        for f in sorted(os.listdir(tmp)):
            if f.endswith(".cubin"):
                out = subprocess.run([os.path.join(cuda, "bin", "nvdisasm"), "-c", "-gi", f], cwd=tmp, capture_output=True, text=True,
                                     timeout=300).stdout
                if "dec_map_kernel" in out:
                    sass = out
                    break
    except Exception as e:  # noqa: BLE001
        return {"error": repr(e)}
    owner = _arith_functions()
    for sec in re.split(r"\n\.text\.", sass):
        name = sec.split(":", 1)[0]
        if "\n" in name or "dec_map_kernel" not in name or wl["kernel"] not in name:
            continue
        where, by_fn, ops, fresh = "kernel", {}, {}, True
        for line in sec.splitlines():
            m = re.search(r'//## File "[^"]*/([^"/]+)", line (\d+)', line)
            if m:                          # an instruction's annotations run innermost first: keep the first of a run
                if fresh:
                    fn = owner.get(int(m.group(2))) if m.group(1) == "decimal_arith.cuh" else None
                    where = fn or m.group(1)
                fresh = False
                continue
            m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s*(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_]*)", line)
            if m:
                fresh = True
                by_fn[where] = by_fn.get(where, 0) + 1
                ops[m.group(1)] = ops.get(m.group(1), 0) + 1
        total = sum(by_fn.values())
        path = sum(v * wl["ran"].get(k, 1.0) for k, v in by_fn.items())
        return {"kernel": name, "kernel_sass_instructions": total, "path_instructions": path, "per_row": path / ROWS_PER_THREAD,
                "by_function_per_row": {k: v / ROWS_PER_THREAD for k, v in sorted(by_fn.items(), key=lambda kv: -kv[1])},
                "share_run": wl["ran"],
                "by_opcode": dict(sorted(ops.items(), key=lambda kv: -kv[1])[:12])}
    return {"error": f"kernel {wl['kernel']} not found"}


def cpu_baseline(wl, ha, hb, n_sample):
    from oracle import decimal as O
    sa, sb, so = wl["scales"]
    a, b = ha[:n_sample], hb[:n_sample]
    t0 = time.perf_counter()
    for x, y in zip(a, b):
        O.row(wl["op"], x, y, sa, sb, so, True)
    sec = time.perf_counter() - t0
    return {"value": n_sample / sec, "unit": "rows/s", "cores": 1, "kind": "Python-integer oracle (oracle/decimal.py)",
            "sample": f"{n_sample} rows"}


def run(args, key):
    import torch
    import srj_b200 as S
    from oracle import decimal as O
    from srj_b200 import _native as N
    torch.cuda.set_device(0)
    wl = WORKLOADS[key]
    op, (sa, sb, so) = wl["op"], wl["scales"]
    n = args.rows
    g = torch.Generator(device="cuda").manual_seed(42)
    av, bv = _operand(torch, g, n, wl["digits"]), _operand(torch, g, n, wl["digits"])
    mask = _mask(torch, g, n, NULLS)
    ca = S.ColumnVector(S.DType(S.DType.DECIMAL128, sa), n, av.view(torch.uint8).view(-1), mask)._c()
    cb = S.ColumnVector(S.DType(S.DType.DECIMAL128, sb), n, bv.view(torch.uint8).view(-1))._c()
    width = 8 if op == INTDIV else 16
    ovf = torch.empty(n, dtype=torch.uint8, device="cuda")
    out = torch.empty(n * width, dtype=torch.uint8, device="cuda")
    out_mask = torch.empty((n + 31) // 32, dtype=torch.int32, device="cuda")
    nulls = C.c_int64(0)
    lib = N.lib()
    stream = torch.cuda.current_stream()
    st = int(stream.cuda_stream)

    def step():
        N.check(lib.srj_decimal128_binary(op, C.byref(ca), C.byref(cb), so, 1, ovf.data_ptr(), out.data_ptr(), out_mask.data_ptr(),
                                          C.byref(nulls), st))

    # correctness gate against the oracle before timing, on a sample of rows
    step()
    torch.cuda.synchronize()
    idx = np.unique(np.concatenate([np.arange(min(n, 1000)), np.random.default_rng(1).integers(0, n, 2000)]))
    ha = O.to_ints(av.cpu().numpy()[idx].view(np.uint8).reshape(-1))
    hb = O.to_ints(bv.cpu().numpy()[idx].view(np.uint8).reshape(-1))
    go, gv = ovf.cpu().numpy()[idx], out.view(torch.int64).cpu().numpy().reshape(n, width // 8)[idx]
    for j in range(len(idx)):
        f, v = O.row(op, ha[j], hb[j], sa, sb, so, True)
        got = (int(gv[j, 0]) & (2**64 - 1)) | (((int(gv[j, 1]) & (2**64 - 1)) << 64) if width == 16 else 0)
        assert bool(go[j]) == f and got == v & (2 ** (8 * width) - 1), f"bench_decimal: row {idx[j]} differs from the oracle"

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
    card = card_info()
    mask_bytes = 4 * ((n + 31) // 32)
    bytes_alg = 32 * n + (1 + width) * n + 2 * mask_bytes        # both operands in, flag + value out, the mask in and out
    hbm_ms = bytes_alg / HBM_PEAK * 1e3
    import tempfile
    with tempfile.TemporaryDirectory() as tmp:
        issue = issue_model(wl, tmp)
    clk = (clocks or {}).get("sm_mhz") or (card or {}).get("sm_max_mhz")
    if "path_instructions" in issue and clk:
        warp_instr = issue["path_instructions"] * (n / ROWS_PER_THREAD) / 32
        issue["bound_ms"] = warp_instr / (SMS * SUBPARTITIONS * clk * 1e6) * 1e3
        issue["clock_mhz"] = clk
        issue["achieved_frac"] = round(issue["bound_ms"] / ms, 4)
    print(json.dumps({
        "metric": f"rows_per_s_{key}", "value": n / (ms * 1e-3), "unit": "rows/s", "n_gpus": 1, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": ms, "ms_per_step_min": ms_min, "higher_is_better": True, "data": "synthetic",
        "config": {"workload": key, "rows": n, "scales": wl["scales"], "digits": wl["digits"], "nulls": NULLS},
        "algorithmic_bytes_per_sec": bytes_alg / (ms * 1e-3), "hbm_peak_frac": round(bytes_alg / (ms * 1e-3) / HBM_PEAK, 4),
        "models": {"note": "models, not measurements", "hbm": {"bytes": bytes_alg, "bound_ms": hbm_ms, "achieved_frac": round(hbm_ms / ms, 4)},
                   "issue": issue},
        "card": card, "cpu_baseline": cpu_baseline(wl, ha, hb, min(len(ha), 2000)), "clocks": clocks}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="mul", choices=sorted(WORKLOADS))
    ap.add_argument("--gpus", type=int, default=1, choices=[1])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rows", type=int, default=ROWS)
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be at least 1")
    run(args, args.workload)


if __name__ == "__main__":
    main()
