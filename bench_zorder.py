#!/usr/bin/env python
"""bench_zorder.py -- benchmark of ZOrder (Delta Lake's InterleaveBits and Hilbert clustering) on one GPU.

    python bench_zorder.py [--workload interleave|interleave_wide|interleave_direct|hilbert|hilbert_2x32] [--steps K]
                           [--warmup W] [--dump-outputs DIR]

Workloads:
  interleave         OPTIMIZE ... ZORDER BY over four INT32 columns, Delta's case: 100M rows, 10% nulls in each column;
                     16-byte rows, 1.6 GB of output.
  interleave_wide    8M rows x 16 INT64 columns: 128-byte rows, the widest rows staged in shared memory.
  interleave_direct  4M rows x 64 INT32 columns: 256-byte rows, past the staging threshold (rows written directly).
  hilbert            100M rows x 3 INT32 columns at 21 bits (a 63-bit index), 10% nulls.
  hilbert_2x32       100M rows x 2 INT32 columns at 32 bits.
A step is the one C-ABI call (srj_interleave_bits / srj_hilbert_index), inputs resident in HBM, outputs preallocated,
CUDA events around each step.  Prints one JSON line: rows/s, algorithmic bytes/s and their share of the H100 SXM
data-sheet HBM3 bandwidth, the issue model, the card and its power limit read in the same run, the SM clock sampled
during the run, and a one-core numpy-oracle baseline on a sample.  Models (computed, not measured):
  HBM    : interleave: values + null masks in, bytes + int32 offsets out; hilbert: values + masks in, 8 B out per row.
  issue  : SMs x 4 warp instructions / clock x SM clock, over the SASS instructions a row executes, counted from
           cuobjdump -sass of the sm_90a build (CUDA 12.9) along the row's path (see IL_STEP / HB below).
--dump-outputs DIR writes a seeded sample of the output plus whole-output checksums (float .npy files).  Shares its
measurement helpers with bench.py.
"""
from __future__ import annotations

import argparse
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
INT32, INT64 = 3, 4
WORKLOADS = {
    "interleave": dict(name="interleaveBits, 100M rows x 4 INT32, 10% nulls", kind="interleave", rows=100_000_000, ncols=4,
                       type_id=INT32, width=4, nulls=0.10),
    "interleave_wide": dict(name="interleaveBits, 8M rows x 16 INT64", kind="interleave", rows=8_000_000, ncols=16,
                            type_id=INT64, width=8, nulls=None),
    "interleave_direct": dict(name="interleaveBits, 4M rows x 64 INT32", kind="interleave", rows=4_000_000, ncols=64,
                              type_id=INT32, width=4, nulls=None),
    "hilbert": dict(name="hilbertIndex, 100M rows x 3 INT32 at 21 bits, 10% nulls", kind="hilbert", rows=100_000_000, ncols=3,
                    bits=21, nulls=0.10),
    "hilbert_2x32": dict(name="hilbertIndex, 100M rows x 2 INT32 at 32 bits", kind="hilbert", rows=100_000_000, ncols=2, bits=32,
                         nulls=None),
}
# SASS instructions a row executes, counted from cuobjdump -sass of the sm_90a build (CUDA 12.9) along the path the row
# takes (predicated-off instructions still issue; not-taken branches cost their own instruction only).
#   interleave_bits_kernel<4> and <8> (identical loop layout; the value loop is unrolled 2x, 144 instructions):
#     step   one (output word, value) pass of interleave_word: 72 with a mask and a valid row, 57 with a null row,
#            66 without a mask.  It reloads the column pointers (indexed constant loads), the mask word and the value,
#            and runs all 5 predicated dilation steps whatever N is.
#     word   per output word outside the value loop: 67 staged (rows <= 128 B, one STS) / 76 direct (one STG)
#     row    staged: 77 (offsets, set-up) + 59 (copy-out set-up) + 9 per 16-byte store of the lane; direct: 80
#   hilbert_index_kernel (N = 2 or 3, the workloads):
#     load   21 + 9 + 37 per column (mask and value loads)
#     undo   per bit q (numBits - 1 of them): 32 at N = 2, 45 at N = 3 (the axis loop's remainder path)
#     gray   25 at N = 2, 37 at N = 3;  t   20 + 6.5 per bit;  xor   20 at N = 2, 30 at N = 3
#     word   per output word: 20 set-up + 50 per value (2x-unrolled loop, 101 for two) + 59 for an odd remainder value
#     store  15
IL_STEP = {"mask_valid": 72, "mask_null": 57, "nomask": 66}
IL_WORD = {"staged": 67, "direct": 76}
HB = {"undo": {2: 32, 3: 45}, "gray": {2: 25, 3: 37}, "xor": {2: 20, 3: 30}}


def issue_instrs_per_row(wl):
    n = wl["ncols"]
    if wl["kind"] == "interleave":
        rb = n * wl["width"]
        words = (rb + 3) // 4
        f = wl["nulls"] or 0.0
        step = (1 - f) * IL_STEP["mask_valid"] + f * IL_STEP["mask_null"] if wl["nulls"] else IL_STEP["nomask"]
        staged = rb <= 128
        row = 77 + 59 + 9 * -(-32 * rb // 512) if staged else 80
        return words * (min(n, 32) * step + IL_WORD["staged" if staged else "direct"]) + row
    b = wl["bits"]
    words = (n * b + 31) // 32
    word = 20 + 50 * (n // 2 * 2) + (59 if n % 2 else 0)
    return (21 + 9 + 37 * n + (b - 1) * HB["undo"][n] + HB["gray"][n] + 20 + 6.5 * (b - 1) + HB["xor"][n] + words * word
            + 15)


def cpu_baseline(wl, hosts, n_sample):
    """oracle/zorder.py (numpy, one core) on a sample of the same work"""
    from oracle import zorder as Z
    if wl["kind"] == "interleave":
        fn = lambda: Z.interleave_bits(hosts, wl["width"], n_sample)      # noqa: E731
    else:
        fn = lambda: Z.hilbert_index(wl["bits"], hosts, n_sample)         # noqa: E731
    fn()
    times = []
    while sum(times) < 5.0 and len(times) < 5:
        t0 = time.perf_counter()
        fn()
        times.append(time.perf_counter() - t0)
    best = min(times)
    return {"value": n_sample / best, "unit": "rows/s", "cores": 1, "kind": "numpy oracle (oracle/zorder.py)",
            "sample": f"{n_sample} rows, best of {len(times)} passes"}


def run(args, wl_key):
    import torch
    import srj_b200 as S
    from srj_b200 import _native as N
    from oracle import zorder as Z
    torch.cuda.set_device(0)
    wl = WORKLOADS[wl_key]
    lib = N.lib()
    stream = torch.cuda.current_stream()
    st = int(stream.cuda_stream)
    g = torch.Generator(device="cuda").manual_seed(42)
    n, ncols = wl["rows"], wl["ncols"]
    width = wl.get("width", 4)
    type_id = wl.get("type_id", INT32)

    cols = []
    for _ in range(ncols):
        data = torch.randint(0, 256, (n * width,), dtype=torch.uint8, device="cuda", generator=g)
        mask = None
        if wl["nulls"]:
            valid = torch.rand(n + (-n % 32), device="cuda", generator=g) >= wl["nulls"]
            w = (valid.view(-1, 32).to(torch.int64) << torch.arange(32, device="cuda", dtype=torch.int64)).sum(1)
            mask = torch.where(w >= 2**31, w - 2**32, w).to(torch.int32)
            del valid, w
        cols.append(S.ColumnVector(S.DType(type_id), n, data, mask))
    carr = S._carray(cols)
    mask_bytes = sum(4 * ((n + 31) // 32) for c in cols if c.mask is not None)
    if wl["kind"] == "interleave":
        total = n * ncols * width
        offs = torch.empty(n + 1, dtype=torch.int32, device="cuda")
        out = torch.empty(total, dtype=torch.uint8, device="cuda")

        def step():
            N.check(lib.srj_interleave_bits(carr, ncols, n, offs.data_ptr(), out.data_ptr(), st))
        bytes_alg = n * ncols * width + mask_bytes + total + 4 * (n + 1)
    else:
        out = torch.empty(n, dtype=torch.int64, device="cuda")

        def step():
            N.check(lib.srj_hilbert_index(wl["bits"], carr, ncols, n, out.data_ptr(), st))
        bytes_alg = n * ncols * 4 + mask_bytes + 8 * n

    # correctness gate against the oracle before timing, on the first rows and on a 32-row-aligned slice in the middle
    step()
    torch.cuda.synchronize()
    n_sample = min(n, 1_000_000)
    for s in (0, (n // 2) & ~31):
        e = min(n, s + n_sample // 4)
        hosts = [(c.data[s * width:e * width].cpu().numpy(),
                  None if c.mask is None else c.mask[s // 32:(e + 31) // 32].cpu().numpy().view(np.uint32)) for c in cols]
        if wl["kind"] == "interleave":
            rb = ncols * width
            _, want = Z.interleave_bits(hosts, width, e - s)
            assert np.array_equal(out[s * rb:e * rb].cpu().numpy(), want), "bench_zorder: bytes differ from the oracle"
            assert np.array_equal(offs[s:e + 1].cpu().numpy().astype(np.int64), np.arange(s, e + 1, dtype=np.int64) * rb)
        else:
            assert np.array_equal(out[s:e].cpu().numpy(), Z.hilbert_index(wl["bits"], hosts, e - s)), \
                "bench_zorder: index differs from the oracle"

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
        res = out.view(torch.uint8)
        idx_np = sample_rows(res.numel())
        arrays["sample_rows"] = idx_np.astype(np.float64)
        arrays["sample_bytes"] = res[torch.from_numpy(idx_np).cuda()].cpu().numpy().astype(np.float64)
        arrays["byte_sum"] = np.array([byte_sum(torch, res)])
        write_dump(args.dump_outputs, arrays)
    card = card_info()
    sm_mhz = clocks.get("sm_mhz") or card.get("sm_max_mhz") or 1980.0
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    sec = ms * 1e-3
    hbm_ms = bytes_alg / HBM_PEAK * 1e3
    ipr = issue_instrs_per_row(wl)
    issue_ms = ipr * n / 32 / (nsm * 4 * sm_mhz * 1e6) * 1e3
    models = {"note": "models, not measurements",
              "hbm": {"bytes": bytes_alg, "bound_ms": hbm_ms, "achieved_frac": round(hbm_ms / ms, 4)},
              "issue": {"sass_instrs_per_row": ipr, "sms": nsm, "sm_mhz": sm_mhz, "bound_ms": issue_ms,
                        "achieved_frac": round(issue_ms / ms, 4)}}
    bound = max(("hbm", "issue"), key=lambda m: models[m]["bound_ms"])
    hosts_sample = [(c.data[: n_sample * width].cpu().numpy(), None if c.mask is None else c.mask[: (n_sample + 31) // 32].cpu().numpy())
                    for c in cols]
    print(json.dumps({
        "metric": f"rows_per_s_{wl_key}", "value": n / sec, "unit": "rows/s", "n_gpus": 1, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": ms, "ms_per_step_min": ms_min, "higher_is_better": True, "data": "synthetic",
        "config": {"workload": wl["name"], "rows": n, "columns": ncols},
        "algorithmic_bytes_per_sec": bytes_alg / sec, "hbm_peak_frac": round(bytes_alg / sec / HBM_PEAK, 4),
        "models": models, "model_bound": bound, "card": card,
        "cpu_baseline": cpu_baseline(wl, hosts_sample, n_sample), "clocks": clocks}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="interleave", choices=sorted(WORKLOADS))
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
