#!/usr/bin/env python
"""bench_c3_phases.py -- where the time of a C3 convert_from_rows batch goes, set against its byte floors.

    python bench_c3_phases.py [--passes P] [--warmup W] [--rows-per-batch N]

Builds the resident pool of C3 batches the way bench.py's run_c3 does (same seeds, same generators, same packed
output slabs) and reports, per batch:
  kernels : the device time of each kernel of the two C-ABI calls (from_rows_wide_kernel, wide_group_scan_kernel,
            strings_wide_kernel), from torch.profiler with CUDA activities, in a run of its own;
  calls   : srj_convert_from_rows_fixed (phase 1) and srj_convert_from_rows_strings (phase 2), CUDA events around each
            call, and the whole batch (events around `passes` passes over the pool, no profiler);
  floors  : the bytes each phase has to move, computed from the actual batches (exact row and chars bytes), over
            3.35 TB/s (H100 SXM data sheet) and 2.73 TB/s (what C2's from_rows reaches), and the fraction of each reached;
  card    : name, power limit and maximum SM clock (nvidia-smi, read in the same run).
Prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, os.path.join(ROOT, "spark-rapids-jni_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402

from bench import DEC128, SIZE, STRING, WORKLOADS, synth_columns_gpu, synth_strings_gpu  # noqa: E402
from bench_sha2 import card_info  # noqa: E402

DATASHEET_GBS = 3350.0
C2_FROM_ROWS_GBS = 2730.0
TMA_WINDOW = 16        # bytes a TMA row copy reads past its 16-byte-aligned ends, per row (upper bound of the rounding)
KERNELS = ("from_rows_wide_kernel", "wide_group_scan_kernel", "strings_wide_kernel")


def phase_bytes(types, nb, size_per_row, row_bytes, chars):
    """(phase 1, phase 2) bytes of one batch.  Phase 1 reads every row's fixed section (+ the TMA window) and writes
    the fixed-width data, the STRING offsets and the masks; phase 2 reads the variable sections (+ window), writes the
    chars, reads and rewrites the STRING offsets and reads the per-group bases."""
    nstr = sum(t == STRING for t in types)
    words = (nb + 31) // 32
    p1 = nb * (size_per_row + TMA_WINDOW)
    p1 += sum(nb * SIZE[t] for t in types if t != STRING) + nstr * 4 * (nb + 1) + len(types) * words * 4
    var = row_bytes - nb * size_per_row
    p2 = var + nb * TMA_WINDOW + chars + 2 * nstr * 4 * (nb + 1) + nstr * 4 * words
    return p1, p2


def run(args):
    import ctypes as C
    import torch
    import srj_b200 as S
    from srj_b200 import _native as N
    from srj_b200 import sharding

    torch.cuda.set_device(0)
    wl = WORKLOADS["c3"]
    types = wl["types"]
    nc = len(types)
    nb = int(args.rows_per_batch or wl["batch_rows"])
    pool = int(wl["pool"])
    dts = [S.DType(t, -11 if t == DEC128 else 0) for t in types]
    plan = S.Plan.get(dts)
    lib = N.lib()
    stream = torch.cuda.current_stream()
    st = int(stream.cuda_stream)
    g = torch.Generator(device="cuda").manual_seed(1234)
    words = (nb + 31) // 32

    # ---- the resident pool, as run_c3 builds it (rank 0) ------------------------------------------------------
    batches = []
    for b in range(pool):
        fixed = iter(synth_columns_gpu(torch, S, [t for t in types if t != STRING], nb, wl["null_frac"], seed=77 + 13 * b))
        cols = [synth_strings_gpu(torch, S, nb, wl["null_frac"], g) if t == STRING else next(fixed) for t in types]
        for c, d in zip(cols, dts):
            c.dtype = d
        rows = S.RowConversion.convertToRows(S.Table(cols))
        assert len(rows) == 1, "batch must fit one LIST column"
        batches.append(dict(cols=cols, rows=rows[0]))
    torch.cuda.synchronize()

    chars_need = [sum((c.data.numel() + 15) & ~15 for c in bt["cols"] if c.dtype.type_id == STRING) for bt in batches]
    lay = sharding.SlabLayout([0 if t == STRING else SIZE[t] for t in types], nb, max(chars_need))
    outs = []
    for bt in batches:
        slab = torch.empty(lay.nbytes, dtype=torch.uint8, device="cuda")
        o, co = [], lay.at_chars
        for i, c in enumerate(bt["cols"]):
            m = slab[lay.at_mask[i]: lay.at_mask[i] + words * 4].view(torch.int32)
            if c.dtype.type_id == STRING:
                offs = slab[lay.at_data[i]: lay.at_data[i] + (nb + 1) * 4].view(torch.int32)
                o.append(S.ColumnVector(c.dtype, nb, slab[co: co + c.data.numel()], m, offs))
                co += (c.data.numel() + 15) & ~15
            else:
                o.append(S.ColumnVector(c.dtype, nb, slab[lay.at_data[i]: lay.at_data[i] + c.data.numel()], m))
        carr = (N.SrjColumn * len(o))()
        for i, c in enumerate(o):
            carr[i] = c._c()
        outs.append(dict(cols=o, carr=carr, totals=slab[lay.at_totals: lay.at_totals + (nc + 1) * 8].view(torch.int64)))
    nulls = torch.zeros(nc, dtype=torch.int64, device="cuda")
    wsb = lib.srj_from_rows_workspace_bytes(plan.handle, nb)
    wss = [torch.empty(max(wsb, 8), dtype=torch.uint8, device="cuda") for _ in range(pool)]

    def fixed_call(k):
        rv, o = batches[k]["rows"], outs[k]
        N.check(lib.srj_convert_from_rows_fixed(plan.handle, rv.child.data.data_ptr(), rv.offsets.data_ptr(), rv.child.size,
                                                nb, o["carr"], nulls.data_ptr(), o["totals"].data_ptr(), None, wss[k].data_ptr(), st))

    def strings_call(k):
        rv, o = batches[k]["rows"], outs[k]
        N.check(lib.srj_convert_from_rows_strings(plan.handle, rv.child.data.data_ptr(), rv.offsets.data_ptr(), rv.child.size,
                                                  nb, o["carr"], o["totals"].data_ptr(), wss[k].data_ptr(), st))

    # correctness: every pool batch round-trips
    for k in range(pool):
        fixed_call(k)
        strings_call(k)
    torch.cuda.synchronize()
    for k in range(pool):
        for a, b in zip(outs[k]["cols"], batches[k]["cols"]):
            assert torch.equal(a.mask, b.mask) and torch.equal(a.data, b.data), "bench_c3_phases: round trip differs"
            if a.offsets is not None:
                assert torch.equal(a.offsets, b.offsets), "bench_c3_phases: offsets differ"

    for _ in range(args.warmup):
        for k in range(pool):
            fixed_call(k)
            strings_call(k)
    torch.cuda.synchronize()

    # ---- whole batch: events around `passes` passes over the pool ---------------------------------------------
    nbatch = args.passes * pool
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record(stream)
    for i in range(nbatch):
        fixed_call(i % pool)
        strings_call(i % pool)
    t1.record(stream)
    torch.cuda.synchronize()
    batch_ms = t0.elapsed_time(t1) / nbatch

    # ---- each call on its own: events around it, synchronised per batch --------------------------------------
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    acc = [0.0, 0.0]
    for i in range(nbatch):
        ev[0].record(stream)
        fixed_call(i % pool)
        ev[1].record(stream)
        strings_call(i % pool)
        ev[2].record(stream)
        torch.cuda.synchronize()
        acc[0] += ev[0].elapsed_time(ev[1])
        acc[1] += ev[1].elapsed_time(ev[2])
    call_ms = {"srj_convert_from_rows_fixed": acc[0] / nbatch, "srj_convert_from_rows_strings": acc[1] / nbatch}

    # ---- kernel times: torch.profiler, a run of its own -------------------------------------------------------
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        torch.zeros(1, device="cuda").add_(1)      # the activity buffer is in place before the first batch ends
        torch.cuda.synchronize()
        for i in range(nbatch):
            fixed_call(i % pool)
            strings_call(i % pool)
        torch.cuda.synchronize()
    kern_us, kern_n = {}, {}
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        for k in KERNELS:
            if k in e.name:
                kern_us[k] = kern_us.get(k, 0.0) + e.device_time
                kern_n[k] = kern_n.get(k, 0) + 1
    for k in KERNELS:
        assert kern_n.get(k, 0) > 0, f"bench_c3_phases: {k} did not run"
    # each kernel launches once per batch: the mean over the records received (the profiler can drop a few)
    kernels = {k: {"ms_per_batch": kern_us[k] / 1e3 / kern_n[k], "launches_recorded": kern_n[k]} for k in KERNELS}

    # ---- byte floors from the actual batches --------------------------------------------------------------------
    spr = plan.layout.size_per_row
    fl = [phase_bytes(types, nb, spr, bt["rows"].child.size,
                      sum(c.data.numel() for c in bt["cols"] if c.dtype.type_id == STRING)) for bt in batches]
    p1b, p2b = float(np.mean([f[0] for f in fl])), float(np.mean([f[1] for f in fl]))
    p1_ms = kernels["from_rows_wide_kernel"]["ms_per_batch"]
    p2_ms = kernels["wide_group_scan_kernel"]["ms_per_batch"] + kernels["strings_wide_kernel"]["ms_per_batch"]

    def floor(b, ms):
        f_ds, f_c2 = b / (DATASHEET_GBS * 1e9) * 1e3, b / (C2_FROM_ROWS_GBS * 1e9) * 1e3
        return {"bytes_per_batch": b, "bytes_per_row": b / nb, "floor_ms_3350": f_ds, "floor_ms_2730": f_c2,
                "kernel_ms": ms, "frac_of_3350_floor": f_ds / ms if ms else None, "x_floor_2730": ms / f_c2 if f_c2 else None}

    print(json.dumps({
        "workload": wl["name"], "rows_per_batch": nb, "pool": pool, "batches_timed": nbatch, "size_per_row": spr,
        "batch_ms": batch_ms, "calls_ms": call_ms, "kernels": kernels,
        "phase1_from_rows_wide": floor(p1b, p1_ms), "phase2_scan_plus_gather": floor(p2b, p2_ms),
        "card": card_info(), "lib": N.LIB_PATH}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passes", type=int, default=25, help="passes over the pool of 4 batches per measurement")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rows-per-batch", type=int, default=0, help="override the batch size (development only)")
    args = ap.parse_args()
    run(args)


if __name__ == "__main__":
    main()
