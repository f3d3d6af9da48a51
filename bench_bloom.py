#!/usr/bin/env python
"""bench_bloom.py -- benchmark of BloomFilter (Spark's runtime-join bloom filter) on one GPU.

    python bench_bloom.py [--workload bloom_probe|bloom_put|bloom_merge] [--version 1|2] [--steps K] [--warmup W]
                          [--dump-outputs DIR]

Workloads (V1 filters by default, --version 2 for V2):
  bloom_probe  the hot path, BloomFilterMightContain: a filter sized by Spark's rule for 4,000,000 expected items at fpp
               0.03 (optimalNumOfBits = 29,193,763 bits = 456,153 longs = 3,649,224 B; k = 5), built from 4M keys; a step
               probes 200M INT64 keys of which 10% are present.  No nulls: Spark probes xxhash64 values, never null.
  bloom_put    BloomFilterAggregate's update: a step puts 50M keys into a 67,108,864-bit (8 MB, Spark's maxNumBits)
               filter, k = 5.
  bloom_merge  BloomFilterAggregate's merge: a step ORs 200 partial filters of the bloom_probe size (3.6 MB each).
A step is the one C-ABI call (srj_bloom_filter_probe / _put / _merge, each with its one 16-byte header read-back), inputs
resident in HBM, outputs preallocated, CUDA events around each step.  Prints one JSON line: rows/s (filters/s for merge),
algorithmic bytes/s and their share of the H100 SXM data-sheet HBM3 bandwidth, the models below, the card and its power
limit read in the same run, and a one-core numpy-oracle baseline on a sample.  Models (computed, not measured):
  HBM     : probe 8 B in + 1 B out per row; put 8 B in per row; merge F filters in + 1 out.
  L2      : each of the k bit positions of a row is one 32-byte sector request to the L2-resident filter; the achieved
            request rate is reported per SM and clock.
  issue   : SMs x 4 warp instructions / clock x SM clock over the kernel's SASS instructions per row.
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
PROBE_BITS, PROBE_K, PROBE_ITEMS = 29_193_763, 5, 4_000_000
WORKLOADS = {
    "bloom_probe": dict(name="probe 200M INT64 keys (10% present) against a 29,193,763-bit k=5 filter built from 4M keys",
                        rows=200_000_000, bits=PROBE_BITS, k=PROBE_K, build=PROBE_ITEMS, present=0.10),
    "bloom_put": dict(name="put 50M INT64 keys into a 67,108,864-bit (8 MB) k=5 filter", rows=50_000_000, bits=67_108_864, k=5),
    "bloom_merge": dict(name="merge 200 partial 29,193,763-bit k=5 filters (3.6 MB each)", filters=200, bits=PROBE_BITS, k=PROBE_K),
}
# SASS instructions of one thread of the put / probe kernels (4 rows, cuobjdump -sass, sm_90a, CUDA 12.9), whole kernel
# body: an upper bound on what runs for k <= 8 (one 8-hash chunk) per 4 rows
SASS_INSTRS_PER_THREAD = {("bloom_probe", 1): 1248, ("bloom_probe", 2): 1832, ("bloom_put", 1): 864, ("bloom_put", 2): 1392}


def cpu_baseline(wl_key, version, wl, filt_host, n_sample=1_000_000):
    """oracle/bloom.py (numpy, one core) on a sample of the same work"""
    from oracle import bloom as B
    rng = np.random.default_rng(3)
    times = []
    if wl_key == "bloom_merge":
        parts = [filt_host] * 20
        work, unit = 20, "filters/s"
        fn = lambda: B.merge(parts)                                        # noqa: E731
    else:
        keys = rng.integers(-2**63, 2**63 - 1, n_sample, dtype=np.int64)
        work, unit = n_sample, "rows/s"
        fn = (lambda: B.probe(filt_host, keys)) if wl_key == "bloom_probe" else (lambda: B.put(filt_host, keys))  # noqa: E731
    fn()
    while sum(times) < 5.0 and len(times) < 5:
        t0 = time.perf_counter()
        fn()
        times.append(time.perf_counter() - t0)
    best = min(times)
    return {"value": work / best, "unit": unit, "cores": 1, "kind": "numpy oracle (oracle/bloom.py)",
            "sample": f"{work} {unit.split('/')[0]}, best of {len(times)} passes"}


def run(args, wl_key):
    import ctypes as C
    import torch
    import srj_b200 as S
    from srj_b200 import _native as N
    from srj_b200.bloom import BloomFilter, list_column
    torch.cuda.set_device(0)
    wl = WORKLOADS[wl_key]
    version = args.version
    lib = N.lib()
    stream = torch.cuda.current_stream()
    st = int(stream.cuda_stream)
    g = torch.Generator(device="cuda").manual_seed(42)

    def rand_keys(n):                       # uniform over all 64-bit values
        w = torch.randint(0, 2**32, (2, n), dtype=torch.int64, device="cuda", generator=g)
        return (w[0] << 32) | w[1]

    def col(keys):
        return S.ColumnVector(S.DType.INT64, keys.numel(), keys.view(torch.uint8))

    filt = BloomFilter.create(version, wl["k"], wl["bits"], 0)
    arrays = {}
    if wl_key == "bloom_probe":
        n = wl["rows"]
        build = rand_keys(wl["build"])
        BloomFilter.put(filt, col(build))
        keys = rand_keys(n)
        present = torch.rand(n, device="cuda", generator=g) < wl["present"]
        keys = torch.where(present, build[torch.randint(0, wl["build"], (n,), device="cuda", generator=g)], keys)
        del present
        out = torch.empty(n, dtype=torch.uint8, device="cuda")
        cin = col(keys)._c()

        def step():
            N.check(lib.srj_bloom_filter_probe(filt.data.data_ptr(), filt.data.numel(), C.byref(cin), out.data_ptr(), None, st))
        work, bytes_alg, sectors = n, 9 * n, n * wl["k"]
    elif wl_key == "bloom_put":
        n = wl["rows"]
        keys = rand_keys(n)
        cin = col(keys)._c()

        def step():
            N.check(lib.srj_bloom_filter_put(filt.data.data_ptr(), filt.data.numel(), C.byref(cin), st))
        work, bytes_alg, sectors = n, 8 * n, n * wl["k"]
    else:
        F = wl["filters"]
        parts = []
        for i in range(F):
            f = BloomFilter.create(version, wl["k"], wl["bits"], 0)
            BloomFilter.put(f, col(rand_keys(20_000)))
            parts.append(f)
        lc = list_column(parts)
        size = parts[0].data.numel()
        child = lc.child.data
        del parts
        out = torch.empty(size, dtype=torch.uint8, device="cuda")
        ws = torch.empty(lib.srj_bloom_filter_merge_workspace_bytes(), dtype=torch.uint8, device="cuda")

        def step():
            N.check(lib.srj_bloom_filter_merge(child.data_ptr(), child.numel(), F, out.data_ptr(), ws.data_ptr(), st))
        work, bytes_alg, sectors = F, (F + 1) * size, 0

    # correctness gate against the oracle before timing
    from oracle import bloom as B
    step()
    torch.cuda.synchronize()
    if wl_key == "bloom_probe":
        idx = torch.from_numpy(sample_rows(n, seed=5)).cuda()
        want = B.probe(filt.data.cpu().numpy(), keys[idx].cpu().numpy())
        assert np.array_equal(out[idx].cpu().numpy().astype(bool), want), "bench_bloom: probe differs from the oracle"
    elif wl_key == "bloom_put":
        sub = keys[:1_000_000].cpu().numpy()
        assert B.probe(filt.data.cpu().numpy(), sub).all(), "bench_bloom: a key put is not found"
    else:
        h = child.cpu().numpy()
        want = B.merge(list(h.reshape(F, size)))
        assert np.array_equal(out.cpu().numpy(), want), "bench_bloom: merge differs from the oracle"

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
        res = out if wl_key != "bloom_put" else filt.data
        idx_np = sample_rows(res.numel())
        arrays["sample_rows"] = idx_np.astype(np.float64)
        arrays["sample_bytes"] = res[torch.from_numpy(idx_np).cuda()].cpu().numpy().astype(np.float64)
        arrays["byte_sum"] = np.array([byte_sum(torch, res)])
        arrays["filter_byte_sum"] = np.array([byte_sum(torch, filt.data)])
        write_dump(args.dump_outputs, arrays)
    card = card_info()
    sm_mhz = clocks.get("sm_mhz") or card.get("sm_max_mhz") or 1980.0
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    sec = ms * 1e-3
    hbm_ms = bytes_alg / HBM_PEAK * 1e3
    models = {"note": "models, not measurements",
              "hbm": {"bytes": bytes_alg, "bound_ms": hbm_ms, "achieved_frac": round(hbm_ms / ms, 4)}}
    if sectors:
        models["l2"] = {"sector_requests": sectors, "requests_per_sm_per_clk": round(sectors / sec / nsm / (sm_mhz * 1e6), 4)}
        instrs = SASS_INSTRS_PER_THREAD[(wl_key, version)] / 4 * work
        issue_ms = instrs / (nsm * 128 * sm_mhz * 1e6) * 1e3
        models["issue"] = {"sass_instrs_per_row": SASS_INSTRS_PER_THREAD[(wl_key, version)] / 4, "sms": nsm, "sm_mhz": sm_mhz,
                           "bound_ms": issue_ms, "achieved_frac": round(issue_ms / ms, 4)}
    bound = max((m for m in ("hbm", "issue") if m in models), key=lambda m: models[m]["bound_ms"])
    unit = "filters/s" if wl_key == "bloom_merge" else "rows/s"
    print(json.dumps({
        "metric": f"{unit.replace('/', '_per_')}_{wl_key}_v{version}", "value": work / sec, "unit": unit, "n_gpus": 1,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms, "ms_per_step_min": ms_min, "higher_is_better": True,
        "data": "synthetic", "config": {"workload": wl["name"], "version": version, "k": wl["k"], "bits": wl["bits"],
                                         "filter_bytes": int(filt.data.numel())},
        "algorithmic_bytes_per_sec": bytes_alg / sec, "hbm_peak_frac": round(bytes_alg / sec / HBM_PEAK, 4),
        "models": models, "model_bound": bound, "card": card,
        "cpu_baseline": cpu_baseline(wl_key, version, wl, filt.data.cpu().numpy()), "clocks": clocks}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="bloom_probe", choices=sorted(WORKLOADS))
    ap.add_argument("--version", type=int, default=1, choices=[1, 2])
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
