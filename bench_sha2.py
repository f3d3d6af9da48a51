#!/usr/bin/env python
"""bench_sha2.py -- benchmark of Hash.sha{224,256,384,512}NullsPreserved on one GPU.

    python bench_sha2.py [--workload sha2|sha2_skew] [--digest 224|256|384|512] [--steps K] [--warmup W]
                         [--rows R] [--dump-outputs DIR]

A step is the two C-ABI calls of one column: srj_sha2_sizes (output offsets + chars total; with a null mask a popcount,
a scan and one read-back) and srj_sha2_hash (mask copy + hash kernel), input resident in HBM, outputs preallocated,
CUDA events around each step.  Prints one JSON line: rows/s, input bytes/s, compression blocks/s, an integer-pipe bound
computed from the block count (a model, not a measurement), the card and its power limit, and a one-core hashlib
baseline.  --dump-outputs DIR writes a seeded row sample of the digests plus whole-output checksums (float .npy files),
so that two builds can be compared output for output.  Shares its measurement helpers with bench.py.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, os.path.join(ROOT, "spark-rapids-jni_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402

from bench import STRING, ClockSampler, byte_sum, gather_lists, sample_rows, valid_count, write_dump  # noqa: E402

WORKLOADS = {
    # 16M rows: SHA-512's 128-char output of every valid row stays under the 2 GiB of one STRING column
    "sha2": dict(name="SHA-2 nulls preserved: 16M-row STRING column, lengths ~N(16,8) in [0,32] B, 20% nulls",
                 rows=16_000_000, null_frac=0.2, long_frac=0.0),
    # the lane-balance case: a warp runs as long as its longest row
    "sha2_skew": dict(name="SHA-2 nulls preserved, skewed: 16M-row STRING column, lengths ~N(16,8) in [0,32] B, 20% nulls, "
                           "1% of the rows 4 KB strings", rows=16_000_000, null_frac=0.2, long_frac=0.01, long_len=4096),
}

# SASS instructions of the block loop of the SHA kernels (cuobjdump -sass of sha256_kernel / sha512_kernel, sm_90a, CUDA 12.9):
# all of them integer-pipe work (SHF, LOP3, IADD3, PRMT, ...), so blocks/s <= SMs x 64 integer lanes x SM clock / this.
SHA2_LOOP_INSTRS = {256: 1750, 512: 4295}


def sha2_blocks(lens, valid, bits):
    """compression blocks of every valid row: message + 0x80 + the 8- (SHA-224/256) or 16-byte (SHA-384/512) length"""
    blk, lenb = (64, 8) if bits <= 256 else (128, 16)
    return int((((lens + lenb) // blk + 1) * valid).sum())


def card_info():
    """name, power limit (W) and maximum SM clock of GPU 0 as nvidia-smi reports them (read-only query)"""
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"name": out[0].strip(), "power_limit_w": float(out[1]), "sm_max_mhz": float(out[2])}
    except Exception as e:
        return {"name": None, "power_limit_w": None, "sm_max_mhz": None, "error": repr(e)}


def cpu_baseline_sha2(bits, h_lens, h_valid, n_sample, seed=7):
    """hashlib (OpenSSL) on one core over a bounded sample of rows of the same length distribution: digest + hex per row,
    the work one row of the GPU step does"""
    import hashlib
    rng = np.random.default_rng(seed)
    idx = rng.integers(0, len(h_lens), n_sample)
    rows = [rng.integers(32, 127, int(h_lens[i]), dtype=np.uint8).tobytes() if h_valid[i] else None for i in idx]
    name = f"sha{bits}"

    def once():
        return [hashlib.new(name, r).hexdigest() if r is not None else None for r in rows]

    once()
    times = []
    while sum(times) < 5.0 and len(times) < 10:
        t0 = time.perf_counter()
        once()
        times.append(time.perf_counter() - t0)
    best = min(times)
    return {"value": n_sample / best, "unit": "rows/s", "cores": 1, "kind": "library",
            "sample": f"{n_sample} rows drawn from the same workload, best of {len(times)} passes, one core: python hashlib "
                      f"(OpenSSL) {name} + hexdigest per row", "ms_per_pass": best * 1e3}


def run(args, wl):
    import ctypes as C
    import hashlib
    import torch
    import srj_b200 as S
    from srj_b200 import _native as N
    torch.cuda.set_device(0)
    bits = args.digest
    width = bits // 4
    n = int(args.rows or wl["rows"])
    g = torch.Generator(device="cuda").manual_seed(42)
    valid = torch.rand(n, device="cuda", generator=g) >= wl["null_frac"]
    lens = torch.clamp(torch.round(torch.randn(n, device="cuda", generator=g) * 8 + 16), 0, 32).to(torch.int64)
    if wl["long_frac"] > 0:
        lens = torch.where(torch.rand(n, device="cuda", generator=g) < wl["long_frac"], wl["long_len"], lens)
    lens = lens * valid
    offs = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    offs[1:] = torch.cumsum(lens, 0)
    in_bytes = int(offs[-1])
    chars = torch.empty(in_bytes, dtype=torch.uint8, device="cuda")
    for o in range(0, in_bytes, 1 << 28):
        m = min(1 << 28, in_bytes - o)
        chars[o:o + m] = torch.randint(32, 127, (m,), dtype=torch.uint8, device="cuda", generator=g)
    words = (n + 31) // 32
    bitsv = torch.cat([valid, torch.zeros(words * 32 - n, dtype=torch.bool, device="cuda")]).view(words, 32).to(torch.int64)
    w = (bitsv * (1 << torch.arange(32, device="cuda", dtype=torch.int64))).sum(dim=1)
    mask = torch.where(w >= 2**31, w - 2**32, w).to(torch.int32)
    col = S.ColumnVector(S.DType(STRING), n, chars, mask, offs.to(torch.int32))
    h_lens, h_valid = lens.cpu().numpy(), valid.cpu().numpy()
    n_valid = int(h_valid.sum())
    blocks = sha2_blocks(h_lens, h_valid, bits)
    del lens, offs, bitsv, w

    lib = N.lib()
    out_offs = torch.empty(n + 1, dtype=torch.int32, device="cuda")
    out_chars = torch.empty(n_valid * width, dtype=torch.uint8, device="cuda")
    out_mask = torch.empty(words, dtype=torch.int32, device="cuda")
    ws = torch.empty(max(lib.srj_sha2_workspace_bytes(n), 8), dtype=torch.uint8, device="cuda")
    cin = col._c()
    cout = S.ColumnVector(S.DType(STRING), n, out_chars, out_mask, out_offs)._c()
    total = C.c_int64(0)
    stream = torch.cuda.current_stream()
    st = int(stream.cuda_stream)

    def step():
        N.check(lib.srj_sha2_sizes(bits, C.byref(cin), out_offs.data_ptr(), C.byref(total), ws.data_ptr(), st))
        N.check(lib.srj_sha2_hash(bits, C.byref(cin), C.byref(cout), st))

    # correctness gate: the chars total, the mask, and the digests of a sample of rows against hashlib
    step()
    torch.cuda.synchronize()
    assert total.value == n_valid * width and torch.equal(out_mask, mask), "bench_sha2: sizes / mask mismatch"
    idx = sample_rows(n, seed=5)[:256]
    h_in_offs = col.offsets[torch.from_numpy(np.concatenate([idx, idx + 1])).cuda()].cpu().numpy()
    h_out_offs = out_offs[torch.from_numpy(idx).cuda()].cpu().numpy()
    for k, r in enumerate(idx):
        if h_valid[r]:
            src = chars[int(h_in_offs[k]):int(h_in_offs[k + len(idx)])].cpu().numpy().tobytes()
            got = out_chars[int(h_out_offs[k]):int(h_out_offs[k]) + width].cpu().numpy().tobytes()
            assert got == hashlib.new(f"sha{bits}", src).hexdigest().encode(), f"bench_sha2: row {r} differs from hashlib"

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
    if args.dump_outputs:
        arrays = {}
        idx_np = sample_rows(n)
        arrays["sample_rows"] = idx_np.astype(np.float64)
        arrays["digest_len"], arrays["digest_chars"] = gather_lists(torch, out_offs, out_chars, torch.from_numpy(idx_np).cuda())
        arrays["chars_byte_sum"] = np.array([byte_sum(torch, out_chars)])
        arrays["offsets_byte_sum"] = np.array([byte_sum(torch, out_offs)])
        arrays["valid_count"] = np.array([valid_count(torch, out_mask, n)])
        write_dump(args.dump_outputs, arrays)
    card = card_info()
    sm_mhz = clocks.get("sm_mhz") or card.get("sm_max_mhz") or 1980.0
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    loop = SHA2_LOOP_INSTRS[256 if bits <= 256 else 512]
    bound_blocks_s = nsm * 64 * sm_mhz * 1e6 / loop
    print(json.dumps({
        "metric": f"rows_per_sec_sha{bits}_nulls_preserved", "value": n / (ms * 1e-3), "unit": "rows/s", "n_gpus": 1, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": ms, "higher_is_better": True, "dtype": "u8", "data": "synthetic",
        "config": {"workload": wl["name"], "digest_bits": bits, "rows": n, "valid_rows": n_valid, "input_chars": in_bytes,
                   "output_chars": n_valid * width, "compression_blocks": blocks,
                   "step": "srj_sha2_sizes (mask popcount + scan + one read-back + offsets) + srj_sha2_hash (mask copy + hash kernel)"},
        "input_bytes_per_sec": in_bytes / (ms * 1e-3), "blocks_per_sec": blocks / (ms * 1e-3),
        "int_pipe_model": {"note": "a model, not a measurement: blocks/s <= SMs x 64 integer lanes/clk x SM clock / SASS instructions of "
                                   "the kernel's block loop", "sass_instrs_per_block": loop, "sms": nsm, "sm_mhz": sm_mhz,
                           "bound_blocks_per_sec": bound_blocks_s, "bound_ms": blocks / bound_blocks_s * 1e3,
                           "achieved_frac": round(blocks / (ms * 1e-3) / bound_blocks_s, 4)},
        "card": card, "cpu_baseline": cpu_baseline_sha2(bits, h_lens, h_valid, 200_000), "clocks": clocks}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="sha2", choices=sorted(WORKLOADS))
    ap.add_argument("--digest", type=int, default=256, choices=[224, 256, 384, 512])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rows", type=int, default=0, help="override the row count (development only)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write a seeded sample of the digests plus checksums as DIR/<name>.npy")
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be at least 1")
    run(args, WORKLOADS[args.workload])


if __name__ == "__main__":
    main()
