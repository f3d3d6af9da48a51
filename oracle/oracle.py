"""ctypes/numpy front-end of the CPU oracle (TEST INFRASTRUCTURE -- see srj_oracle.c header).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this module.  The product package (spark-rapids-jni_b200/srj_b200) never does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from dataclasses import dataclass
from typing import List, Optional, Sequence

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libsrj_oracle.so")
_SRC = os.path.join(_HERE, "srj_oracle.c")

# cudf type ids (thirdparty/cudf/cpp/include/cudf/types.hpp:191-224)
(EMPTY, INT8, INT16, INT32, INT64, UINT8, UINT16, UINT32, UINT64, FLOAT32, FLOAT64, BOOL8,
 TIMESTAMP_DAYS, TIMESTAMP_SECONDS, TIMESTAMP_MILLISECONDS, TIMESTAMP_MICROSECONDS,
 TIMESTAMP_NANOSECONDS, DURATION_DAYS, DURATION_SECONDS, DURATION_MILLISECONDS,
 DURATION_MICROSECONDS, DURATION_NANOSECONDS, DICTIONARY32, STRING, LIST, DECIMAL32, DECIMAL64,
 DECIMAL128, STRUCT) = range(29)


def build(force: bool = False) -> str:
    """Compile srj_oracle.c -> libsrj_oracle.so (system gcc; see Makefile for why not $CC)."""
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(_SRC):
        subprocess.check_call(["make", "-C", _HERE, "-B", "libsrj_oracle.so"],
                              stdout=subprocess.DEVNULL)
    return _SO


class _OrcCol(C.Structure):
    _fields_ = [("type_id", C.c_int32), ("scale", C.c_int32), ("size", C.c_int64),
                ("data", C.c_void_p), ("null_mask", C.c_void_p), ("offsets", C.c_void_p)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        _lib.orc_xxh64_bytes.restype = C.c_uint64
        _lib.orc_xxh64_bytes.argtypes = [C.c_void_p, C.c_int64, C.c_uint64]
        _lib.orc_murmur3_bytes.restype = C.c_uint32
        _lib.orc_murmur3_bytes.argtypes = [C.c_void_p, C.c_int32, C.c_uint32]
    return _lib


def size_of(t: int) -> int:
    return lib().orc_size_of(int(t))


@dataclass
class HCol:
    """Host column: the cudf column_view fields the path reads, as numpy arrays."""
    type_id: int
    data: Optional[np.ndarray]            # fixed width: typed or uint8 array; STRING: uint8 chars
    mask: Optional[np.ndarray] = None     # uint32 words, bit i%32 of word i/32, 1 = valid
    offsets: Optional[np.ndarray] = None  # STRING / LIST: int32[size+1]
    scale: int = 0
    size: int = -1
    children: Optional[list] = None       # LIST: [element column]; STRUCT: the fields

    def __post_init__(self):
        if self.size < 0:
            if self.type_id in (STRING, LIST):
                self.size = len(self.offsets) - 1
            elif self.type_id == STRUCT:
                self.size = self.children[0].size if self.children else 0
            else:
                self.size = (self.data.nbytes // size_of(self.type_id)) if self.data is not None else 0

    def valid(self) -> np.ndarray:
        if self.mask is None:
            return np.ones(self.size, dtype=bool)
        bits = np.unpackbits(self.mask.view(np.uint8), bitorder="little")[: self.size]
        return bits.astype(bool)

    def null_count(self) -> int:
        return int(self.size - self.valid().sum())


def pack_mask(valid: np.ndarray) -> np.ndarray:
    n = len(valid)
    words = (n + 31) // 32
    b = np.zeros(words * 32, dtype=np.uint8)
    b[:n] = valid.astype(np.uint8)
    return np.packbits(b, bitorder="little").view(np.uint32).copy()


def strings_col(values: Sequence[Optional[bytes]]) -> HCol:
    offs = np.zeros(len(values) + 1, dtype=np.int32)
    chunks = []
    valid = np.ones(len(values), dtype=bool)
    for i, v in enumerate(values):
        if v is None:
            valid[i] = False
            v = b""
        if isinstance(v, str):
            v = v.encode("utf-8")
        chunks.append(v)
        offs[i + 1] = offs[i] + len(v)
    chars = np.frombuffer(b"".join(chunks), dtype=np.uint8).copy() if chunks else np.zeros(0, np.uint8)
    return HCol(STRING, chars, None if valid.all() else pack_mask(valid), offs)


def _carr(cols: Sequence[HCol]):
    arr = (_OrcCol * max(1, len(cols)))()
    keep = []
    for i, c in enumerate(cols):
        arr[i].type_id = c.type_id
        arr[i].scale = c.scale
        arr[i].size = c.size
        for name, a in (("data", c.data), ("null_mask", c.mask), ("offsets", c.offsets)):
            if a is not None:
                a = np.ascontiguousarray(a)
                keep.append(a)
                setattr(arr[i], name, a.ctypes.data if a.size else None)
                if a.size == 0 and name == "data":
                    z = np.zeros(1, np.uint8); keep.append(z)
                    setattr(arr[i], name, z.ctypes.data)
            else:
                setattr(arr[i], name, None)
    return arr, keep


def _check(rc: int, what: str):
    if rc < 0:
        raise {-1: ValueError, -2: NotImplementedError, -3: OverflowError}.get(rc, RuntimeError)(
            f"oracle {what} failed: {rc}")


def compute_layout(types: Sequence[int]):
    """-> (starts[ncols], sizes[ncols], validity_offset, size_per_row)   (RC:1332-1371)"""
    n = len(types)
    t = np.asarray(types, dtype=np.int32)
    starts = np.zeros(n + 1, dtype=np.int32)
    sizes = np.zeros(max(n, 1), dtype=np.int32)
    spr = lib().orc_compute_layout(t.ctypes.data_as(C.c_void_p), n, starts.ctypes.data_as(C.c_void_p),
                                   sizes.ctypes.data_as(C.c_void_p))
    _check(spr, "compute_layout")
    return starts[:n].copy(), sizes[:n].copy(), int(starts[n]), int(spr)


def row_sizes(cols: Sequence[HCol]) -> np.ndarray:
    nrows = cols[0].size if cols else 0
    _, _, _, spr = compute_layout([c.type_id for c in cols])
    out = np.zeros(max(nrows, 1), dtype=np.uint64)
    arr, keep = _carr(cols)
    _check(lib().orc_row_sizes(arr, len(cols), C.c_int64(nrows), spr, out.ctypes.data_as(C.c_void_p)),
           "row_sizes")
    return out[:nrows]


def build_batches(sizes: np.ndarray) -> List[int]:
    sizes = np.ascontiguousarray(sizes, dtype=np.uint64)
    bounds = np.zeros(4096, dtype=np.int64)
    nb = lib().orc_build_batches(sizes.ctypes.data_as(C.c_void_p), C.c_int64(len(sizes)),
                                 bounds.ctypes.data_as(C.c_void_p), 4095)
    _check(nb, "build_batches")
    return [int(b) for b in bounds[: nb + 1]]


def convert_to_rows(cols: Sequence[HCol]):
    """-> list of (offsets int32[n+1], data uint8[bytes]) per <=2 GiB batch  (RC:1994-2055)."""
    nrows = cols[0].size if cols else 0
    rs = row_sizes(cols)
    bounds = build_batches(rs)
    arr, keep = _carr(cols)
    out = []
    for b in range(len(bounds) - 1):
        r0, r1 = bounds[b], bounds[b + 1]
        nbytes = int(rs[r0:r1].sum())
        offs = np.zeros(r1 - r0 + 1, dtype=np.int32)
        data = np.zeros(max(nbytes, 1), dtype=np.uint8)
        _check(lib().orc_convert_to_rows(arr, len(cols), C.c_int64(r0), C.c_int64(r1 - r0),
                                         offs.ctypes.data_as(C.c_void_p), data.ctypes.data_as(C.c_void_p),
                                         C.c_int64(nbytes)), "convert_to_rows")
        out.append((offs, data[:nbytes]))
    if nrows == 0:
        out.append((np.zeros(1, np.int32), np.zeros(0, np.uint8)))
    return out


_NP = {INT8: np.int8, INT16: np.int16, INT32: np.int32, INT64: np.int64, UINT8: np.uint8,
       UINT16: np.uint16, UINT32: np.uint32, UINT64: np.uint64, FLOAT32: np.float32,
       FLOAT64: np.float64, BOOL8: np.uint8, TIMESTAMP_DAYS: np.int32, DECIMAL32: np.int32,
       DECIMAL64: np.int64}


def np_dtype(t: int):
    if t in _NP:
        return _NP[t]
    s = size_of(t)
    return {4: np.int32, 8: np.int64}.get(s, np.uint8)


def convert_from_rows(data: np.ndarray, offsets: Optional[np.ndarray], nrows: int,
                      types: Sequence[int], scales: Optional[Sequence[int]] = None):
    """-> (cols: List[HCol], null_counts)   (RC:2149-2441).  offsets=None => fixed-width stride."""
    ncols = len(types)
    words = (nrows + 31) // 32
    cols = []
    for i, t in enumerate(types):
        sc = scales[i] if scales else 0
        if t == STRING:
            cols.append(HCol(t, None, np.zeros(max(words, 1), np.uint32), np.zeros(nrows + 1, np.int32), sc, nrows))
        else:
            cols.append(HCol(t, np.zeros(max(nrows * size_of(t), 1), np.uint8), np.zeros(max(words, 1), np.uint32),
                             None, sc, nrows))
    arr, keep = _carr(cols)
    nulls = np.zeros(max(ncols, 1), dtype=np.int64)
    totals = np.zeros(max(ncols, 1), dtype=np.int64)
    data = np.ascontiguousarray(data, dtype=np.uint8)
    dptr = data.ctypes.data if data.size else np.zeros(1, np.uint8).ctypes.data
    optr = None
    if offsets is not None:
        offsets = np.ascontiguousarray(offsets, dtype=np.int32)
        optr = offsets.ctypes.data
    _check(lib().orc_convert_from_rows_fixed(C.c_void_p(dptr), C.c_void_p(optr), C.c_int64(nrows), arr, ncols,
                                             nulls.ctypes.data_as(C.c_void_p),
                                             totals.ctypes.data_as(C.c_void_p)), "from_rows_fixed")
    any_str = False
    for i, t in enumerate(types):
        if t == STRING:
            any_str = True
            cols[i].data = np.zeros(max(int(totals[i]), 1), np.uint8)
    if any_str:
        arr, keep = _carr(cols)
        _check(lib().orc_convert_from_rows_strings(C.c_void_p(dptr), C.c_void_p(optr), C.c_int64(nrows), arr,
                                                   ncols), "from_rows_strings")
    for i, t in enumerate(types):
        c = cols[i]
        c.mask = c.mask[:words]
        if t == STRING:
            c.data = c.data[: int(totals[i])]
        else:
            c.data = c.data[: nrows * size_of(t)].view(np_dtype(t)) if size_of(t) != 16 else c.data[: nrows * 16]
    return cols, nulls[:ncols]


def xxhash64(cols: Sequence[HCol], seed: int = 42) -> np.ndarray:
    n = cols[0].size if cols else 0
    out = np.zeros(max(n, 1), dtype=np.int64)
    arr, keep = _carr(cols)
    _check(lib().orc_xxhash64(arr, len(cols), C.c_int64(n), C.c_int64(seed), out.ctypes.data_as(C.c_void_p)),
           "xxhash64")
    return out[:n]


def murmur_hash3_32(cols: Sequence[HCol], seed: int = 0) -> np.ndarray:
    n = cols[0].size if cols else 0
    out = np.zeros(max(n, 1), dtype=np.int32)
    arr, keep = _carr(cols)
    _check(lib().orc_murmur3_32(arr, len(cols), C.c_int64(n), C.c_uint32(seed & 0xFFFFFFFF),
                                out.ctypes.data_as(C.c_void_p)), "murmur3_32")
    return out[:n]


def hive_hash(cols: Sequence[HCol]) -> np.ndarray:
    n = cols[0].size if cols else 0
    out = np.zeros(max(n, 1), dtype=np.int32)
    arr, keep = _carr(cols)
    _check(lib().orc_hive_hash(arr, len(cols), C.c_int64(n), out.ctypes.data_as(C.c_void_p)), "hive_hash")
    return out[:n]


# ---- nested keys (LIST / STRUCT): the tree walk of xxhash64.cu:446-506 / murmur_hash.cu:119-144 / hive_hash.cu:363-433,
# restated recursively over small tables; leaves go through the C element hashers above -------------------------------
def list_col(offsets, child: HCol, valid=None) -> HCol:
    offsets = np.asarray(offsets, dtype=np.int32)
    mask = None if valid is None or all(valid) else pack_mask(np.asarray(valid, dtype=bool))
    return HCol(LIST, None, mask, offsets, 0, len(offsets) - 1, [child])


def struct_col(*fields: HCol, valid=None) -> HCol:
    mask = None if valid is None or all(valid) else pack_mask(np.asarray(valid, dtype=bool))
    return HCol(STRUCT, None, mask, None, 0, fields[0].size if fields else 0, list(fields))


def _leaf_c(c: HCol):
    arr, keep = _carr([c])
    return arr, keep


def nested_hash(kind: str, cols: Sequence[HCol], seed: int = 0) -> np.ndarray:
    """kind in {"xxhash64", "murmur3", "hive"}; cols may hold LIST / STRUCT columns."""
    L = lib()
    L.orc_xx_elem.restype = C.c_uint64
    L.orc_xx_elem.argtypes = [C.c_void_p, C.c_int64, C.c_uint64]
    L.orc_mm_elem.restype = C.c_uint32
    L.orc_mm_elem.argtypes = [C.c_void_p, C.c_int64, C.c_uint32]
    L.orc_hive_leaf.restype = C.c_int32
    L.orc_hive_leaf.argtypes = [C.c_void_p, C.c_int64]
    cache = {}

    def cptr(c):
        if id(c) not in cache:
            cache[id(c)] = _leaf_c(c)
        return C.cast(cache[id(c)][0], C.c_void_p)

    # xxhash64 does not look at LIST / STRUCT level nulls (xxhash64.cu:460-462).  murmur3 hashes the table the cudf row
    # hasher prepared (murmur_hash.cu:210): struct nulls pushed down into the fields and null list rows emptied
    # (cudf row_operators.cu:845-852, structs/utilities.cu:617-633), so a null LIST or STRUCT element contributes nothing.
    def live(c, i):
        return kind == "xxhash64" or c.mask is None or bool((int(c.mask[i >> 5]) >> (i & 31)) & 1)

    def chain(c, lo, hi, h):                       # xxhash64 / murmur3: depth-first over the leaves of [lo, hi)
        if c.type_id == LIST:
            if kind == "xxhash64" or c.mask is None:
                return chain(c.children[0], int(c.offsets[lo]), int(c.offsets[hi]), h)
            for i in range(lo, hi):
                if live(c, i):
                    h = chain(c.children[0], int(c.offsets[i]), int(c.offsets[i + 1]), h)
            return h
        if c.type_id == STRUCT:
            for i in range(lo, hi):
                if live(c, i):
                    for f in c.children:
                        h = chain(f, i, i + 1, h)
            return h
        for i in range(lo, hi):
            h = L.orc_xx_elem(cptr(c), i, h) if kind == "xxhash64" else L.orc_mm_elem(cptr(c), i, h)
        return h

    def hive(c, i):                                # hive: structural 31-fold
        if c.type_id == LIST:
            h = 0
            for e in range(int(c.offsets[i]), int(c.offsets[i + 1])):
                h = (31 * h + hive(c.children[0], e)) & 0xFFFFFFFF
            return h
        if c.type_id == STRUCT:
            h = 0
            for f in c.children:
                h = (31 * h + hive(f, i)) & 0xFFFFFFFF
            return h
        return L.orc_hive_leaf(cptr(c), i) & 0xFFFFFFFF
    n = cols[0].size if cols else 0
    if kind == "xxhash64":
        out = np.zeros(n, np.uint64)
        for r in range(n):
            h = seed & (2**64 - 1)
            for c in cols:
                h = chain(c, r, r + 1, h)
            out[r] = h
        return out.view(np.int64)
    out = np.zeros(n, np.uint32)
    for r in range(n):
        h = (seed & 0xFFFFFFFF) if kind == "murmur3" else 0
        for c in cols:
            h = chain(c, r, r + 1, h) if kind == "murmur3" else (31 * h + hive(c, r)) & 0xFFFFFFFF
        out[r] = h
    return out.view(np.int32)


def xxh64_bytes(b: bytes, seed: int) -> int:
    a = np.frombuffer(b, dtype=np.uint8) if b else np.zeros(1, np.uint8)
    return int(lib().orc_xxh64_bytes(C.c_void_p(a.ctypes.data), C.c_int64(len(b)), C.c_uint64(seed & (2**64 - 1))))


def num_threads() -> int:
    return int(lib().orc_num_threads())


# ---- threaded CPU baseline entry points (bench.py only) -------------------------------------
def from_rows_fixed_mt(data: np.ndarray, nrows: int, cols: Sequence[HCol], nthreads: int) -> None:
    arr, keep = _carr(cols)
    _check(lib().orc_from_rows_fixed_mt(C.c_void_p(data.ctypes.data), C.c_int64(nrows), arr, len(cols),
                                        int(nthreads)), "from_rows_fixed_mt")


def from_rows_mt(data: np.ndarray, offsets: Optional[np.ndarray], nrows: int, cols: Sequence[HCol],
                 nthreads: int) -> None:
    arr, keep = _carr(cols)
    optr = offsets.ctypes.data if offsets is not None else None
    _check(lib().orc_from_rows_mt(C.c_void_p(data.ctypes.data), C.c_void_p(optr), C.c_int64(nrows), arr,
                                  len(cols), int(nthreads)), "from_rows_mt")


def to_rows_mt(cols: Sequence[HCol], row_start: int, row_count: int, offsets: np.ndarray, out: np.ndarray,
               nthreads: int) -> None:
    arr, keep = _carr(cols)
    _check(lib().orc_to_rows_mt(arr, len(cols), C.c_int64(row_start), C.c_int64(row_count),
                                C.c_void_p(offsets.ctypes.data), C.c_void_p(out.ctypes.data), int(nthreads)),
           "to_rows_mt")


# ---- Spark HashPartitioning (SURVEY 8f rank 1): the plugin-side consumer of murmur_hash3_32 -----------------------------
def spark_pmod(h: np.ndarray, n: int) -> np.ndarray:
    """Spark's Pmod on int32: r = a % n (truncated, like the JVM); r < 0 ? (r + n) % n : r."""
    a = h.astype(np.int64)
    r = np.fmod(a, n)                       # truncated remainder, sign of the dividend
    return np.where(r < 0, np.fmod(r + n, n), r).astype(np.int32)


def partition_ids(keys: Sequence[HCol], num_partitions: int, seed: int = 42) -> np.ndarray:
    """GpuHashPartitioning: pmod(murmur3_32(seed, keys), numPartitions)."""
    nested = any(k.type_id in (LIST, STRUCT) for k in keys)
    h = nested_hash("murmur3", keys, seed) if nested else murmur_hash3_32(keys, seed)
    return spark_pmod(h.astype(np.int32), num_partitions)


def take(col: HCol, idx: np.ndarray) -> HCol:
    """Rows idx of a fixed-width or STRING column (null payload bytes are carried along)."""
    n = len(idx)
    mask = None if col.mask is None else pack_mask(col.valid()[idx])
    if col.type_id == STRING:
        lens = np.diff(col.offsets.astype(np.int64))[idx]
        offs = np.zeros(n + 1, dtype=np.int32)
        np.cumsum(lens, out=offs[1:])
        chars = np.zeros(int(offs[-1]), dtype=np.uint8)
        for d, s in enumerate(idx):
            chars[offs[d]:offs[d + 1]] = col.data[col.offsets[s]:col.offsets[s + 1]]
        return HCol(STRING, chars, mask, offs, col.scale, n)
    sz = size_of(col.type_id)
    data = np.ascontiguousarray(col.data).view(np.uint8).reshape(col.size, sz)[idx].reshape(-1).copy()
    return HCol(col.type_id, data, mask, None, col.scale, n)


def stable_partition(cols: Sequence[HCol], ids: np.ndarray, num_partitions: int):
    """cudf Table.partition with the rows of a partition in input order: (columns, offsets[P + 1], gather map)."""
    gmap = np.argsort(ids, kind="stable").astype(np.int32)
    offsets = np.zeros(num_partitions + 1, dtype=np.int32)
    np.cumsum(np.bincount(ids, minlength=num_partitions), out=offsets[1:])
    return [take(c, gmap) for c in cols], offsets, gmap
