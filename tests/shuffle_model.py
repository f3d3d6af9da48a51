"""An independent model of the shuffle producers: Spark HashPartitioning (partition ids and the stable partition) and the
Kudo wire format (split and assemble of flat tables), in plain Python integers and bytes.

It imports nothing from oracle/: partition ids come from the row-hash model (spark_hash_model.py), the stable partition
from Python's stable sort, and the Kudo writer and reader are written from the reference's Java (file:line below, in
src/main/java/com/nvidia/spark/rapids/jni/kudo/), not from oracle/kudo.py.  Input columns are read through the
attributes every host column of the suite has (type_id, data, mask, offsets, size); results are MCol.

Kudo (flat tables: fixed width, decimals, STRING):
  KudoSerializer.java:49-171         partition = header | validity | offsets | data
  KudoTableHeader.java:186-200       header = "KUD0", offset, numRows, validityBufferLen, offsetBufferLen,
                                     totalDataLen, numColumns (big-endian ints), then the hasValidity bitset
  KudoTableHeaderCalc.java:59-75    validityBufferLen padded so that header + validity is a multiple of 4
                                     (KudoSerializer.java:493-499), offsets and data padded to 4; totalDataLen = the
                                     three padded lengths
  KudoTableHeaderCalc.java:140-149   hasValidity(c) = the column has a validity vector and the slice has rows
  KudoTableHeaderCalc.java:163-195   validity bytes of the slice; STRING offsets (rowCount + 1) ints when rowCount > 0;
                                     data rowCount * size, or the chars between the slice's first and last offsets
  SlicedValidityBufferInfo.java:63-77  bytes [rowOffset / 8, (rowOffset + numRows - 1) / 8], the first bit at
                                     rowOffset % 8
  KudoTableMerger.java:204-222       assemble: a partition with validity contributes its bits, one without contributes
                                     valid rows (ValidityBufferMerger.appendAllValid)
  KudoTableMerger.java:270-301       offsets rebased: out = in - first offset of the partition + chars so far; the last
                                     output offset is the total
  MergedInfoCalc.java:98-108         the assembled column is nullable iff some partition has its hasValidity bit
                                     (also shuffle_assemble.cu:1759: null count 0 for a column without validity)
"""
from __future__ import annotations

import struct
from dataclasses import dataclass
from typing import List, Optional, Sequence

import numpy as np

import spark_hash_model as H

STRING = H.STRING
MAGIC = 0x4B554430               # "KUD0"


@dataclass
class MCol:
    """A column of the model: raw bytes, validity as a list of bools (None = no mask), STRING offsets as ints."""
    type_id: int
    data: bytes
    valid: Optional[List[bool]]
    offsets: Optional[List[int]] = None
    nullable: bool = True        # for assembled columns: the reference's rule (some partition carried validity)

    @property
    def size(self) -> int:
        return len(self.offsets) - 1 if self.type_id == STRING else len(self.data) // H._SIZE[self.type_id]

    def mask_words(self) -> bytes:
        """The validity as uint32 words, bit r % 32 of word r / 32, tail bits zero (b"" when there is no mask)."""
        if self.valid is None:
            return b""
        return _pack(self.valid, (len(self.valid) + 31) // 32 * 4)

    def null_count(self) -> int:
        return 0 if self.valid is None else self.valid.count(False)


def elem_size(type_id: int) -> int:
    return 0 if type_id == STRING else H._SIZE[type_id]


# ---- reading the suite's host columns ------------------------------------------------------------------------------------
def _bytes(a) -> bytes:
    return b"" if a is None else np.ascontiguousarray(a).view(np.uint8).tobytes()


_BYTE_BITS = [tuple(bool((b >> j) & 1) for j in range(8)) for b in range(256)]


def _unpack(b: bytes, n: int) -> List[bool]:
    """Bits 0 .. n - 1 of b, bit j of byte i being bit 8 i + j."""
    return [x for byte in b[:(n + 7) // 8] for x in _BYTE_BITS[byte]][:n]


def _pack(valid: Sequence[bool], nbytes: int) -> bytes:
    out = bytearray(nbytes)
    for i, v in enumerate(valid):
        if v:
            out[i >> 3] |= 1 << (i & 7)
    return bytes(out)


def _valid_bits(col) -> Optional[List[bool]]:
    if col.mask is None:
        return None
    return _unpack(_bytes(col.mask), col.size)


def _offsets(col) -> List[int]:
    return [int(x) for x in col.offsets]


def from_host(col) -> MCol:
    """A host column as the model sees it (its mask, if any, kept even when every bit is set)."""
    if col.type_id == STRING:
        return MCol(STRING, _bytes(col.data), _valid_bits(col), _offsets(col))
    return MCol(col.type_id, _bytes(col.data)[:col.size * H._SIZE[col.type_id]], _valid_bits(col))


# ---- HashPartitioning ----------------------------------------------------------------------------------------------------
def partition_ids(keys, num_partitions: int, seed: int = 42) -> List[int]:
    """GpuHashPartitioning: Spark's Pmod of the Murmur3 row hash (seed 42 by default)."""
    return [H.pmod(int(h), num_partitions) for h in H.hash_rows("murmur3", keys, seed)]


def stable_partition(ids: Sequence[int], num_partitions: int):
    """-> (offsets[P + 1], gather map (destination -> source), scatter map (source -> destination))."""
    n = len(ids)
    gather = sorted(range(n), key=ids.__getitem__)          # Python's sort is stable: input order inside a partition
    counts = [0] * num_partitions
    for p in ids:
        counts[p] += 1
    offsets = [0]
    for c in counts:
        offsets.append(offsets[-1] + c)
    scatter = [0] * n
    for d, s in enumerate(gather):
        scatter[s] = d
    return offsets, gather, scatter


def take(col, gather: Sequence[int]) -> MCol:
    """Rows `gather` of a host column, null payload bytes and the chars of null strings included."""
    valid = _valid_bits(col)
    out_valid = None if valid is None else [valid[s] for s in gather]
    data = _bytes(col.data)
    if col.type_id == STRING:
        o = _offsets(col)
        chunks = [data[o[s]:o[s + 1]] for s in gather]
        offs = [0]
        for c in chunks:
            offs.append(offs[-1] + len(c))                   # offsets rebuilt from the lengths
        return MCol(STRING, b"".join(chunks), out_valid, offs)
    sz = H._SIZE[col.type_id]
    return MCol(col.type_id, b"".join(data[s * sz:(s + 1) * sz] for s in gather), out_valid)


# ---- Kudo writer ---------------------------------------------------------------------------------------------------------
def _pad4(x: int) -> int:
    return (x + 3) // 4 * 4


def header_size(ncols: int) -> int:
    return 28 + (ncols + 7) // 8                              # KudoTableHeader.getSerializedSize


def validity_slice(row_offset: int, num_rows: int):
    """SlicedValidityBufferInfo.calc: (first byte, byte length, first bit)."""
    length = (row_offset + num_rows - 1) // 8 - row_offset // 8 + 1 if num_rows > 0 else 0
    return row_offset // 8, length, row_offset % 8


class _Raw:
    """A host column read once: bytes of data and mask, offsets as ints, validity as bools on demand."""

    def __init__(self, col):
        self.type_id, self.size = col.type_id, col.size
        self.data = _bytes(col.data)
        self.mask = None if col.mask is None else _bytes(col.mask)
        self.offsets = _offsets(col) if col.type_id == STRING else None
        self._valid = None

    def valid(self) -> Optional[List[bool]]:
        if self.mask is not None and self._valid is None:
            self._valid = _unpack(self.mask, self.size)
        return self._valid


def _raw(cols) -> List[_Raw]:
    return [c if isinstance(c, _Raw) else _Raw(c) for c in cols]


def pad_for_host_alignment(orig: int) -> int:
    return _pad4(orig)                                        # KudoSerializer.java:493-495


def pad_for_validity_alignment(orig: int, header_bytes: int) -> int:
    return _pad4(orig + header_bytes) - header_bytes          # KudoSerializer.java:497-499: relative to the header


def _header_calc(cols: List[_Raw], row_offset: int, num_rows: int):
    """KudoTableHeaderCalc: visit every column (KudoTableHeaderCalc.java:140-149), sum the unpadded buffer lengths
    (dataLenOf*Buffer, :163-195) and set hasValidity; then getHeader (:59-75) pads them."""
    validity_buffer_len = offset_buffer_len = data_only_len = 0
    has_validity = bytearray((len(cols) + 7) // 8)
    for next_col_idx, col in enumerate(cols):
        if col.mask is not None and num_rows > 0:
            validity_buffer_len += validity_slice(row_offset, num_rows)[1]
        if col.type_id == STRING and num_rows > 0:
            offset_buffer_len += (num_rows + 1) * 4
        if col.type_id == STRING:
            data_only_len += col.offsets[row_offset + num_rows] - col.offsets[row_offset]
        else:
            data_only_len += H._SIZE[col.type_id] * num_rows
        if col.mask is not None and num_rows > 0:                               # setHasValidity
            has_validity[next_col_idx // 8] |= 1 << (next_col_idx % 8)
    header_bytes = header_size(len(cols))
    padded_validity = pad_for_validity_alignment(validity_buffer_len, header_bytes)
    padded_offsets = pad_for_host_alignment(offset_buffer_len)
    padded_data = pad_for_host_alignment(data_only_len)
    # KudoTableHeader.writeTo (KudoTableHeader.java:186-200): seven big-endian ints, then the bitset
    return struct.pack(">7i", MAGIC, row_offset, num_rows, padded_validity, padded_offsets,
                       padded_validity + padded_offsets + padded_data, len(cols)) + bytes(has_validity)


def _sliced_buffer(col: _Raw, buffer_type: str, row_offset: int, num_rows: int) -> bytes:
    """SlicedBufferSerializer.copySliced{Validity,Offset,Data} (SlicedBufferSerializer.java:187-245)."""
    if num_rows <= 0:
        return b""
    if buffer_type == "VALIDITY":
        if col.mask is None:
            return b""
        first, length, _ = validity_slice(row_offset, num_rows)
        return col.mask[first:first + length]
    if buffer_type == "OFFSET":
        if col.type_id != STRING:
            return b""
        return struct.pack("<%di" % (num_rows + 1), *col.offsets[row_offset:row_offset + num_rows + 1])
    if col.type_id == STRING:
        return col.data[col.offsets[row_offset]:col.offsets[row_offset + num_rows]]
    size = H._SIZE[col.type_id]
    return col.data[row_offset * size:(row_offset + num_rows) * size]


def write_partition(cols, row_offset: int, num_rows: int) -> bytes:
    """KudoSerializer.writeSliced (KudoSerializer.java:431-463) for rows [row_offset, row_offset + num_rows) of a flat
    table: the header of the header calculation, then one SlicedBufferSerializer pass per buffer type, each visiting
    every column and padding at its end (done(), SlicedBufferSerializer.java:167-181)."""
    cols = _raw(cols)
    header = _header_calc(cols, row_offset, num_rows)
    out = bytearray(header)
    body_bytes = 0
    for buffer_type in ("VALIDITY", "OFFSET", "DATA"):
        written = 0
        for col in cols:
            b = _sliced_buffer(col, buffer_type, row_offset, num_rows)
            out += b
            written += len(b)
        padded = pad_for_validity_alignment(written, len(header)) if buffer_type == "VALIDITY" else pad_for_host_alignment(written)
        out += bytes(padded - written)
        body_bytes += padded
    assert body_bytes == struct.unpack(">i", header[20:24])[0], "header total data length != bytes written"
    return bytes(out)


def split(cols, splits: Sequence[int]):
    """shuffle_split at P + 1 row indices -> (the partitions back to back, byte offsets[P + 1])."""
    cols = _raw(cols)
    parts = [write_partition(cols, int(splits[p]), int(splits[p + 1]) - int(splits[p])) for p in range(len(splits) - 1)]
    offs = [0]
    for b in parts:
        offs.append(offs[-1] + len(b))
    return b"".join(parts), offs


# ---- Kudo reader ---------------------------------------------------------------------------------------------------------
def read_header(buf: bytes, at: int, ncols: int):
    magic, roff, n, vlen, olen, total, nc = struct.unpack(">7i", buf[at:at + 28])
    assert magic == MAGIC and nc == ncols, "not a Kudo header of this schema"
    bits = buf[at + 28:at + header_size(ncols)]
    return roff, n, vlen, olen, total, [bool((bits[c // 8] >> (c % 8)) & 1) for c in range(ncols)]


def assemble(buf: bytes, part_offsets: Sequence[int], types: Sequence[int]) -> List[MCol]:
    """KudoTableMerger over the partitions in order.  Every column gets a validity list; `nullable` says whether the
    reference would give it a mask at all."""
    nc = len(types)
    hs = header_size(nc)
    valid = [[] for _ in types]
    nullable = [False] * nc
    data = [bytearray() for _ in types]
    offs = [[0] for _ in types]
    rows = 0
    for p in range(len(part_offsets) - 1):
        at = int(part_offsets[p])
        roff, n, vlen, olen, _, has_v = read_header(buf, at, nc)
        v_at, o_at, d_at = at + hs, at + hs + vlen, at + hs + vlen + olen
        _, blen, bit = validity_slice(roff, n)
        for c, t in enumerate(types):
            if has_v[c]:
                nullable[c] = True
                valid[c] += _unpack(buf[v_at:v_at + blen], bit + n)[bit:]
                v_at += blen
            else:
                valid[c] += [True] * n                               # appendAllValid
            if t == STRING:
                if n > 0:
                    o = struct.unpack("<%di" % (n + 1), buf[o_at:o_at + 4 * (n + 1)])
                    o_at += 4 * (n + 1)
                    base = offs[c][-1]
                    offs[c][-1:] = [x - o[0] + base for x in o]
                    data[c] += buf[d_at:d_at + o[n] - o[0]]
                    d_at += o[n] - o[0]
            else:
                sz = H._SIZE[t]
                data[c] += buf[d_at:d_at + n * sz]
                d_at += n * sz
        rows += n
    return [MCol(t, bytes(data[c]), valid[c], offs[c] if t == STRING else None, nullable[c]) for c, t in enumerate(types)]


def concat_slices(tables, parts) -> List[MCol]:
    """What assembling the partitions `parts` = [(table, first row, rows)] must give: their rows one after the other;
    a column is nullable iff some part of it has a mask and rows."""
    out = []
    tables = [_raw(t) for t in tables]
    for c in range(len(tables[0])):
        t = tables[0][c].type_id
        valid, chunks, offs, nullable = [], [], [0], False
        for ti, s, n in parts:
            col = tables[ti][c]
            v = col.valid()
            nullable |= v is not None and n > 0
            valid += v[s:s + n] if v is not None else [True] * n
            if t == STRING:
                o = col.offsets
                chunks.append(col.data[o[s]:o[s + n]])
                offs += [x - o[s] + offs[-1] for x in o[s + 1:s + n + 1]]
            else:
                sz = H._SIZE[t]
                chunks.append(col.data[s * sz:(s + n) * sz])
        out.append(MCol(t, b"".join(chunks), valid, offs if t == STRING else None, nullable))
    return out


# ---- golden tables (tests/golden/kudo_golden.py) as host columns ----------------------------------------------------------
TYPE_IDS = {"INT8": H.INT8, "INT16": H.INT16, "INT32": H.INT32, "INT64": H.INT64, "FLOAT32": H.FLOAT32,
            "FLOAT64": H.FLOAT64, "DECIMAL32": H.DECIMAL32, "DECIMAL64": H.DECIMAL64, "DECIMAL128": H.DECIMAL128,
            "STRING": STRING}


@dataclass
class HostCol:
    """A numpy-backed host column with the attributes the suite's host columns have."""
    type_id: int
    data: np.ndarray                 # uint8
    mask: Optional[np.ndarray]       # uint32 words
    offsets: Optional[np.ndarray]    # int32, STRING
    scale: int
    size: int
    children: Optional[list] = None


def pack_valid(valid: Sequence[bool]) -> np.ndarray:
    words = max(1, (len(valid) + 31) // 32)
    return np.frombuffer(_pack(valid, words * 4), np.uint32).copy()


def golden_col(spec) -> HostCol:
    tname, values, validity, scale = spec
    t = TYPE_IDS[tname]
    if isinstance(values, tuple):                        # ("seeded", seed, lo, hi, n)
        _, seed, lo, hi, n = values
        rng = np.random.Generator(np.random.Philox(seed))
        ints = rng.integers(lo, hi, n, endpoint=True, dtype=np.int64)
    else:
        n = len(values)
    if validity is None:
        valid = None
    elif isinstance(validity, tuple) and validity[0] == "mod":
        valid = [i % validity[1] != 0 for i in range(n)]
    elif isinstance(validity, tuple):                    # ("seeded", seed)
        valid = (np.random.Generator(np.random.Philox(validity[1])).random(n) < 0.5).tolist()
    else:
        valid = [bool(x) for x in validity]
    mask = None if valid is None else pack_valid(valid)
    if t == STRING:
        b = [v.encode() if isinstance(v, str) else b"" for v in values]
        offs = np.zeros(n + 1, np.int32)
        offs[1:] = np.cumsum([len(x) for x in b]) if n else []
        return HostCol(t, np.frombuffer(b"".join(b), np.uint8).copy(), mask, offs, scale, n)
    sz = H._SIZE[t]
    if isinstance(values, tuple):
        data = ints.astype({4: np.int32, 8: np.int64}.get(sz, np.int64))
        if sz == 16:                                     # sign-extended to 128 bits
            data = np.stack([ints, ints >> 63], axis=1).reshape(-1)
        data = data.view(np.uint8)
    elif t in (H.FLOAT32, H.FLOAT64):
        data = np.array(values, np.float32 if sz == 4 else np.float64).view(np.uint8)
    else:
        data = np.frombuffer(b"".join(int(v).to_bytes(sz, "little", signed=True) for v in values), np.uint8)
    return HostCol(t, np.ascontiguousarray(data).copy(), mask, None, scale, n)


def golden_tables(case):
    """-> (tables, parts, expected MCol list)"""
    tables = [[golden_col(s) for s in tbl] for tbl in case["tables"]]
    want = concat_slices(tables, case["parts"])
    if case["expected"] is not None:
        exp = [from_host(golden_col(s)) for s in case["expected"]]
        for w, e in zip(want, exp):                      # the stated table, with the nullability the rule gives
            e.nullable = w.nullable
            e.valid = e.valid if e.valid is not None else [True] * e.size
        want = exp
    return tables, case["parts"], want


# masked column counts and slice lengths that between them put the validity padding at 0, 1, 2 and 3
PADDING_COLUMN_COUNTS, PADDING_ROW_COUNTS = (1, 8, 9, 17), (1, 9, 17, 25)


def validity_padding(partition: bytes) -> int:
    """Zero bytes after a partition's validity buffers: its validityBufferLen minus the slices of the columns whose
    hasValidity bit is set."""
    _, n, vlen, _, _, has_v = read_header(partition, 0, struct.unpack(">i", partition[24:28])[0])
    return vlen - sum(has_v) * validity_slice(struct.unpack(">i", partition[4:8])[0], n)[1]


def validity_slice_schedule(masked, unmasked):
    """Partitions that put every validity slice (row offset mod 8, 1 <= n <= 40) at every output bit offset mod 32.
    masked(rows) / unmasked(rows) build one-column tables; before every slice of the masked table, a slice of 0-31 rows
    of the unmasked one moves the output to the wanted offset.  -> (tables, parts)"""
    tables = [masked(200), unmasked(32)]
    parts, at = [], 0
    for r8 in range(8):
        for n in range(1, 41):
            for o32 in range(32):
                k = (o32 - at) % 32
                parts.append((1, 0, k))
                parts.append((0, 8 * ((r8 + n + o32) % 16) + r8, n))
                at += k + n
    return tables, parts


def write_parts(tables, parts):
    """The partitions `parts` written one by one and laid back to back -> (bytes, offsets)."""
    tables = [_raw(t) for t in tables]
    blobs = [write_partition(tables[ti], s, n) for ti, s, n in parts]
    offs = [0]
    for b in blobs:
        offs.append(offs[-1] + len(b))
    return b"".join(blobs), offs
