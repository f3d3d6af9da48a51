"""CPU restatement of the reference's Kudo shuffle wire format for FLAT tables -- TEST INFRASTRUCTURE ONLY.

Follows (file:line in the reference repository's src/main/java/com/nvidia/spark/rapids/jni/kudo/):
  KudoSerializer.java:49-171        the format: header | validity | offsets | data
  KudoTableHeader.java:42,186-200   header = "KUD0" (0x4B554430), offset, numRows, validityBufferLen, offsetBufferLen,
                                    totalDataLen, numColumns -- seven BIG-ENDIAN ints -- then the hasValidity bitset,
                                    (numColumns + 7) / 8 bytes, bit c%8 of byte c/8
  KudoTableHeaderCalc.java:62-79    validityBufferLen is padded so that header + validity is a multiple of 4
                                    (KudoSerializer.java:497-499), offsets and data sections are padded to 4;
                                    totalDataLen = the three padded sizes
  KudoTableHeaderCalc.java:143-195  a column has validity in a partition iff it has a validity vector and rowCount > 0;
                                    STRING offsets: (rowCount + 1) ints when rowCount > 0; data: rowCount * size, or the
                                    chars [offsets[rowOffset], offsets[rowOffset + rowCount])
  SlicedValidityBufferInfo.java:63-77  the validity bytes of rows [o, o + n): from byte o / 8, (o + n - 1) / 8 - o / 8 + 1
                                    bytes, copied as they are (the reader skips o % 8 bits)
  SlicedBufferSerializer.java       buffers are copied raw (little-endian offsets, NOT rebased)
and src/main/cpp/src/shuffle_split.cu:640-690,940-1075 (the GPU writer emits the same bytes, partitions back to back).
Nested types (LIST / STRUCT) are not restated.  Pinned by the header known answer of KudoSerializerTest.java:77-87
(no columns, 5 rows -> 28 bytes) and hand-derived partitions in tests/test_oracle_kudo.py.
"""
import struct
from typing import List, Sequence, Tuple

import numpy as np

from . import oracle as O

MAGIC = 0x4B554430


def header_size(ncols: int) -> int:
    return 28 + (ncols + 7) // 8


def _pad4(x: int) -> int:
    return (x + 3) & ~3


def write_partition(cols: Sequence[O.HCol], row_offset: int, num_rows: int) -> bytes:
    nc = len(cols)
    hs = header_size(nc)
    bitset = bytearray((nc + 7) // 8)
    validity, offsets, data = bytearray(), bytearray(), bytearray()
    for c, col in enumerate(cols):
        if col.mask is not None and num_rows > 0:
            bitset[c // 8] |= 1 << (c % 8)
            b0 = row_offset // 8
            blen = (row_offset + num_rows - 1) // 8 - b0 + 1
            validity += col.mask.view(np.uint8)[b0:b0 + blen].tobytes()
        if col.type_id == O.STRING:
            if num_rows > 0:
                offsets += col.offsets[row_offset:row_offset + num_rows + 1].astype("<i4").tobytes()
            data += col.data[col.offsets[row_offset]:col.offsets[row_offset + num_rows]].tobytes()
        else:
            sz = O.size_of(col.type_id)
            data += np.ascontiguousarray(col.data).view(np.uint8)[row_offset * sz:(row_offset + num_rows) * sz].tobytes()
    vlen = _pad4(len(validity) + hs) - hs
    olen = _pad4(len(offsets))
    dlen = _pad4(len(data))
    head = struct.pack(">7i", MAGIC, row_offset, num_rows, vlen, olen, vlen + olen + dlen, nc) + bytes(bitset)
    return head + bytes(validity) + bytes(vlen - len(validity)) + bytes(offsets) + bytes(olen - len(offsets)) + bytes(data) + bytes(dlen - len(data))


def split(cols: Sequence[O.HCol], splits: Sequence[int]) -> Tuple[np.ndarray, np.ndarray]:
    """shuffle_split: `splits` = P + 1 row indices (0 ... n).  -> (uint8 buffer, int64 offsets[P + 1])."""
    parts = [write_partition(cols, int(splits[p]), int(splits[p + 1] - splits[p])) for p in range(len(splits) - 1)]
    offs = np.zeros(len(parts) + 1, dtype=np.int64)
    np.cumsum([len(p) for p in parts], out=offs[1:])
    return np.frombuffer(b"".join(parts), dtype=np.uint8).copy(), offs


def assemble(buf: np.ndarray, part_offsets: np.ndarray, types: Sequence[int]) -> List[O.HCol]:
    """shuffle_assemble / KudoTableMerger: the partitions concatenated into one table (rows in partition order)."""
    nc = len(types)
    hs = header_size(nc)
    raw = buf.tobytes()
    valid = [[] for _ in types]
    fixed = [bytearray() for _ in types]
    strs = [[] for _ in types]
    for p in range(len(part_offsets) - 1):
        base = int(part_offsets[p])
        magic, roff, n, vlen, olen, total, ncols = struct.unpack(">7i", raw[base:base + 28])
        assert magic == MAGIC and ncols == nc
        bitset = raw[base + 28:base + hs]
        v_at, o_at, d_at = base + hs, base + hs + vlen, base + hs + vlen + olen
        for c, t in enumerate(types):
            has_v = (bitset[c // 8] >> (c % 8)) & 1
            if has_v:
                blen = (roff + n - 1) // 8 - roff // 8 + 1
                bits = np.unpackbits(np.frombuffer(raw[v_at:v_at + blen], dtype=np.uint8), bitorder="little")
                valid[c].append(bits[roff % 8: roff % 8 + n].astype(bool))
                v_at += blen
            else:
                valid[c].append(np.ones(n, dtype=bool))
            if t == O.STRING:
                if n > 0:
                    o = np.frombuffer(raw[o_at:o_at + 4 * (n + 1)], dtype="<i4")
                    o_at += 4 * (n + 1)
                    chars = raw[d_at:d_at + int(o[-1] - o[0])]
                    d_at += len(chars)
                    strs[c] += [chars[int(o[i] - o[0]):int(o[i + 1] - o[0])] for i in range(n)]
            else:
                sz = O.size_of(t)
                fixed[c] += raw[d_at:d_at + n * sz]
                d_at += n * sz
    out = []
    for c, t in enumerate(types):
        v = np.concatenate(valid[c]) if valid[c] else np.zeros(0, bool)
        mask = None if v.all() else O.pack_mask(v)
        if t == O.STRING:
            offs = np.zeros(len(strs[c]) + 1, dtype=np.int32)
            np.cumsum([len(s) for s in strs[c]], out=offs[1:])
            out.append(O.HCol(O.STRING, np.frombuffer(b"".join(strs[c]), dtype=np.uint8).copy(), mask, offs, 0, len(strs[c])))
        else:
            out.append(O.HCol(t, np.frombuffer(bytes(fixed[c]), dtype=np.uint8).copy(), mask, None, 0, len(v)))
    return out
