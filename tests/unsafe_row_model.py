"""An independent model of Apache Spark's UnsafeRow format, in plain numpy.

Written from the format's definition: the comment block at the top of csrc/unsafe_row.cu and DESIGN.md §3.6c, which
restate Spark's UnsafeRow.java and UnsafeRowWriter.java.  It shares no code with oracle/unsafe_row.py or the product
package, so a misreading of the format that both of those made would show up as a difference here.

The format, as this model reads it:
  * a row starts with the null bitset: ceil(fields / 64) little-endian 8-byte words, bit f % 64 of word f // 64 SET
    when field f is NULL;
  * then one 8-byte slot per field.  A fixed-width value sits in the low bytes of its slot, the rest of the slot zero;
    only DECIMAL32 is widened with its sign (decimals of precision <= 18 are longs), every other type is zero-extended
    (UINT32 >= 2^31, a negative TIMESTAMP_DAYS, ...).  A NULL fixed-width field has slot 0.  Floats are bit patterns;
  * then the variable-length region, entries in field order, each padded with zeros to a multiple of 8 bytes.  A
    STRING's slot is (offset from the row start << 32) | length; a NULL string has slot 0 and no entry.  A DECIMAL128
    always reserves 16 zeroed bytes holding BigInteger.toByteArray() of the unscaled value (big-endian two's
    complement, bitLength() / 8 + 1 bytes); its slot is (offset << 32) | byte count, and a NULL keeps the offset with
    count 0;
  * every row is a multiple of 8 bytes, so every row starts 8-byte aligned in a table of rows.

Columns are duck-typed: anything with `type_id`, `size`, `data` (bytes of the values, or the chars), `mask` (uint32
words, None = all valid) and `offsets` (STRING: int32[size + 1]).  Work is vectorised over rows, one pass per field;
chars and decimal payloads move through index arrays, with no per-row Python loop.  Rows do not depend on each other,
so `to_rows(cols, lo, hi)` builds any range of rows on its own and a large table can be checked in chunks."""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Sequence

import numpy as np

# cudf type ids (cudf/types.hpp)
(INT8, INT16, INT32, INT64, UINT8, UINT16, UINT32, UINT64, FLOAT32, FLOAT64, BOOL8) = range(1, 12)
(TIMESTAMP_DAYS, TIMESTAMP_SECONDS, TIMESTAMP_MILLISECONDS, TIMESTAMP_MICROSECONDS, TIMESTAMP_NANOSECONDS) = range(12, 17)
(DURATION_DAYS, DURATION_SECONDS, DURATION_MILLISECONDS, DURATION_MICROSECONDS, DURATION_NANOSECONDS) = range(17, 22)
STRING, LIST, DECIMAL32, DECIMAL64, DECIMAL128, STRUCT = 23, 24, 25, 26, 27, 28

# width in the column of every fixed-width type the codec accepts
FIXED_WIDTH = {INT8: 1, UINT8: 1, BOOL8: 1, INT16: 2, UINT16: 2, INT32: 4, UINT32: 4, FLOAT32: 4, TIMESTAMP_DAYS: 4,
               DECIMAL32: 4, INT64: 8, UINT64: 8, FLOAT64: 8, TIMESTAMP_SECONDS: 8, TIMESTAMP_MILLISECONDS: 8,
               TIMESTAMP_MICROSECONDS: 8, TIMESTAMP_NANOSECONDS: 8, DECIMAL64: 8}
SUPPORTED = frozenset(FIXED_WIDTH) | {STRING, DECIMAL128}
MAX_FIELDS = 256

# launch rules of csrc/unsafe_row.cu (pinned against the source by tests/test_unsafe_row_model.py)
STAGE = 12 * 1024           # kUrStage: shared-memory stage of one warp's 32 rows
BATCH = 16                  # kUrBatch: fields whose column loads to_rows issues together
THREADS = 256               # every kernel runs 256-thread CTAs (8 warps, a row per lane)
WARPS = THREADS // 32
ROWS_GRID_PER_SM = 8        # ur_grid: to_rows / from_rows run at most 8 CTAs per SM
CHARS_GRID_PER_SM = 16      # the chars gather runs at most 16 CTAs per SM
DESC_BYTES = 40             # sizeof(UrCol): three pointers and four int32


class UnsupportedSchema(ValueError):
    pass


@dataclass
class Layout:
    fields: int
    bitset_bytes: int
    slot_bytes: int
    fixed_bytes: int        # bitset + slots
    ndec: int               # DECIMAL128 fields: 16 bytes each in every row's variable region
    nstr: int

    @property
    def row_base(self) -> int:
        """Bytes of every row before its strings: fixed + 16 * ndec (the stride of a table without STRING)."""
        return self.fixed_bytes + 16 * self.ndec


def layout(types: Sequence[int]) -> Layout:
    if not 1 <= len(types) <= MAX_FIELDS:
        raise UnsupportedSchema(f"{len(types)} fields: an UnsafeRow schema here has 1 to {MAX_FIELDS}")
    bad = [t for t in types if t not in SUPPORTED]
    if bad:
        raise UnsupportedSchema(f"type ids {sorted(set(bad))} are not supported")
    bs = (len(types) + 63) // 64 * 8
    return Layout(len(types), bs, 8 * len(types), bs + 8 * len(types), sum(t == DECIMAL128 for t in types),
                  sum(t == STRING for t in types))


# ---------------------------------------------------------------------------------------------- column access
def _valid(col, lo: int, hi: int) -> np.ndarray:
    if col.mask is None:
        return np.ones(hi - lo, bool)
    w = np.ascontiguousarray(col.mask).view(np.uint32)
    r = np.arange(lo, hi)
    return ((w[r >> 5] >> (r & 31).astype(np.uint32)) & 1).astype(bool)


def _pack(valid: np.ndarray) -> np.ndarray:
    bits = np.zeros((len(valid) + 31) // 32 * 32, np.uint8)
    bits[:len(valid)] = valid
    return np.packbits(bits, bitorder="little").view(np.uint32)


def _slot_values(col, lo: int, hi: int) -> np.ndarray:
    """uint64 slot of each value of a fixed-width column, valid or not."""
    raw = np.ascontiguousarray(col.data).view(np.uint8)
    w = FIXED_WIDTH[col.type_id]
    v = raw[lo * w:hi * w].view({1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[w])
    if col.type_id == DECIMAL32:
        return v.view(np.int32).astype(np.int64).view(np.uint64)
    return v.astype(np.uint64)


def _str_bounds(col, lo: int, hi: int):
    o = np.asarray(col.offsets).astype(np.int64)
    return o[lo:hi], o[lo + 1:hi + 1] - o[lo:hi]


def _pad8(x):
    return (x + 7) // 8 * 8


def _bit_length(x: np.ndarray) -> np.ndarray:
    """Bits of each uint64 without its leading zeros (0 for 0)."""
    x = x.copy()
    n = np.zeros(len(x), np.int64)
    for s in (32, 16, 8, 4, 2, 1):
        big = x >= (np.uint64(1) << np.uint64(s))
        n += s * big
        x = np.where(big, x >> np.uint64(s), x)
    return n + (x > 0)


def dec128_bytes(raw16: np.ndarray) -> tuple:
    """(n, 16) little-endian two's complement values -> (their BigInteger.toByteArray() lengths, the 16 bytes
    big-endian).  toByteArray() has bitLength() / 8 + 1 bytes, bitLength() counting the bits after the sign bits."""
    lo = raw16[:, :8].copy().view(np.uint64).ravel()
    hi = raw16[:, 8:].copy().view(np.uint64).ravel()
    neg = (hi >> np.uint64(63)).astype(bool)
    flip = np.where(neg, np.uint64(0xFFFFFFFFFFFFFFFF), np.uint64(0))
    mh, ml = hi ^ flip, lo ^ flip
    bitlen = _bit_length(np.where(mh != 0, mh, ml)) + 64 * (mh != 0)
    return bitlen // 8 + 1, raw16[:, ::-1]


def _shl128(hi: np.ndarray, lo: np.ndarray, s: np.ndarray):
    """(hi, lo) 128-bit values shifted left by s bits, 0 <= s <= 128."""
    s = s.astype(np.uint64)
    z = np.uint64(0)
    big = s >= 64
    sb = np.where(big, s - np.uint64(64), z)          # shift counts kept below 64
    ss = np.where(big, z, s)
    carry = np.where(ss == 0, z, lo >> np.where(ss == 0, np.uint64(1), np.uint64(64) - ss))
    nh = np.where(big, np.where(s >= 128, z, lo << sb), (hi << ss) | carry)
    nl = np.where(big, z, lo << ss)
    return nh, nl


def _copy_words(words: np.ndarray, dst_word: np.ndarray, chars: np.ndarray, src: np.ndarray, lens: np.ndarray):
    """Byte strings chars[src[i] : src[i] + lens[i]] into words[dst_word[i]:], zero-padded to whole 8-byte words.
    Moved 8 bytes at a time: the source is read through 8-byte windows that start at every byte."""
    nw = (lens + 7) // 8
    if not nw.sum():
        return
    padded = np.zeros(len(chars) + 8, np.uint8)
    padded[:len(chars)] = chars
    windows = np.ndarray((len(chars) + 1,), np.dtype("<u8"), padded, 0, (1,))
    k = _gather(np.zeros(len(nw), np.int64), nw)                # word index inside each string
    row = np.repeat(np.arange(len(nw)), nw)
    v = windows[src[row] + 8 * k]
    tail = lens[row] - 8 * k                                     # bytes of this word inside the string
    keep = np.where(tail >= 8, np.uint64(0xFFFFFFFFFFFFFFFF),
                    (np.uint64(1) << (8 * np.minimum(tail, 7)).astype(np.uint64)) - np.uint64(1))
    words[dst_word[row] + k] = v & keep


def _sar128(hi: np.ndarray, lo: np.ndarray, s: np.ndarray):
    """(hi, lo) 128-bit two's complement values shifted right arithmetically by s bits, 0 <= s <= 128 (128: 0)."""
    s = s.astype(np.uint64)
    z, u64 = np.uint64(0), np.uint64(64)
    sign = np.where(hi >> np.uint64(63) == 1, np.uint64(0xFFFFFFFFFFFFFFFF), z)
    big = s >= u64
    sb = np.where(big, np.minimum(s - u64, np.uint64(63)), z)
    ss = np.where(big, z, s)
    hs = hi.view(np.int64)
    nl_small = (lo >> ss) | np.where(ss == 0, z, hi << np.where(ss == 0, np.uint64(1), u64 - ss))
    nh_small = (hs >> ss.astype(np.int64)).view(np.uint64)
    nl_big = np.where(s - u64 >= u64, sign, (hs >> sb.astype(np.int64)).view(np.uint64))
    nh = np.where(big, sign, nh_small)
    nl = np.where(big, nl_big, nl_small)
    zero = s >= np.uint64(128)
    return np.where(zero, z, nh), np.where(zero, z, nl)


def _gather(starts: np.ndarray, lens: np.ndarray) -> np.ndarray:
    """Indices of the bytes [starts[i], starts[i] + lens[i]) of every i, back to back."""
    total = int(lens.sum())
    if total == 0:
        return np.zeros(0, np.int64)
    ends = np.cumsum(lens)
    return np.repeat(starts - (ends - lens), lens) + np.arange(total, dtype=np.int64)


# ---------------------------------------------------------------------------------------------- columns -> rows
def _encode(cols, lo: int, hi: Optional[int], var_order: Sequence[int], gap: int):
    types = [c.type_id for c in cols]
    lay = layout(types)
    hi = cols[0].size if hi is None else hi
    n = hi - lo
    valid = [_valid(c, lo, hi) for c in cols]
    str_len = {f: np.where(valid[f], _str_bounds(c, lo, hi)[1], 0) for f, c in enumerate(cols) if c.type_id == STRING}
    sizes = np.full(n, lay.row_base + gap * (lay.ndec + lay.nstr), np.int64)
    for ln in str_len.values():
        sizes += _pad8(ln)
    offsets = np.zeros(n + 1, np.int64)
    np.cumsum(sizes, out=offsets[1:])
    out = np.zeros(int(offsets[-1]), np.uint8)
    words = out.view(np.uint64)
    start = offsets[:-1]
    w0 = start // 8                                   # every row starts on an 8-byte boundary
    head = np.zeros((n, lay.fixed_bytes // 8), np.uint64, order="F")   # bitset words and slots of every row
    sw = lay.bitset_bytes // 8
    for f, c in enumerate(cols):
        head[:, f // 64] |= (~valid[f]).astype(np.uint64) << np.uint64(f % 64)
        if c.type_id in FIXED_WIDTH:
            head[:, sw + f] = np.where(valid[f], _slot_values(c, lo, hi), np.uint64(0))
    cursor = np.full(n, lay.fixed_bytes, np.int64)    # the variable region, entry by entry
    for f in var_order:
        c = cols[f]
        cursor += gap
        if c.type_id == STRING:
            ln = str_len[f]
            head[:, sw + f] = np.where(valid[f], (cursor.astype(np.uint64) << np.uint64(32)) | ln.astype(np.uint64),
                                       np.uint64(0))
            s0, _ = _str_bounds(c, lo, hi)
            _copy_words(words, (start + cursor) // 8, np.ascontiguousarray(c.data).view(np.uint8), s0, ln)
            cursor += _pad8(ln)
        else:                                         # DECIMAL128
            raw = np.ascontiguousarray(c.data).view(np.uint8)[lo * 16:hi * 16].reshape(n, 16)
            nb = np.where(valid[f], dec128_bytes(raw)[0], 0)
            head[:, sw + f] = (cursor.astype(np.uint64) << np.uint64(32)) | nb.astype(np.uint64)
            # the payload is the low nb bytes of the value, big-endian, from the first reserved byte: the value
            # shifted up by 16 - nb bytes, stored big-endian
            v = raw.copy().view(np.uint64)
            hi_w, lo_w = _shl128(v[:, 1], v[:, 0], 8 * (16 - nb))
            at = (start + cursor) // 8
            words[at] = hi_w.byteswap()
            words[at + 1] = lo_w.byteswap()
            cursor += 16
    if n:
        words[w0[:, None] + np.arange(head.shape[1])] = head
    assert np.array_equal(cursor, sizes), "row sizes and entries disagree"
    return offsets, out


def to_rows(cols, lo: int = 0, hi: Optional[int] = None):
    """-> (int64 offsets[hi - lo + 1] relative to row lo, uint8 bytes of rows [lo, hi))."""
    types = [c.type_id for c in cols]
    return _encode(cols, lo, hi, [f for f, t in enumerate(types) if t in (STRING, DECIMAL128)], 0)


def to_rows_permuted(cols, lo: int = 0, hi: Optional[int] = None):
    """Valid UnsafeRows in a layout the encoder never writes: the variable-length entries in reverse field order, each
    behind 8 zero bytes, every slot pointing at its entry.  A reader that follows the slots decodes them; a reader that
    assumes field order or contiguous entries does not."""
    types = [c.type_id for c in cols]
    return _encode(cols, lo, hi, [f for f, t in enumerate(types) if t in (STRING, DECIMAL128)][::-1], 8)


# ---------------------------------------------------------------------------------------------- rows -> columns
@dataclass
class FromRows:
    data: List[np.ndarray]          # every output byte: values (the slot's low bytes, also under a NULL) or chars
    masks: List[np.ndarray]         # uint32 words, 1 = valid, tail bits zero
    offsets: List[Optional[np.ndarray]]   # STRING: int32[n + 1]
    null_counts: np.ndarray


def from_rows(data: np.ndarray, offsets: Optional[np.ndarray], types: Sequence[int], n: Optional[int] = None) -> FromRows:
    """Rows -> columns, reading through the slots.  offsets: int[n + 1] byte offsets of the rows in `data`, or None for
    rows layout(types).row_base bytes apart (then n is needed)."""
    lay = layout(types)
    if offsets is None:
        offsets = np.arange(n + 1, dtype=np.int64) * lay.row_base
    offsets = np.asarray(offsets).astype(np.int64)
    n = len(offsets) - 1
    start = offsets[:-1]
    assert not (start % 8).any(), "rows start on 8-byte boundaries"
    words = np.ascontiguousarray(data).view(np.uint8)[: (len(data) // 8) * 8].view(np.uint64)
    raw = np.ascontiguousarray(data).view(np.uint8)
    w0 = start // 8
    padded = np.zeros(len(raw) + 16, np.uint8)        # 8-byte windows at every byte, readable up to the end + 16
    padded[:len(raw)] = raw
    windows = np.ndarray((len(raw) + 9,), np.dtype("<u8"), padded, 0, (1,))
    res = FromRows([], [], [], np.zeros(len(types), np.int64))
    head = np.asfortranarray(words[w0[:, None] + np.arange(lay.fixed_bytes // 8)])   # bitset words and slots
    for f, t in enumerate(types):
        isnull = ((head[:, f // 64] >> np.uint64(f % 64)) & np.uint64(1)).astype(bool)
        valid = ~isnull
        slot = head[:, lay.bitset_bytes // 8 + f]
        res.masks.append(_pack(valid))
        res.null_counts[f] = int(isnull.sum())
        at = (slot >> np.uint64(32)).astype(np.int64)
        size = (slot & np.uint64(0xFFFFFFFF)).astype(np.int64)
        if t == STRING:
            ln = np.where(valid, size, 0)
            o = np.zeros(n + 1, np.int64)
            np.cumsum(ln, out=o[1:])
            res.offsets.append(o.astype(np.int32))
            res.data.append(raw[_gather(start + at, ln)])
        elif t == DECIMAL128:
            nb = np.where(valid, size, 0)
            # the 16 bytes from the payload's start, big-endian: the payload in the top nb bytes; an arithmetic
            # shift down by the other 16 - nb bytes gives the value with its sign
            p = np.where(nb > 0, start + at, 0)
            top, bot = windows[p].byteswap(), windows[p + 8].byteswap()
            vh, vl = _sar128(top, bot, 8 * (16 - nb))
            res.data.append(np.stack([vl, vh], axis=1).reshape(-1).view(np.uint8).copy())
            res.offsets.append(None)
        else:
            w = FIXED_WIDTH[t]
            res.data.append(np.ascontiguousarray(slot).view(np.uint8).reshape(n, 8)[:, :w].reshape(-1).copy())
            res.offsets.append(None)
    return res


# ---------------------------------------------------------------------------------------------- launch rules
@dataclass
class Plan:
    stage: int                  # bytes of one warp's shared-memory stage
    staged: np.ndarray          # per 32-row warp of the table: assembled / parsed in its stage (else in place)
    rows_grid: int              # CTAs of to_rows / from_rows
    rows_per_sweep: int         # rows one grid-stride step of those CTAs covers
    rows_sweeps: int
    chars_grid: int             # CTAs of the chars gather
    chars_per_sweep: int
    chars_sweeps: int
    smem: int                   # dynamic shared memory of to_rows / from_rows


def _ceil(a: int, b: int) -> int:
    return -(-a // b)


def plan(types: Sequence[int], n: int, sms: int, row_offsets: Optional[np.ndarray] = None) -> Plan:
    """The launch of a table of n rows on a device with `sms` SMs.  row_offsets (int[n + 1]) is given when the call
    passes row offsets; without them rows are row_base bytes apart and the stage shrinks to 32 rows of them."""
    lay = layout(types)
    if row_offsets is not None:
        stage = STAGE
        ro = np.asarray(row_offsets).astype(np.int64)
    else:
        stage = min(STAGE, _pad16(32 * lay.row_base))
        ro = np.arange(n + 1, dtype=np.int64) * lay.row_base
    first = np.arange(0, n, 32)
    last = np.minimum(first + 32, n)
    staged = (ro[last] - ro[first]) <= stage
    rgrid = max(1, min(_ceil(n, THREADS), sms * ROWS_GRID_PER_SM))
    cgrid = max(1, min(_ceil(n, THREADS), sms * CHARS_GRID_PER_SM))
    return Plan(stage, staged, rgrid, rgrid * THREADS, _ceil(n, rgrid * THREADS), cgrid, cgrid * THREADS,
                _ceil(n, cgrid * THREADS), WARPS * stage + lay.fields * (DESC_BYTES + 4) + 16)


def _pad16(x: int) -> int:
    return (x + 15) // 16 * 16
