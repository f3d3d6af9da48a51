"""com.nvidia.spark.rapids.jni.JoinPrimitives (JoinPrimitives.java) over the C ABI (include/srj_b200.h: srj_hash_inner_join*,
srj_join_*): the hash inner join of two key tables and the helpers that turn its gather maps into outer, semi and anti joins.

    left, right = JoinPrimitives.hashInnerJoin(left_keys, right_keys, compareNullsEqual)   # Tables of key columns
    left, right = JoinPrimitives.makeLeftOuter(left, right, left_rows, right_rows)
    rows        = JoinPrimitives.makeSemi(left, left_rows)
    flags       = JoinPrimitives.getMatchedRows(left, left_rows)                            # BOOL8 ColumnVector

A GatherMap holds int32 row indices; INT32_MIN marks the missing side of an outer row.  The inner join's left map is
non-decreasing; the order of the right rows of one left row is unspecified.  A null argument raises TypeError
(NullPointerException); errors of the native layer raise CudfException.
"""
import ctypes as C

import torch

from . import _native as N
from . import ColumnVector, DType, Table, _carray, _empty, _stream_ptr

INT32_MIN = -(2 ** 31)


class GatherMap:
    """ai.rapids.cudf.GatherMap: an int32 device tensor of row indices."""

    def __init__(self, data: torch.Tensor):
        self.data = data

    def getRowCount(self) -> int:
        return self.data.numel()

    def getBufferLength(self) -> int:
        return 4 * self.data.numel()

    def getBufferAddress(self) -> int:
        return self.data.data_ptr() if self.data.numel() else 0

    def close(self):
        self.data = None


def _device(*ts):
    for t in ts:
        if t is not None:
            return t.device
    return torch.device("cuda", torch.cuda.current_device())


def _ptr(t):
    return t.data_ptr() if t is not None and t.numel() else None


def _map(m: GatherMap, what: str) -> torch.Tensor:
    if m is None:
        raise TypeError(f"{what}: gather map is null")
    return m.data


def _masks(maps, rows, dev):
    """Mark each map into its own match mask; returns the workspaces and their matched counts (one synchronisation)."""
    wss = []
    for m, n in zip(maps, rows):
        ws = _empty(N.lib().srj_join_mask_workspace_bytes(n), torch.uint8, dev)
        N.check(N.lib().srj_join_mark(_ptr(m), m.numel(), n, _ptr(ws), _stream_ptr()), "JoinPrimitives")
        wss.append(ws)
    ptrs = (C.c_void_p * len(wss))(*[w.data_ptr() for w in wss])
    matched = (C.c_int64 * len(wss))()
    N.check(N.lib().srj_join_matched_counts(ptrs, len(wss), matched, _stream_ptr()), "JoinPrimitives")
    return wss, list(matched)


def _outer(left: GatherMap, right: GatherMap, left_size: int, right_size: int, full: bool, what: str):
    lm, rm = _map(left, what), _map(right, what)
    if lm.numel() != rm.numel():
        raise ValueError(f"{what}: left and right gather maps must have the same length")   # IllegalArgumentException
    dev = _device(lm, rm)
    with torch.cuda.device(dev):
        maps, rows = ([lm, rm], [left_size, right_size]) if full else ([lm], [left_size])
        wss, matched = _masks(maps, rows, dev)
        un = [n - m for n, m in zip(rows, matched)] + [0]
        total = lm.numel() + un[0] + (un[1] if full else 0)
        ol, orr = _empty(total, torch.int32, dev), _empty(total, torch.int32, dev)
        N.check(N.lib().srj_join_make_outer(_ptr(lm), _ptr(rm), lm.numel(), left_size, right_size, _ptr(wss[0]), un[0],
                                            _ptr(wss[1]) if full else None, un[1], _ptr(ol), _ptr(orr), _stream_ptr()), what)
        return [GatherMap(ol), GatherMap(orr)]


def _semi_anti(gather_map: GatherMap, size: int, set_rows: bool, what: str) -> GatherMap:
    m = _map(gather_map, what)
    dev = _device(m)
    with torch.cuda.device(dev):
        (ws,), (matched,) = _masks([m], [size], dev)
        out = _empty(matched if set_rows else size - matched, torch.int32, dev)
        if out.numel():
            N.check(N.lib().srj_join_compact(_ptr(ws), size, 1 if set_rows else 0, _ptr(out), _stream_ptr()), what)
        return GatherMap(out)


class JoinPrimitives:
    @staticmethod
    def hashInnerJoin(leftKeys: Table, rightKeys: Table, compareNullsEqual: bool):
        """[left map, right map]: every pair of a left and a right row with equal keys, once; the left map non-decreasing."""
        what = "JoinPrimitives.hashInnerJoin"
        if leftKeys is None or rightKeys is None:
            raise TypeError(f"{what}: keys table is null")                            # JNI_NULL_CHECK
        lc, rc = leftKeys.columns, rightKeys.columns
        dev = _device(*[t for c in lc + rc for t in (c.data, c.offsets, c.mask)])
        with torch.cuda.device(dev):
            la, ra = _carray(lc), _carray(rc)
            ws = _empty(N.lib().srj_hash_join_workspace_bytes(leftKeys.getRowCount(), rightKeys.getRowCount()), torch.uint8, dev)
            pairs = C.c_int64(0)
            N.check(N.lib().srj_hash_inner_join_size(la, len(lc), ra, len(rc), int(bool(compareNullsEqual)), C.byref(pairs), _ptr(ws),
                                                     _stream_ptr()), what)
            lm, rm = _empty(pairs.value, torch.int32, dev), _empty(pairs.value, torch.int32, dev)
            if pairs.value:
                N.check(N.lib().srj_hash_inner_join(la, len(lc), ra, len(rc), int(bool(compareNullsEqual)), _ptr(lm), _ptr(rm), _ptr(ws),
                                                    _stream_ptr()), what)
            return [GatherMap(lm), GatherMap(rm)]

    @staticmethod
    def makeLeftOuter(leftGatherMap: GatherMap, rightGatherMap: GatherMap, leftTableSize: int, rightTableSize: int):
        """The inner pairs, then every left row no in-range left entry names, ascending, with INT32_MIN on the right."""
        return _outer(leftGatherMap, rightGatherMap, leftTableSize, rightTableSize, False, "JoinPrimitives.makeLeftOuter")

    @staticmethod
    def makeFullOuter(leftGatherMap: GatherMap, rightGatherMap: GatherMap, leftTableSize: int, rightTableSize: int):
        """makeLeftOuter, then every unmatched right row, ascending, with INT32_MIN on the left."""
        return _outer(leftGatherMap, rightGatherMap, leftTableSize, rightTableSize, True, "JoinPrimitives.makeFullOuter")

    @staticmethod
    def makeSemi(gatherMap: GatherMap, tableSize: int) -> GatherMap:
        """The distinct in-range indices of the map, ascending."""
        return _semi_anti(gatherMap, tableSize, True, "JoinPrimitives.makeSemi")

    @staticmethod
    def makeAnti(gatherMap: GatherMap, tableSize: int) -> GatherMap:
        """The rows of [0, tableSize) no in-range entry of the map names, ascending."""
        return _semi_anti(gatherMap, tableSize, False, "JoinPrimitives.makeAnti")

    @staticmethod
    def getMatchedRows(gatherMap: GatherMap, tableSize: int) -> ColumnVector:
        """A BOOL8 column of tableSize rows, no null mask: true where an in-range entry of the map names the row."""
        what = "JoinPrimitives.getMatchedRows"
        m = _map(gatherMap, what)
        dev = _device(m)
        with torch.cuda.device(dev):
            out = _empty(max(0, tableSize), torch.uint8, dev)
            N.check(N.lib().srj_join_matched_rows(_ptr(m), m.numel(), tableSize, _ptr(out), _stream_ptr()), what)
            return ColumnVector(DType(DType.BOOL8), tableSize, out, None, null_count=0)
