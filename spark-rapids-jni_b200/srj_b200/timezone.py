"""com.nvidia.spark.rapids.jni.GpuTimeZoneDB's natives (GpuTimeZoneDB.java) over the C ABI (include/srj_b200.h:
srj_timezone_convert*, srj_orc_convert_timezones): from_utc_timestamp / to_utc_timestamp, per-row zones of a string cast,
and ORC's writer -> reader zone conversion.

    tbl = TimeZoneTable.from_zoneinfo(["America/Los_Angeles", "Asia/Shanghai"])    # host-side, no JVM needed
    info = tbl.to_device()                                                          # Table(LIST<STRUCT>, LIST<INT32>)
    utc = GpuTimeZoneDB.convertTimestampColumnToUTC(col, info, tbl.index("America/Los_Angeles"))
    loc = GpuTimeZoneDB.convertUTCTimestampColumnToTimeZone(col, info, 0)

The single-zone conversions keep the input's type, mask and null count.  convertTimestampColumnToUTCWithTzCv returns
TIMESTAMP_MICROSECONDS with a mask only when a row is null.  A null column or table raises TypeError
(NullPointerException), except ORC's tables, where None means a fixed offset; errors of the native layer raise
CudfException.

TimeZoneTable builds GpuTimeZoneDB.loadData's table from TZif files: transitions that change the UT offset, each with
its local instant (utc + offsetAfter for a gap, utc + offsetBefore for an overlap), and the POSIX footer's DST rules as
Java's two ZoneOffsetTransitionRules, ordered by their date in the year.
"""
import ctypes as C
import os
import re
import struct

import numpy as np
import torch

from . import _native as N
from . import ColumnVector, ColumnView, DType, Table, _empty, _stream_ptr

TO_UTC, FROM_UTC = 0, 1       # SRJ_TIMEZONE_*
FIXED_TZ = 1                  # tz type of a row with a fixed offset (convertTimestampColumnToUTCWithTzCv)
INT64_MIN = -(2**63)
# java.time.ZoneId.SHORT_IDS of region zones (EST, HST and MST are fixed offsets a TZif table does not hold)
SHORT_IDS = {"ACT": "Australia/Darwin", "AET": "Australia/Sydney", "AGT": "America/Argentina/Buenos_Aires", "ART": "Africa/Cairo",
             "AST": "America/Anchorage", "BET": "America/Sao_Paulo", "BST": "Asia/Dhaka", "CAT": "Africa/Harare", "CNT": "America/St_Johns",
             "CST": "America/Chicago", "CTT": "Asia/Shanghai", "EAT": "Africa/Addis_Ababa", "ECT": "Europe/Paris",
             "IET": "America/Indiana/Indianapolis", "IST": "Asia/Kolkata", "JST": "Asia/Tokyo", "MIT": "Pacific/Apia", "NET": "Asia/Yerevan",
             "NST": "Pacific/Auckland", "PLT": "Asia/Karachi", "PNT": "America/Phoenix", "PRT": "America/Puerto_Rico",
             "PST": "America/Los_Angeles", "SST": "Pacific/Guadalcanal", "VST": "Asia/Ho_Chi_Minh"}
UTC_NAMES = ("UTC", "Etc/UTC", "Etc/GMT", "GMT")


def _device(*cols):
    for c in cols:
        if c is None:
            continue
        for t in (c.data, c.offsets, c.mask):
            if t is not None:
                return t.device
    return torch.device("cuda", torch.cuda.current_device())


def _ptr(t):
    return t.data_ptr() if t is not None and t.numel() else None


def _info(tz_info, what):
    if tz_info is None:
        raise TypeError(f"{what}: timezone info table is null")                   # JNI_NULL_CHECK
    if tz_info.getNumberOfColumns() < 2:
        raise N.CudfException(f"{what}: the timezone info table needs its transitions and DST rules columns")
    return tz_info.getColumn(0), tz_info.getColumn(1)


def _convert(direction, input, tz_info, tz_index, what):
    if input is None:
        raise TypeError(f"{what}: column is null")
    fixed, dst = _info(tz_info, what)
    n = input.size
    dev = _device(input)
    with torch.cuda.device(dev):
        out = _empty(n * 8, torch.uint8, dev)
        mask = _empty((n + 31) // 32, torch.int32, dev) if input.mask is not None else None
        N.check(N.lib().srj_timezone_convert(direction, C.byref(input._c()), C.byref(fixed._c()), C.byref(dst._c()), int(tz_index),
                                             _ptr(out), _ptr(mask), _stream_ptr()), what)
        return ColumnVector(DType(input.dtype.type_id), n, out, mask, null_count=input.getNullCount())


class GpuTimeZoneDB:
    @staticmethod
    def convertTimestampColumnToUTC(input: ColumnView, tz_info: Table, tz_index: int) -> ColumnVector:
        """Local timestamps of zone tz_index (seconds .. nanoseconds) -> UTC."""
        return _convert(TO_UTC, input, tz_info, tz_index, "GpuTimeZoneDB.convertTimestampColumnToUTC")

    @staticmethod
    def convertUTCTimestampColumnToTimeZone(input: ColumnView, tz_info: Table, tz_index: int) -> ColumnVector:
        """UTC timestamps -> local timestamps of zone tz_index."""
        return _convert(FROM_UTC, input, tz_info, tz_index, "GpuTimeZoneDB.convertUTCTimestampColumnToTimeZone")

    @staticmethod
    def convertTimestampColumnToUTCWithTzCv(seconds: ColumnView, micros: ColumnView, invalid: ColumnView, tz_type: ColumnView,
                                            tz_offset: ColumnView, tz_info: Table, tz_indices: ColumnView) -> ColumnVector:
        """One zone per row (a parsed string's): seconds - offset, plus micros, as TIMESTAMP_MICROSECONDS; invalid rows,
        unknown zones and overflows are null."""
        what = "GpuTimeZoneDB.convertTimestampColumnToUTCWithTzCv"
        cols = (seconds, micros, invalid, tz_type, tz_offset, tz_indices)
        for c, name in zip(cols, ("seconds", "microseconds", "invalid", "tz type", "tz offset", "tz indices")):
            if c is None:
                raise TypeError(f"{what}: {name} column is null")
        fixed, dst = _info(tz_info, what)
        n = seconds.size
        dev = _device(*cols)
        with torch.cuda.device(dev):
            out = _empty(n * 8, torch.uint8, dev)
            mask = _empty((n + 31) // 32, torch.int32, dev)
            nulls = C.c_int64(0)
            cs = [c._c() for c in cols]
            N.check(N.lib().srj_timezone_convert_multi(*[C.byref(c) for c in cs[:5]], C.byref(fixed._c()), C.byref(dst._c()), C.byref(cs[5]),
                                                       _ptr(out), _ptr(mask), C.byref(nulls), _stream_ptr()), what)
            return ColumnVector(DType(DType.TIMESTAMP_MICROSECONDS), n, out, mask if nulls.value else None, null_count=nulls.value)

    @staticmethod
    def convertOrcTimezones(input: ColumnView, writer_table, writer_raw_offset: int, reader_table, reader_raw_offset: int) -> ColumnVector:
        """ORC's convertBetweenTimezones of TIMESTAMP_MICROSECONDS: each table is None (a fixed offset) or a Table of
        (INT64 transitions, INT32 offsets) in milliseconds; raw offsets in milliseconds."""
        what = "GpuTimeZoneDB.convertOrcTimezones"
        if input is None:
            raise TypeError(f"{what}: input column is null")
        sides = []
        for t in (writer_table, reader_table):
            if t is None:
                sides.append((None, None))
            else:
                if t.getNumberOfColumns() < 2:
                    raise N.CudfException(f"{what}: an ORC time zone table needs its transitions and offsets")
                sides.append((t.getColumn(0)._c(), t.getColumn(1)._c()))
        n = input.size
        dev = _device(input)
        ref = lambda c: C.byref(c) if c is not None else None                      # noqa: E731
        with torch.cuda.device(dev):
            out = _empty(n * 8, torch.uint8, dev)
            mask = _empty((n + 31) // 32, torch.int32, dev) if input.mask is not None else None
            N.check(N.lib().srj_orc_convert_timezones(C.byref(input._c()), ref(sides[0][0]), ref(sides[0][1]), int(writer_raw_offset),
                                                      ref(sides[1][0]), ref(sides[1][1]), int(reader_raw_offset), _ptr(out), _ptr(mask),
                                                      _stream_ptr()), what)
            return ColumnVector(DType(DType.TIMESTAMP_MICROSECONDS), n, out, mask, null_count=input.getNullCount())


# ---- the table, built on the host ---------------------------------------------------------------------------------------
_MIN_LENGTH = (31, 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31)      # Month.minLength()


def _parse_tzif(data: bytes):
    """-> (transition times, utoff of each transition's type, utoff of type 0, POSIX footer) of a TZif file (RFC 8536),
    from its 64-bit block when it has one."""
    def header(at):
        if data[at:at + 4] != b"TZif":
            raise ValueError("not a TZif file")
        return data[at + 4:at + 5], struct.unpack(">6l", data[at + 20:at + 44])

    ver, (isut, isstd, leap, timecnt, typecnt, charcnt) = header(0)
    size = 4
    at = 44
    if ver >= b"2":
        at += timecnt * 5 + typecnt * 6 + charcnt + leap * 8 + isstd + isut
        _, (isut, isstd, leap, timecnt, typecnt, charcnt) = header(at)
        at += 44
        size = 8
    times = struct.unpack(">%d%s" % (timecnt, "q" if size == 8 else "l"), data[at:at + timecnt * size])
    at += timecnt * size
    idx = data[at:at + timecnt]
    at += timecnt
    types = [struct.unpack(">lBB", data[at + 6 * i:at + 6 * i + 6])[0] for i in range(typecnt)]
    at += typecnt * 6 + charcnt + leap * (size + 4) + isstd + isut
    footer = ""
    if size == 8 and data[at:at + 1] == b"\n":
        footer = data[at + 1:data.index(b"\n", at + 1)].decode("ascii")
    return list(times), [types[i] for i in idx], types[0], footer


def _posix_offset(s):
    """[+-]hh[:mm[:ss]] -> seconds."""
    m = re.fullmatch(r"([+-]?)(\d+)(?::(\d+))?(?::(\d+))?", s)
    if not m:
        raise ValueError(f"bad POSIX time {s!r}")
    v = int(m.group(2)) * 3600 + int(m.group(3) or 0) * 60 + int(m.group(4) or 0)
    return -v if m.group(1) == "-" else v


def posix_rules(footer: str):
    """The two Java rules (12 ints) of a POSIX TZ string's DST, or [] without DST.  Mm.w.d/t: w 1..4 is the next-or-same
    weekday from day 1 + 7 (w - 1); w 5 is Java's `lastDay`: dom = minLength(month) - 6, next-or-same, except February's
    -1 (previous-or-same from the end).  Day 0 = Monday; t is wall time (secondsFromMidnight, may be negative or past 24h).
    Jn and n dates are rejected."""
    m = re.fullmatch(r"(<[^>]*>|[A-Za-z]+)([-+]?[\d:]+)(?:(<[^>]*>|[A-Za-z]+)([-+]?[\d:]+)?(?:,(.*),(.*))?)?", footer)
    if not m:
        raise ValueError(f"unsupported POSIX TZ string {footer!r}")
    std = -_posix_offset(m.group(2))
    if not m.group(3):
        return []
    if not m.group(5):
        raise ValueError(f"POSIX TZ string {footer!r} has DST but no rules")
    dst = -_posix_offset(m.group(4)) if m.group(4) else std + 3600
    rules = []
    for spec, before, after in ((m.group(5), std, dst), (m.group(6), dst, std)):
        r = re.fullmatch(r"M(\d+)\.(\d)\.(\d)(?:/([-+]?[\d:]+))?", spec)
        if not r:
            raise ValueError(f"unsupported POSIX rule {spec!r} (only Mm.w.d)")
        month, week, day = int(r.group(1)), int(r.group(2)), int(r.group(3))
        t = _posix_offset(r.group(4)) if r.group(4) else 7200
        dow = (day + 6) % 7
        if week == 5:
            dom = -1 if month == 2 else _MIN_LENGTH[month - 1] - 6
        else:
            dom = 1 + 7 * (week - 1)
        rules.append([month, dom, dow, t, before, after])
    rules.sort(key=lambda r: (r[0], r[1] if r[1] > 0 else 32 + r[1]))
    return rules[0] + rules[1]


def zone_entries(times, utoffs, first_off):
    """[(utcInstant, localInstant, offset)] of a zone: entry 0 at INT64_MIN, then each transition that changes the offset."""
    out = [(INT64_MIN, INT64_MIN, first_off)]
    prev = first_off
    for t, after in zip(times, utoffs):
        if after == prev:
            continue
        out.append((t, t + (after if after > prev else prev), after))
        prev = after
    return out


class TimeZoneTable:
    """GpuTimeZoneDB.loadData's table on the host: names[i] is zone i."""

    def __init__(self, names, entries, rules):
        self.names = list(names)
        self.entries = [list(e) for e in entries]        # per zone: [(utc, local, offset)]
        self.rules = [list(r) for r in rules]            # per zone: [] or 12 ints

    @staticmethod
    def from_tzif(name: str, data: bytes):
        times, utoffs, first, footer = _parse_tzif(data)
        return zone_entries(times, utoffs, first), (posix_rules(footer) if footer else [])

    @staticmethod
    def from_zoneinfo(names, root: str = "/usr/share/zoneinfo") -> "TimeZoneTable":
        ents, rules = [], []
        for name in names:
            with open(os.path.join(root, name), "rb") as f:
                e, r = TimeZoneTable.from_tzif(name, f.read())
            ents.append(e)
            rules.append(r)
        return TimeZoneTable(names, ents, rules)

    def index(self, name: str) -> int:
        return self.names.index(name)

    def name_to_index(self) -> dict:
        """Every name a string may give for a zone of the table -> its index: the zones' own names, the SHORT_IDS whose zone
        the table holds, and "Z" for the table's UTC zone (GpuTimeZoneDB's zoneIdToTable)."""
        out = {n: i for i, n in enumerate(self.names)}
        for short, region in SHORT_IDS.items():
            if region in out and short not in out:
                out[short] = out[region]
        utc = [out[n] for n in UTC_NAMES if n in out]
        if utc and "Z" not in out:
            out["Z"] = utc[0]
        return out

    def name_to_index_map(self, device="cuda") -> ColumnVector:
        """GpuTimeZoneDB.getTzNameToIndexMap: STRUCT<name STRING, index INT32> sorted by the names' bytes."""
        items = sorted((n.encode(), i) for n, i in self.name_to_index().items())
        chars = b"".join(k for k, _ in items)
        offs = np.concatenate([[0], np.cumsum([len(k) for k, _ in items])]).astype(np.int32)
        idx = np.array([i for _, i in items], np.int32)
        names = ColumnVector(DType(DType.STRING), len(items), torch.from_numpy(np.frombuffer(chars, np.uint8).copy()).to(device),
                             None, torch.from_numpy(offs).to(device), null_count=0)
        index = ColumnVector(DType(DType.INT32), len(items), torch.from_numpy(idx.view(np.uint8).copy()).to(device), null_count=0)
        return ColumnVector(DType(DType.STRUCT), len(items), None, None, null_count=0, children=[names, index])

    def arrays(self):
        """-> (list offsets, utc, local, offset, rule list offsets, rules) as numpy arrays."""
        lst = np.concatenate([[0], np.cumsum([len(e) for e in self.entries])]).astype(np.int32)
        flat = [x for e in self.entries for x in e]
        utc = np.array([x[0] for x in flat], np.int64)
        local = np.array([x[1] for x in flat], np.int64)
        off = np.array([x[2] for x in flat], np.int32)
        rl = np.concatenate([[0], np.cumsum([len(r) for r in self.rules])]).astype(np.int32)
        rules = np.array([x for r in self.rules for x in r], np.int32)
        return lst, utc, local, off, rl, rules

    def to_device(self, device="cuda") -> Table:
        """The two columns GpuTimeZoneDB.getTimezoneInfo returns: LIST<STRUCT<INT64, INT64, INT32>>, LIST<INT32>."""
        lst, utc, local, off, rl, rules = self.arrays()
        up = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).copy()).to(device)     # noqa: E731
        fields = [ColumnView(DType.INT64, len(utc), up(utc)), ColumnView(DType.INT64, len(local), up(local)),
                  ColumnView(DType.INT32, len(off), up(off))]
        trans = ColumnView.makeListView(torch.from_numpy(lst).to(device), ColumnView.makeStructView(*fields))
        dst = ColumnView.makeListView(torch.from_numpy(rl).to(device), ColumnView(DType.INT32, len(rules), up(rules)))
        return Table(trans, dst)
