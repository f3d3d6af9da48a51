"""com.nvidia.spark.rapids.jni.CastStrings' string-to-timestamp and string-to-date casts (CastStrings.java) over the C ABI
(include/srj_b200.h: srj_cast_parse_timestamps, srj_cast_parse_dates), and its radix casts (srj_long_to_binary_*,
srj_integers_to_string_*, srj_bytes_to_hex_*).

    tbl = TimeZoneTable.from_zoneinfo(["America/Los_Angeles", "UTC"])
    ts = CastStrings.toTimestamp(strings, "America/Los_Angeles", False, Version(Version.VANILLA_SPARK, 3, 5, 0), tbl)
    dates = CastStrings.toDate(strings, False)

parseTimestampStrings returns the intermediate STRUCT (result, seconds, microseconds, tz type, tz offset, tz index);
toTimestamp composes it with GpuTimeZoneDB.convertTimestampColumnToUTCWithTzCv.

    b = CastStrings.fromLongToBinary(longs)              # bin(): "1010", 64 digits for a negative value
    s = CastStrings.fromIntegersWithBase(ints, 16)       # hex() of integers ("FF" for INT8 -1); base 10: decimal
    h = CastStrings.bytesToHex(strings_or_binary)        # hex() of STRING / LIST<UINT8>: two digits a byte

fromIntegersWithBase with a base other than 10 or 16 raises CastException on row 0, as the reference does.  Under ANSI both casts return None when
the result has more nulls than the input, as the reference does.  A null argument raises TypeError (NullPointerException),
an unknown default zone ValueError (IllegalArgumentException), errors of the native layer CudfException.
"""
import ctypes as C
import datetime as _dt
import time

import torch

from . import _native as N
from . import ColumnVector, ColumnView, DType, Table, _empty, _stream_ptr
from .timezone import GpuTimeZoneDB, TimeZoneTable, _device, _ptr


class Version:
    """com.nvidia.spark.rapids.jni.Version: a Spark platform (SparkPlatformType's ordinal) and version."""
    VANILLA_SPARK, DATABRICKS, CLOUDERA, UNKNOWN = 0, 1, 2, 3

    def __init__(self, platform: int, major: int, minor: int, patch: int):
        self.platform, self.major, self.minor, self.patch = int(platform), int(major), int(minor), int(patch)

    def getPlatformOrdinal(self) -> int:
        return self.platform

    def getMajor(self) -> int:
        return self.major

    def getMinor(self) -> int:
        return self.minor

    def getPatch(self) -> int:
        return self.patch


_TABLE = None


def _default_table() -> TimeZoneTable:
    """Every zone of the system's tzdata that TimeZoneTable can encode (zones whose POSIX rules use Julian days are left
    out), built once."""
    global _TABLE
    if _TABLE is None:
        import zoneinfo
        names = []
        for name in sorted(zoneinfo.available_timezones()):
            try:
                TimeZoneTable.from_zoneinfo([name])
            except (ValueError, OSError):
                continue
            names.append(name)
        _TABLE = TimeZoneTable.from_zoneinfo(names)
    return _TABLE


def _epoch_day_now(zone: str) -> int:
    """LocalDate.now(ZoneId.of(zone, SHORT_IDS)).toEpochDay()."""
    import zoneinfo
    from .timezone import SHORT_IDS
    z = SHORT_IDS.get(zone, zone)
    tz = _dt.timezone.utc if z in ("Z", "UTC") else zoneinfo.ZoneInfo(z)
    return (_dt.datetime.now(tz).date() - _dt.date(1970, 1, 1)).days


class CastException(RuntimeError):
    """com.nvidia.spark.rapids.jni.CastException: "Error casting data on row <row>: <string>"."""

    def __init__(self, stringWithError: str, rowWithError: int):
        super().__init__(f"Error casting data on row {rowWithError}: {stringWithError}")
        self.stringWithError, self.rowWithError = stringWithError, rowWithError

    def getRowWithError(self) -> int:
        return self.rowWithError

    def getStringWithError(self) -> str:
        return self.stringWithError


def _radix_cast(input: ColumnView, what: str, sizes, write, ws_bytes=None) -> ColumnVector:
    """sizes -> chars -> write of one radix cast; the result's mask is a copy of the input's"""
    from .radix import _device as _radix_device, strings_result
    if input is None:
        raise TypeError(f"{what}: input column is null")
    n = input.size
    dev = _radix_device(input)
    with torch.cuda.device(dev):
        stream = _stream_ptr()
        cin = input._c()
        offsets = _empty(n + 1, torch.int32, dev)
        total = C.c_int64(0)
        if ws_bytes is None:
            N.check(sizes(C.byref(cin), offsets.data_ptr(), C.byref(total), stream), what)
        else:
            ws = _empty(max(ws_bytes(n), 8), torch.uint8, dev)
            N.check(sizes(C.byref(cin), offsets.data_ptr(), C.byref(total), ws.data_ptr(), stream), what)
        chars = _empty(total.value, torch.uint8, dev)
        mask = _empty((n + 31) // 32, torch.int32, dev) if input.mask is not None else None
        out = strings_result(n, offsets, chars, mask, input.getNullCount())
        N.check(write(C.byref(cin), C.byref(out._c()), stream), what)
        return out


class CastStrings:
    @staticmethod
    def parseTimestampStrings(input: ColumnView, defaultTimeZoneIndex: int, defaultEpochDay: int, tzNameToIndexMap: ColumnView,
                              timezoneInfo: Table, sparkVersion: Version, now: int = None) -> ColumnVector:
        """The first phase of CAST(string AS TIMESTAMP): a STRUCT of six columns, one row per string.  now (seconds since
        the epoch, the clock's when None) dates the strings that are a time alone and name a zone."""
        what = "CastStrings.parseTimestampStrings"
        for c, msg in ((input, "input column is null"), (tzNameToIndexMap, "timezone name to index column is null"),
                       (timezoneInfo, "timezone info table is null"), (sparkVersion, "spark version is null")):
            if c is None:
                raise TypeError(f"{what}: {msg}")
        if timezoneInfo.getNumberOfColumns() < 2:
            raise N.CudfException(f"{what}: the timezone info table needs its transitions and DST rules columns")
        fixed, dst = timezoneInfo.getColumn(0), timezoneInfo.getColumn(1)
        now = int(time.time()) if now is None else int(now)
        n = input.size
        dev = _device(input, tzNameToIndexMap)
        with torch.cuda.device(dev):
            outs = [_empty(n * w, torch.uint8, dev) for w in (1, 8, 4, 1, 4, 4)]
            N.check(N.lib().srj_cast_parse_timestamps(C.byref(input._c()), C.byref(tzNameToIndexMap._c()), C.byref(fixed._c()), C.byref(dst._c()),
                                                      int(defaultTimeZoneIndex), int(defaultEpochDay), now, sparkVersion.getPlatformOrdinal(),
                                                      sparkVersion.getMajor(), sparkVersion.getMinor(), sparkVersion.getPatch(),
                                                      *[_ptr(o) for o in outs], _stream_ptr()), what)
            types = (DType.UINT8, DType.INT64, DType.INT32, DType.UINT8, DType.INT32, DType.INT32)
            kids = [ColumnVector(DType(t), n, o, null_count=0) for t, o in zip(types, outs)]
            return ColumnVector(DType(DType.STRUCT), n, None, None, null_count=0, children=kids)

    @staticmethod
    def toTimestamp(input: ColumnView, defaultTimeZone: str, ansi_enabled: bool, sparkVersion: Version,
                    table: TimeZoneTable = None) -> ColumnVector:
        """CAST(string AS TIMESTAMP) in a session whose zone is defaultTimeZone: TIMESTAMP_MICROSECONDS, null where a string
        does not parse; None under ANSI when any string does not.  table defaults to every zone of the system's tzdata."""
        what = "CastStrings.toTimestamp"
        if input is None:
            raise TypeError(f"{what}: input column is null")
        table = _default_table() if table is None else table
        names = table.name_to_index()
        if defaultTimeZone not in names:
            raise ValueError(f"Invalid default timezone: {defaultTimeZone}")
        dev = _device(input)
        name_map = table.name_to_index_map(dev)
        info = table.to_device(dev)
        parsed = CastStrings.parseTimestampStrings(input, names[defaultTimeZone], _epoch_day_now(defaultTimeZone), name_map, info, sparkVersion)
        k = parsed.children
        result = GpuTimeZoneDB.convertTimestampColumnToUTCWithTzCv(k[1], k[2], k[0], k[3], k[4], info, k[5])
        if ansi_enabled and result.getNullCount() > input.getNullCount():
            return None
        return result

    @staticmethod
    def toDate(input: ColumnView, ansiEnabled: bool) -> ColumnVector:
        """CAST(string AS DATE): TIMESTAMP_DAYS, null where a string does not parse; None under ANSI when any does not."""
        what = "CastStrings.toDate"
        if input is None:
            raise TypeError(f"{what}: input column is null")
        n = input.size
        dev = _device(input)
        with torch.cuda.device(dev):
            out = _empty(n * 4, torch.uint8, dev)
            mask = _empty((n + 31) // 32, torch.int32, dev)
            nulls = C.c_int64(0)
            N.check(N.lib().srj_cast_parse_dates(C.byref(input._c()), _ptr(out), _ptr(mask), C.byref(nulls), _stream_ptr()), what)
            result = ColumnVector(DType(DType.TIMESTAMP_DAYS), n, out, mask if nulls.value else None, null_count=nulls.value)
        if ansiEnabled and result.getNullCount() > input.getNullCount():
            return None
        return result

    @staticmethod
    def fromLongToBinary(cv: ColumnView) -> ColumnVector:
        """bin(): each INT64 as its 64-bit two's complement in binary without leading zeros ("0" for zero)."""
        lib = N.lib()
        return _radix_cast(cv, "CastStrings.fromLongToBinary", lib.srj_long_to_binary_sizes, lib.srj_long_to_binary,
                           lib.srj_long_to_binary_workspace_bytes)

    @staticmethod
    def fromIntegersWithBase(cv: ColumnView, base: int) -> ColumnVector:
        """Integers as strings: base 10 decimal with '-', base 16 upper-case hex of the value's own width without leading
        zeros.  Any other base raises CastException on row 0."""
        what = "CastStrings.fromIntegersWithBase"
        if cv is None:
            raise TypeError(f"{what}: input column is null")
        base = int(base)
        if base not in (10, 16):
            raise CastException(f"Bases supported 10, 16; Actual: {base}", 0)
        lib = N.lib()
        return _radix_cast(cv, what, lambda c, o, t, w, s: lib.srj_integers_to_string_sizes(c, base, o, t, w, s),
                           lambda c, o, s: lib.srj_integers_to_string(c, base, o, s), lib.srj_integers_to_string_workspace_bytes)

    @staticmethod
    def bytesToHex(cv: ColumnView) -> ColumnVector:
        """hex() of STRING or LIST<UINT8> (BinaryType): two upper-case digits a byte."""
        lib = N.lib()
        return _radix_cast(cv, "CastStrings.bytesToHex", lib.srj_bytes_to_hex_sizes, lib.srj_bytes_to_hex)
