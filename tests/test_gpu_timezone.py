"""GPU tests of GpuTimeZoneDB against the numpy oracle (oracle/timezone.py): values, masks and null counts of the four
natives over the fixture zones of tests/golden/timezone_golden.py, in every unit and both directions, around every
transition, on the rule path, the table path and both, outside the precomputed years, at int64 extremes, at tile and
mask-word edges, on unaligned buffers, at 100 M rows and on four threads with their own streams."""
import threading

import numpy as np
import pytest

from golden import timezone_golden as G
from oracle import timezone as OT

pytestmark = pytest.mark.gpu

UNITS = [OT.TIMESTAMP_SECONDS, OT.TIMESTAMP_MILLISECONDS, OT.TIMESTAMP_MICROSECONDS, OT.TIMESTAMP_NANOSECONDS]
ROWS = [1, 3, 4, 31, 33, 1023, 1024, 1025, 262_147]


@pytest.fixture(scope="module")
def S():
    import gpu_util
    gpu_util.require_cuda()
    import srj_b200
    return srj_b200


@pytest.fixture(scope="module")
def Z(S):
    from srj_b200.timezone import TimeZoneTable
    t = TimeZoneTable(G.ZONES, G.ENTRIES, G.RULES)
    return t, OT.Table(*t.arrays()), t.to_device()


def _pack(valid):
    if valid is None:
        return None
    bits = np.zeros(((len(valid) + 31) // 32) * 32, np.uint8)
    bits[:len(valid)] = valid
    return np.packbits(bits, bitorder="little").view(np.uint32)


def _col(S, t, vals, valid=None, misalign=False):
    import torch
    c = S.ColumnVector.from_numpy(t, np.ascontiguousarray(vals), _pack(valid), size=len(vals))
    if misalign and len(vals):
        w = vals.itemsize
        buf = torch.empty(len(vals) * w + w, dtype=torch.uint8, device="cuda")
        buf[w:] = c.data
        c = S.ColumnVector(S.DType(t), len(vals), buf[w:], c.mask)
        assert c.data.data_ptr() % 16 != 0
    return c


def _host(c):
    n = c.size
    vals = c.data.cpu().numpy().view(np.int64)[:n] if n else np.zeros(0, np.int64)
    if c.mask is None:
        return vals, None
    return vals, np.unpackbits(c.mask.cpu().numpy().view(np.uint8), bitorder="little")[:n].astype(bool)


def _check(S, Z, direction, t, zone, vals, valid=None, misalign=False):
    from srj_b200.timezone import GpuTimeZoneDB
    tbl, otbl, info = Z
    fn = GpuTimeZoneDB.convertTimestampColumnToUTC if direction == OT.TO_UTC else GpuTimeZoneDB.convertUTCTimestampColumnToTimeZone
    out = fn(_col(S, t, vals, valid, misalign), info, zone)
    got, mask = _host(out)
    want = OT.convert(direction, t, vals, otbl, zone)
    assert out.dtype.type_id == t and out.size == len(vals)
    bad = np.nonzero(got != want)[0]
    assert len(bad) == 0, (tbl.names[zone], [(int(vals[i]), int(got[i]), int(want[i])) for i in bad[:5]])
    if valid is None:
        assert mask is None and out.getNullCount() == 0
    else:
        assert np.array_equal(mask, valid) and out.getNullCount() == int((~valid).sum())


def _around_transitions(otbl, zone, unit):
    """Seconds +-1 s and +-1 unit around every transition instant (UTC and local), and negative sub-second values."""
    utc, local, _, rules = otbl.zone(zone)
    inst = np.concatenate([utc[1:], local[1:]])
    if rules is not None:
        years = np.arange(1900, 2301)
        inst = np.concatenate([inst] + [OT.rule_instant(years, r) + d for r in rules for d in (0, r[4], r[5])])
    inst = inst[np.abs(inst) < 2**62 // unit]
    base = inst * unit
    vals = np.concatenate([base + d for d in (-unit, -1, 0, 1, unit)] + [np.array([0, -1, 1], np.int64)])
    return np.unique(vals)


@pytest.mark.parametrize("t", UNITS)
@pytest.mark.parametrize("direction", [OT.TO_UTC, OT.FROM_UTC])
def test_every_zone_around_every_transition(S, Z, t, direction):
    for zone in range(len(G.ZONES)):
        _check(S, Z, direction, t, zone, _around_transitions(Z[1], zone, OT.UNITS[t]))


@pytest.mark.parametrize("span", ["table", "rules", "both", "outside_window", "extremes"])
@pytest.mark.parametrize("direction", [OT.TO_UTC, OT.FROM_UTC])
def test_paths(S, Z, span, direction):
    rng = np.random.default_rng(7)
    n = 200_003
    for t in UNITS:
        unit = OT.UNITS[t]
        lim = (2**63 - 1) // unit
        if span == "table":
            s = rng.integers(-2208988800, 946684800, n)                     # 1900 .. 2000
        elif span == "rules":
            s = rng.integers(2240524800, 7258118400, n)                     # 2041 .. 2200
        elif span == "both":
            s = rng.integers(946684800, 4102444800, n)                      # 2000 .. 2100
        elif span == "outside_window":
            s = np.concatenate([rng.integers(7289654400, min(lim, 10**13), n // 2), rng.integers(-min(lim, 10**13), -2208988800, n // 2)])
        else:
            s = rng.integers(-lim, lim, n, endpoint=True)
        vals = s.astype(np.int64) * unit + rng.integers(0, unit, len(s)) if span != "extremes" else \
            np.concatenate([rng.integers(-2**63, 2**63 - 1, n, dtype=np.int64, endpoint=True), [-2**63, 2**63 - 1, -2**63 + 1, 2**63 - 2]]).astype(np.int64)
        for zone in (G.ZONES.index("America/Los_Angeles"), G.ZONES.index("Australia/Lord_Howe"), G.ZONES.index("Europe/Dublin"),
                     G.ZONES.index("America/Nuuk"), G.ZONES.index("Asia/Gaza"), G.ZONES.index("Asia/Kathmandu"), G.ZONES.index("UTC")):
            _check(S, Z, direction, t, zone, vals)


@pytest.mark.parametrize("n", ROWS)
def test_rows_masks_and_alignment(S, Z, n):
    rng = np.random.default_rng(n)
    vals = rng.integers(-2208988800 * 10**6, 4102444800 * 10**6, n).astype(np.int64)
    valid = rng.random(n) >= 0.3
    zone = G.ZONES.index("America/New_York")
    for direction in (OT.TO_UTC, OT.FROM_UTC):
        _check(S, Z, direction, OT.TIMESTAMP_MICROSECONDS, zone, vals)
        _check(S, Z, direction, OT.TIMESTAMP_MICROSECONDS, zone, vals, valid)
        _check(S, Z, direction, OT.TIMESTAMP_MICROSECONDS, zone, vals, valid, misalign=True)


def test_empty_and_errors(S, Z):
    from srj_b200.timezone import GpuTimeZoneDB
    info = Z[2]
    out = GpuTimeZoneDB.convertTimestampColumnToUTC(S.ColumnVector.from_numpy(OT.TIMESTAMP_MICROSECONDS, np.zeros(0, np.int64)), info, 0)
    assert out.size == 0
    col = S.ColumnVector.from_numpy(OT.TIMESTAMP_MICROSECONDS, np.arange(5, dtype=np.int64))
    for bad in (-1, len(G.ZONES)):
        with pytest.raises(S.CudfException):
            GpuTimeZoneDB.convertTimestampColumnToUTC(col, info, bad)
    with pytest.raises(S.CudfException):
        GpuTimeZoneDB.convertTimestampColumnToUTC(S.ColumnVector.from_numpy(S.DType.INT64, np.arange(5, dtype=np.int64)), info, 0)
    # a zone without entries, and one with 6 rule integers
    from srj_b200.timezone import TimeZoneTable
    for entries, rules in (([], []), ([(-2**63, -2**63, 0)], [3, 8, 6, 7200, 0, 3600])):
        bad = TimeZoneTable(["X"], [entries], [rules]).to_device()
        with pytest.raises(S.CudfException):
            GpuTimeZoneDB.convertUTCTimestampColumnToTimeZone(col, bad, 0)


def test_hundred_million_rows(S, Z):
    import torch
    from srj_b200.timezone import GpuTimeZoneDB
    n = 100_000_000
    zone = G.ZONES.index("America/Los_Angeles")
    g = torch.Generator(device="cuda").manual_seed(3)
    d = torch.randint(-2208988800 * 10**6, 4102444800 * 10**6, (n,), generator=g, device="cuda", dtype=torch.int64)
    col = S.ColumnVector(S.DType(OT.TIMESTAMP_MICROSECONDS), n, d.view(torch.uint8))
    for direction, fn in ((OT.TO_UTC, GpuTimeZoneDB.convertTimestampColumnToUTC), (OT.FROM_UTC, GpuTimeZoneDB.convertUTCTimestampColumnToTimeZone)):
        out = fn(col, Z[2], zone)
        idx = np.unique(np.concatenate([np.random.default_rng(1).integers(0, n, 1_000_000), np.arange(n - 4099, n), np.arange(4099)]))
        ti = torch.from_numpy(idx).cuda()
        vals = d[ti].cpu().numpy()
        got = out.data.view(torch.int64)[ti].cpu().numpy()
        assert np.array_equal(got, OT.convert(direction, OT.TIMESTAMP_MICROSECONDS, vals, Z[1], zone))
        del out


def test_four_threads_own_streams(S, Z):
    import torch
    from srj_b200.timezone import GpuTimeZoneDB
    errs = []

    def work(k):
        try:
            rng = np.random.default_rng(100 + k)
            vals = rng.integers(-2**62, 2**62, 300_001).astype(np.int64)
            zone = [0, 3, 6, 9][k]
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                for _ in range(3):
                    out = GpuTimeZoneDB.convertUTCTimestampColumnToTimeZone(_col(S, OT.TIMESTAMP_NANOSECONDS, vals), Z[2], zone)
                    s.synchronize()
                    assert np.array_equal(_host(out)[0], OT.convert(OT.FROM_UTC, OT.TIMESTAMP_NANOSECONDS, vals, Z[1], zone))
        except Exception as e:        # noqa: BLE001
            errs.append(e)
    th = [threading.Thread(target=work, args=(k,)) for k in range(4)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    assert not errs, errs


def test_java_cases(S, Z):
    alias = {"US/Pacific": "America/Los_Angeles"}
    from srj_b200.timezone import GpuTimeZoneDB
    for name, t, direction, zone, inp, exp in G.JAVA_CASES:
        valid = np.array([v is not None for v in inp])
        fn = GpuTimeZoneDB.convertTimestampColumnToUTC if direction == OT.TO_UTC else GpuTimeZoneDB.convertUTCTimestampColumnToTimeZone
        out = fn(_col(S, t, np.array([v or 0 for v in inp], np.int64), valid if not valid.all() else None), Z[2], Z[0].index(alias.get(zone, zone)))
        got, mask = _host(out)
        assert np.array_equal(got[valid], np.array([e for e in exp if e is not None], np.int64)), name
        assert out.getNullCount() == int((~valid).sum())


# ---- one zone per row ---------------------------------------------------------------------------------------------------
def _multi(S, Z, sec, us, invalid, ttype, toff, idx):
    from srj_b200.timezone import GpuTimeZoneDB
    cols = [S.ColumnVector.from_numpy(tid, np.ascontiguousarray(a), size=len(sec)) for tid, a in
            ((S.DType.INT64, sec), (S.DType.INT32, us), (S.DType.BOOL8, invalid.astype(np.uint8)), (S.DType.UINT8, ttype),
             (S.DType.INT32, toff), (S.DType.INT32, idx))]
    out = GpuTimeZoneDB.convertTimestampColumnToUTCWithTzCv(*cols[:5], Z[2], cols[5])
    want, valid = OT.convert_multi(sec, us, invalid, ttype, toff, Z[1], idx)
    got, mask = _host(out)
    assert out.dtype.type_id == OT.TIMESTAMP_MICROSECONDS
    assert np.array_equal(got, want), [(i, int(got[i]), int(want[i])) for i in np.nonzero(got != want)[0][:5]]
    assert out.getNullCount() == int((~valid).sum())
    if valid.all():
        assert mask is None
    else:
        assert np.array_equal(mask, valid)


@pytest.mark.parametrize("n", [1, 31, 32, 33, 255, 256, 257, 1_000_003])
def test_multi_rows(S, Z, n):
    rng = np.random.default_rng(n)
    sec = rng.integers(-2208988800, 7258118400, n).astype(np.int64)
    us = rng.integers(0, 10**6, n).astype(np.int32)
    invalid = rng.random(n) < 0.1
    ttype = rng.integers(0, 3, n).astype(np.uint8)
    toff = rng.integers(-18 * 3600, 18 * 3600, n).astype(np.int32)
    idx = rng.integers(-2, len(G.ZONES) + 2, n).astype(np.int32)               # some out of range
    _multi(S, Z, sec, us, invalid, ttype, toff, idx)
    _multi(S, Z, sec, us, np.zeros(n, bool), np.full(n, 2, np.uint8), toff, rng.integers(0, len(G.ZONES), n).astype(np.int32))


def test_multi_overflow_boundary(S, Z):
    mx, mn = (2**63 - 1) // 10**6, -(2**63 // 10**6) - 1
    sec = np.array([mx, mx, mx + 1, mn, mn, mn - 1, mn + 1, 0, -1, mx - 1], np.int64)
    us = np.array([775807, 775808, 0, 224191, 224192, 0, 0, 999999, 0, 999999], np.int32)
    n = len(sec)
    utc = G.ZONES.index("UTC")
    _multi(S, Z, sec, us, np.zeros(n, bool), np.zeros(n, np.uint8), np.zeros(n, np.int32), np.full(n, utc, np.int32))
    _multi(S, Z, sec, us, np.zeros(n, bool), np.ones(n, np.uint8), np.zeros(n, np.int32), np.full(n, -7, np.int32))


def test_multi_transitions_and_rules(S, Z):
    otbl = Z[1]
    secs, idxs = [], []
    for zone in range(len(G.ZONES)):
        s = _around_transitions(otbl, zone, 1)
        secs.append(s)
        idxs.append(np.full(len(s), zone, np.int32))
    sec, idx = np.concatenate(secs), np.concatenate(idxs)
    n = len(sec)
    _multi(S, Z, sec, np.zeros(n, np.int32), np.zeros(n, bool), np.zeros(n, np.uint8), np.zeros(n, np.int32), idx)


# ---- ORC --------------------------------------------------------------------------------------------------------------------
def _orc_table(S, name):
    if name is None:
        return None, None, 0
    raw, tr, of = G.ORC[name]
    if not tr:
        return None, None, raw
    return S.Table(S.ColumnVector.from_numpy(S.DType.INT64, np.array(tr, np.int64)),
                   S.ColumnVector.from_numpy(S.DType.INT32, np.array(of, np.int32))), (np.array(tr, np.int64), np.array(of, np.int32)), raw


@pytest.mark.parametrize("writer,reader", [("Asia/Shanghai", "UTC"), ("UTC", "Asia/Kolkata"), ("Etc/GMT+5", "Asia/Tokyo"),
                                           ("America/Los_Angeles", "Europe/Paris"), ("Africa/Casablanca", "Asia/Kathmandu"),
                                           ("Europe/Paris", "America/Los_Angeles"), ("Asia/Kathmandu", "Asia/Kathmandu")])
def test_orc(S, writer, reader):
    from srj_b200.timezone import GpuTimeZoneDB
    wt, wh, wraw = _orc_table(S, writer)
    rt, rh, rraw = _orc_table(S, reader)
    rng = np.random.default_rng(11)
    trans = np.concatenate([G.ORC[writer][1], G.ORC[reader][1], [0]]).astype(np.int64)
    near = np.concatenate([(trans + d) * 1000 + e for d in (-3600001, -1, 0, 1, 3600000) for e in (-1, 0, 1, 999)])
    vals = np.concatenate([near, rng.integers(-2**62, 2**62, 300_000), rng.integers(-2208988800 * 10**6, 4102444800 * 10**6, 300_000)]).astype(np.int64)
    valid = rng.random(len(vals)) >= 0.25
    for v in (None, valid):
        for mis in (False, True):
            out = GpuTimeZoneDB.convertOrcTimezones(_col(S, OT.TIMESTAMP_MICROSECONDS, vals, v, mis), wt, wraw, rt, rraw)
            got, mask = _host(out)
            want = OT.convert_orc(vals, wh[0] if wh else None, wh[1] if wh else None, wraw, rh[0] if rh else None, rh[1] if rh else None, rraw)
            assert np.array_equal(got, want), [(int(vals[i]), int(got[i]), int(want[i])) for i in np.nonzero(got != want)[0][:5]]
            assert (mask is None) if v is None else np.array_equal(mask, v)


def test_orc_large_tables_read_global_memory(S):
    from srj_b200.timezone import GpuTimeZoneDB
    rng = np.random.default_rng(5)
    tr = np.unique(rng.integers(-2**40, 2**40, 3000)).astype(np.int64)
    of = rng.integers(-14 * 3600000, 14 * 3600000, len(tr)).astype(np.int32)
    tbl = S.Table(S.ColumnVector.from_numpy(S.DType.INT64, tr), S.ColumnVector.from_numpy(S.DType.INT32, of))
    vals = np.concatenate([tr * 1000, tr * 1000 - 1, rng.integers(-2**50, 2**50, 100_000)]).astype(np.int64)
    out = GpuTimeZoneDB.convertOrcTimezones(_col(S, OT.TIMESTAMP_MICROSECONDS, vals), tbl, 3600000, None, -7200000)
    assert np.array_equal(_host(out)[0], OT.convert_orc(vals, tr, of, 3600000, None, None, -7200000))
    out = GpuTimeZoneDB.convertOrcTimezones(_col(S, OT.TIMESTAMP_MICROSECONDS, vals), None, 0, tbl, 3600000)
    assert np.array_equal(_host(out)[0], OT.convert_orc(vals, None, None, 0, tr, of, 3600000))


def test_large_zone_reads_global_memory(S):
    """A zone of more entries than a CTA stages is searched in global memory."""
    from srj_b200.timezone import GpuTimeZoneDB, TimeZoneTable
    rng = np.random.default_rng(9)
    utc = np.unique(rng.integers(-2**40, 2**40, 3000)).astype(np.int64)
    offs = rng.integers(-12, 13, len(utc)) * 3600
    ents = [(-2**63, -2**63, 0)] + [(int(u), int(u), int(o)) for u, o in zip(utc, offs)]
    t = TimeZoneTable(["big"], [ents], [[3, 8, 6, 7200, 0, 3600, 11, 1, 6, 7200, 3600, 0]])
    otbl = OT.Table(*t.arrays())
    vals = np.concatenate([utc, utc - 1, rng.integers(-2**41, 2**41, 100_000)]).astype(np.int64)
    for direction, fn in ((OT.TO_UTC, GpuTimeZoneDB.convertTimestampColumnToUTC), (OT.FROM_UTC, GpuTimeZoneDB.convertUTCTimestampColumnToTimeZone)):
        out = fn(_col(S, OT.TIMESTAMP_SECONDS, vals), t.to_device(), 0)
        assert np.array_equal(_host(out)[0], OT.convert(direction, OT.TIMESTAMP_SECONDS, vals, otbl, 0))
