"""GPU tests of CastStrings' string-to-timestamp (first phase and end to end) and string-to-date casts against the
restatement in oracle/cast_datetime.py, itself checked against the independent model (tests/cast_datetime_model.py) on every
generated string: the reference's literal cases, 10 M generated rows under each version gate, 100 M rows, null rows whose
offsets span garbage, rows past the 32-byte register window, tile and mask-word edges, an empty column, an unaligned
chars buffer, the native argument errors, and four threads with their own streams."""
import random
import threading

import numpy as np
import pytest

import cast_datetime_gen as GEN
import cast_datetime_model as CM
from golden import cast_datetime_golden as G
from golden import timezone_golden as TG
from oracle import cast_datetime as OC
from oracle import timezone as OTZ

pytestmark = pytest.mark.gpu

GATES = {"320": (0, 3, 2, 0), "330": (0, 3, 3, 0), "400": (0, 4, 0, 0), "db143": (1, 14, 3, 0)}
ROWS = [1, 31, 32, 33, 255, 256, 257, 1025]
NOW = 1_760_000_000


@pytest.fixture(scope="module")
def S():
    import gpu_util
    gpu_util.require_cuda()
    import srj_b200
    return srj_b200


@pytest.fixture(scope="module")
def Z(S):
    from srj_b200.timezone import TimeZoneTable
    t = TimeZoneTable(TG.ZONES, TG.ENTRIES, TG.RULES)
    return t, OTZ.Table(*t.arrays()), t.to_device()


def _strings(S, values, shift=0, garbage_nulls=False):
    """A STRING column of bytes / None; shift moves the chars off their allocation's alignment; garbage_nulls gives every
    null row a span of random bytes."""
    rng = np.random.default_rng(7)
    parts, offs, valid = [], [0], []
    for v in values:
        if v is None and garbage_nulls:
            v_bytes = rng.integers(0, 256, rng.integers(1, 40), dtype=np.uint8).tobytes()
        else:
            v_bytes = v or b""
        parts.append(v_bytes)
        offs.append(offs[-1] + len(v_bytes))
        valid.append(v is not None)
    chars = np.frombuffer(b"\0" * shift + b"".join(parts), np.uint8)
    mask = None
    if not all(valid):
        bits = np.zeros(((len(values) + 31) // 32) * 32, np.uint8)
        bits[:len(values)] = valid
        mask = np.packbits(bits, bitorder="little").view(np.uint32)
    col = S.ColumnVector.from_numpy(S.DType.STRING, chars if len(chars) else np.zeros(0, np.uint8), mask,
                                    np.array(offs, np.int32), size=len(values))
    if shift:
        col.data = col.data[shift:] if col.data is not None else col.data
    return col


def _map(S, pairs):
    names = S.ColumnVector.from_numpy(S.DType.STRING, np.frombuffer(b"".join(k for k, _ in pairs), np.uint8),
                                      None, np.concatenate([[0], np.cumsum([len(k) for k, _ in pairs])]).astype(np.int32))
    idx = S.ColumnVector.from_numpy(S.DType.INT32, np.array([i for _, i in pairs], np.int32))
    return S.ColumnView.makeStructView(names, idx)


def _parse(S, info, col, name_map, version, default_tz=1, epoch_day=1, now=NOW):
    from srj_b200.cast import CastStrings, Version
    out = CastStrings.parseTimestampStrings(col, default_tz, epoch_day, name_map, info, Version(*version), now=now)
    cols = [c.data.cpu().numpy() for c in out.children]
    dts = (np.uint8, np.int64, np.int32, np.uint8, np.int32, np.int32)
    return list(zip(*[c.view(d).tolist() for c, d in zip(cols, dts)]))


def _want(values, name_map, table, version, default_tz=1, epoch_day=1, now=NOW):
    gates = OC.version_gates(*version)
    return [OC.parse_timestamp(v, default_tz, epoch_day, name_map, table, now, *gates) for v in values]


@pytest.mark.parametrize("rows", ["JUST_TIME", "FIRST_PHASE"])
def test_first_phase_goldens(S, Z, rows):
    _, _, info = Z
    cases = getattr(G, rows)
    got = _parse(S, info, _strings(S, [c[0].encode() for c in cases]), _map(S, G.NAME_MAP), GATES["330"], now=0)
    for c, g in zip(cases, got):
        assert g == tuple(c[1:]), c[0]


def _names(table):
    return sorted((n.encode(), i) for n, i in table.name_to_index().items())


DTS = (np.uint8, np.int64, np.int32, np.uint8, np.int32, np.int32)
NULL_ROW = (1, 0, 0, 0, 0, -1)


def _reference(pool, t, ot, version, default_tz, epoch_day):
    """The expected six columns of each pool string: the restatement's, checked against the independent model wherever the
    model defines them (its valid rows and unknown names; the result alone elsewhere)."""
    names, name_dict = _names(t), {k: v for k, v in _names(t)}
    g320, g400 = OC.version_gates(*version)
    import timezone_model as TZM
    tzdata = TZM.available("Asia/Tokyo")             # the model dates a time alone in a named zone through tzdata
    rows = []
    for p in pool:
        want = OC.parse_timestamp(p, default_tz, epoch_day, names, ot, NOW, g320, g400)
        if not tzdata and want[0] == 0 and want[3] == 2 and want[5] != default_tz:
            rows.append(want)
            continue
        valid, row = CM.timestamp(p, default_tz, epoch_day, name_dict, TG.ZONES, NOW, g320, g400)
        assert (row == want) if (valid or row is not None) else want[0] == 1, (p, want, row)
        rows.append(want)
    return [np.array([r[j] for r in rows], d) for j, d in enumerate(DTS)]


def _padded_column(S, pool, pick, width, null_every):
    """A STRING column of len(pick) rows, row r = pool[pick[r]] padded with trailing spaces to width (trimmed by the cast,
    so the padding changes no result), built on the device; every null_every-th row is null over its bytes."""
    import torch
    mat = torch.from_numpy(np.frombuffer(b"".join(p.ljust(width) for p in pool), np.uint8).reshape(len(pool), width).copy()).cuda()
    n = pick.numel()
    chars = mat[pick].reshape(-1)
    offsets = torch.arange(0, (n + 1) * width, width, device="cuda", dtype=torch.int64).to(torch.int32)
    valid = (torch.arange(((n + 31) // 32) * 32, device="cuda") % null_every != 0).to(torch.uint8).reshape(-1, 8)
    bits = (valid * (2 ** torch.arange(8, device="cuda", dtype=torch.uint8))).sum(1, dtype=torch.uint8)
    mask = bits.view(torch.int32)
    return S.ColumnVector(S.DType(S.DType.STRING), n, chars, mask, offsets), (torch.arange(n, device="cuda") % null_every != 0)


def _check_parse(S, info, t, col, pick, valid, ref, version, default_tz, epoch_day):
    import torch
    from srj_b200.cast import CastStrings, Version
    out = CastStrings.parseTimestampStrings(col, default_tz, epoch_day, t.name_to_index_map(), info, Version(*version), now=NOW)
    tdt = (torch.uint8, torch.int64, torch.int32, torch.uint8, torch.int32, torch.int32)
    for j, (kid, d) in enumerate(zip(out.children, tdt)):
        want = torch.from_numpy(ref[j]).cuda()[pick]
        want = torch.where(valid, want, torch.tensor(NULL_ROW[j], dtype=d, device="cuda"))
        got = kid.data.view(d)
        bad = torch.nonzero(got != want).flatten()
        assert bad.numel() == 0, (j, bad[:5].tolist(), got[bad[:5]].tolist(), want[bad[:5]].tolist())


@pytest.mark.parametrize("gate", sorted(GATES))
def test_generated_strings_match_reference(S, Z, gate):
    """10 M rows per version gate, drawn from 100,000 distinct generated strings, 1 % null rows over their bytes."""
    import torch
    t, ot, info = Z
    rng = random.Random(sum(gate.encode()))
    pool = sorted({GEN.timestamp(rng, t.name_to_index()) for _ in range(100_000)})
    ref = _reference(pool, t, ot, GATES[gate], 3, -5)
    n = 10_000_000
    width = max(len(p) for p in pool)
    pick = torch.randint(0, len(pool), (n,), device="cuda", generator=torch.Generator(device="cuda").manual_seed(len(pool)))
    col, valid = _padded_column(S, pool, pick, width, 101)
    _check_parse(S, info, t, col, pick, valid, ref, GATES[gate], 3, -5)


def test_100m_rows(S, Z):
    """100 M rows (the most a STRING column of 21-byte rows holds under 2^31 chars): the timestamp parse and the date
    parse, over generated strings of at most 21 bytes."""
    import torch
    from srj_b200.cast import CastStrings
    t, ot, info = Z
    rng = random.Random(100)
    pool = set()
    while len(pool) < 20_000:
        v = GEN.timestamp(rng, t.name_to_index()) if len(pool) % 2 else GEN.date(rng)
        if len(v) <= 21:
            pool.add(v)
    pool = sorted(pool)
    ref = _reference(pool, t, ot, GATES["330"], 1, 7)
    n, width = 100_000_000, 21
    pick = torch.randint(0, len(pool), (n,), device="cuda", generator=torch.Generator(device="cuda").manual_seed(5))
    col, valid = _padded_column(S, pool, pick, width, 997)
    _check_parse(S, info, t, col, pick, valid, ref, GATES["330"], 1, 7)
    dref = [OC.parse_date(p) for p in pool]
    assert all(CM.date(p) == w for p, w in zip(pool, dref))
    dval = torch.tensor([w is not None for w in dref], device="cuda")[pick] & valid
    dwant = torch.tensor([w or 0 for w in dref], dtype=torch.int32, device="cuda")[pick]
    got = CastStrings.toDate(col, False)
    gvalid = ((got.mask.view(torch.uint8)[torch.arange(n, device="cuda") // 8] >> (torch.arange(n, device="cuda") % 8).to(torch.uint8)) & 1).bool()
    assert torch.equal(gvalid, dval)
    assert torch.equal(got.data.view(torch.int32), torch.where(dval, dwant, torch.zeros_like(dwant)))
    assert got.getNullCount() == int((~dval).sum())


@pytest.mark.parametrize("n", ROWS)
@pytest.mark.parametrize("shift", [0, 1, 3])
def test_tile_edges_unaligned_and_long_rows(S, Z, n, shift):
    t, ot, info = Z
    base = [b"2023-11-05 03:04:55.123456789 America/Los_Angeles", b"  \t-2000-02-29T23:59:59.999999 Australia/Lord_Howe \n",
            b"T12:34:56 Pacific/Chatham", b"2023-03-12 02:30:00", None, b"12:00 +05:45", b"1999-12-31 23:59:60"]
    vals = [base[i % len(base)] for i in range(n)]
    got = _parse(S, info, _strings(S, vals, shift=shift, garbage_nulls=True), t.name_to_index_map(), GATES["330"])
    assert got == _want(vals, _names(t), ot, GATES["330"])


def test_empty_column_and_errors(S, Z):
    from srj_b200 import _native as N
    from srj_b200.cast import CastStrings, Version
    t, _, info = Z
    assert _parse(S, info, _strings(S, []), t.name_to_index_map(), GATES["330"]) == []
    col = _strings(S, [b"2020-01-01"])
    with pytest.raises(N.CudfException):
        CastStrings.parseTimestampStrings(col, len(TG.ZONES), 0, t.name_to_index_map(), info, Version(0, 3, 3, 0))
    with pytest.raises(N.CudfException):
        CastStrings.parseTimestampStrings(S.ColumnVector.from_numpy(S.DType.INT32, np.zeros(1, np.int32)), 0, 0, t.name_to_index_map(), info,
                                          Version(0, 3, 3, 0))
    bad_map = S.ColumnView.makeStructView(t.name_to_index_map().children[1], t.name_to_index_map().children[0])
    with pytest.raises(N.CudfException):
        CastStrings.parseTimestampStrings(col, 0, 0, bad_map, info, Version(0, 3, 3, 0))
    with pytest.raises(TypeError):
        CastStrings.parseTimestampStrings(None, 0, 0, t.name_to_index_map(), info, Version(0, 3, 3, 0))
    with pytest.raises(ValueError):
        CastStrings.toTimestamp(col, "Nowhere/City", False, Version(0, 3, 3, 0), t)
    assert CastStrings.toDate(_strings(S, []), True).size == 0
    no_chars = _strings(S, [b"2020-01-01", b""])
    no_chars.data = None                                 # offsets that span bytes, but no chars buffer
    with pytest.raises(N.CudfException):
        CastStrings.parseTimestampStrings(no_chars, 0, 0, t.name_to_index_map(), info, Version(0, 3, 3, 0))
    with pytest.raises(N.CudfException):
        CastStrings.toDate(no_chars, False)
    empties = _strings(S, [b"", b""])                   # rows that hold no chars may come without a chars buffer
    empties.data = None
    assert CastStrings.toDate(empties, False).getNullCount() == 2


def test_to_timestamp_goldens_and_ansi(S, Z):
    from srj_b200.cast import CastStrings, Version
    t = Z[0]
    vals = [s.encode() for s, _ in G.TO_TIMESTAMP]
    got = CastStrings.toTimestamp(_strings(S, vals), "Z", False, Version(0, 3, 3, 0), t)
    data = got.data.cpu().numpy().view(np.int64)
    valid = np.unpackbits(got.mask.cpu().numpy().view(np.uint8), bitorder="little")[:len(vals)].astype(bool)
    for (s, want), v, ok in zip(G.TO_TIMESTAMP, data, valid):
        assert (int(v) if ok else None) == want, s
    assert CastStrings.toTimestamp(_strings(S, vals), "Z", True, Version(0, 3, 3, 0), t) is None
    good = [s.encode() for s, w in G.TO_TIMESTAMP if w is not None]
    assert CastStrings.toTimestamp(_strings(S, good + [None]), "Z", True, Version(0, 3, 3, 0), t).getNullCount() == 1


def test_to_timestamp_across_dst_in_every_zone(S, Z):
    """End to end against the table: local wall times around each zone's transitions, named in the string and as the
    session zone."""
    from srj_b200.cast import CastStrings, Version
    t, ot, _ = Z
    vals, want = [], []
    for z, name in enumerate(TG.ZONES):
        utc, local, off, rules = ot.zone(z)
        picks = [int(x) for x in local[1:][(local[1:] > -2_000_000_000) & (local[1:] < 4_000_000_000)][-6:]] or [0]
        for inst in picks:
            for d in (-3601, -1, 0, 1, 3599, 86400 * 200):
                s = inst + d
                days, sec = divmod(s, 86400)
                y, m, dd = _civil(days)
                text = b"%04d-%02d-%02d %02d:%02d:%02d %s" % (y, m, dd, sec // 3600, sec // 60 % 60, sec % 60, name.encode())
                vals.append(text)
                conv = s - int(OTZ.zone_offset(OTZ.TO_UTC, [s], utc, local, off, rules)[0])
                want.append(conv * 10**6)
    got = CastStrings.toTimestamp(_strings(S, vals), "UTC", False, Version(0, 3, 5, 0), t)
    assert got.getNullCount() == 0
    assert got.data.cpu().numpy().view(np.int64).tolist() == want


def _civil(days):
    import datetime as dt
    d = dt.date(1970, 1, 1) + dt.timedelta(days=int(days))
    return d.year, d.month, d.day


def test_to_date_goldens_mask_and_ansi(S):
    from srj_b200.cast import CastStrings
    vals = [None if s is None else s.encode() for s, _ in G.TO_DATE]
    got = CastStrings.toDate(_strings(S, vals), False)
    data = got.data.cpu().numpy().view(np.int32)
    valid = np.unpackbits(got.mask.cpu().numpy().view(np.uint8), bitorder="little")[:len(vals)].astype(bool)
    assert [int(v) if ok else None for v, ok in zip(data, valid)] == [w for _, w in G.TO_DATE]
    assert got.getNullCount() == sum(w is None for _, w in G.TO_DATE)
    assert CastStrings.toDate(_strings(S, [b"2025", b"2025x"]), True) is None
    assert CastStrings.toDate(_strings(S, [b"2025", None]), True).getNullCount() == 1


@pytest.mark.parametrize("n", ROWS + [100_003])
def test_generated_dates_match_oracle(S, n):
    from srj_b200.cast import CastStrings
    rng = random.Random(n)
    vals = [None if i % 41 == 5 else GEN.date(rng) for i in range(n)]
    got = CastStrings.toDate(_strings(S, vals, shift=n % 3, garbage_nulls=True), False)
    want = [OC.parse_date(v) for v in vals]
    data = got.data.cpu().numpy().view(np.int32)
    words = (got.mask.cpu().numpy().view(np.uint8) if got.mask is not None else np.full((n + 31) // 32 * 4, 255, np.uint8))
    valid = np.unpackbits(words, bitorder="little")[:n].astype(bool)
    assert [int(v) if ok else None for v, ok in zip(data, valid)] == want
    assert all(int(v) == 0 for v, ok in zip(data, valid) if not ok)
    assert got.getNullCount() == sum(w is None for w in want)


def test_large_column_and_four_streams(S, Z):
    import torch
    from srj_b200.cast import CastStrings, Version
    t, ot, info = Z
    base = [b"2023-11-05 03:04:55.123456 +01:00", b"2024-02-29T12:00:00 Asia/Kolkata", b"bogus", b"1970-01-01"]
    n = 10_000_000                                        # 4 strings repeated: row r is base[r % 4]
    lens = np.array([len(b) for b in base], np.int64)
    offs = np.concatenate([[0], np.cumsum(np.tile(lens, n // 4))]).astype(np.int32)
    col = S.ColumnVector.from_numpy(S.DType.STRING, np.tile(np.frombuffer(b"".join(base), np.uint8), n // 4), None, offs, size=n)
    names = _names(t)
    want4 = _want(base, names, ot, GATES["330"])
    errors = []

    def run(k):
        try:
            with torch.cuda.stream(torch.cuda.Stream()):
                got = CastStrings.parseTimestampStrings(col, 1, 0, t.name_to_index_map(), info, Version(0, 3, 3, 0), now=NOW)
                for j, (c, d) in enumerate(zip(got.children, (np.uint8, np.int64, np.int32, np.uint8, np.int32, np.int32))):
                    a = c.data.cpu().numpy().view(d)
                    for r in range(4):
                        vals = a[r::4]
                        if not (vals == want4[r][j]).all():
                            errors.append((k, j, r))
        except Exception as e:                           # noqa: BLE001
            errors.append(e)
    ts = [threading.Thread(target=run, args=(k,)) for k in range(4)]
    for th in ts:
        th.start()
    for th in ts:
        th.join()
    assert not errors, errors[:4]
