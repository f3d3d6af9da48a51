"""CPU checks of the time zone oracle and of TimeZoneTable: the oracle reproduces the reference's TimeZoneTest values; a
table built from the system's TZif files, run through the oracle, agrees with an independent zoneinfo model around every
transition of 1900-2300 and at random instants; the POSIX footer becomes Java's rules; the documented quirks hold."""
import os
import sys
import zlib

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "spark-rapids-jni_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

from golden import timezone_golden as G                 # noqa: E402
from oracle import timezone as OT                       # noqa: E402
import timezone_model as M                              # noqa: E402

ZONEINFO = "/usr/share/zoneinfo"
ALIAS = {"US/Pacific": "America/Los_Angeles"}


def _golden():
    from srj_b200.timezone import TimeZoneTable
    t = TimeZoneTable(G.ZONES, G.ENTRIES, G.RULES)
    return t, OT.Table(*t.arrays())


@pytest.mark.parametrize("case", G.JAVA_CASES, ids=[c[0] for c in G.JAVA_CASES])
def test_oracle_reproduces_the_reference_tests(case):
    name, type_id, direction, zone, inp, exp = case
    t, tbl = _golden()
    valid = np.array([v is not None for v in inp])
    got = OT.convert(direction, type_id, np.array([v or 0 for v in inp], np.int64), tbl, t.index(ALIAS.get(zone, zone)))
    assert np.array_equal(got[valid], np.array([e for e in exp if e is not None], np.int64))


def _system_table(zones):
    from srj_b200.timezone import TimeZoneTable
    if not os.path.isdir(ZONEINFO) or not all(M.available(z) and os.path.exists(os.path.join(ZONEINFO, z)) for z in zones):
        pytest.skip("tzdata is not installed")
    t = TimeZoneTable.from_zoneinfo(zones, ZONEINFO)
    return t, OT.Table(*t.arrays())


@pytest.mark.parametrize("zone", G.ZONES)
def test_table_and_oracle_agree_with_zoneinfo_at_every_transition(zone):
    t, tbl = _system_table([zone])
    trans = M.transitions(zone, 1900, 2300)
    utc = np.array(sorted({s + d for s in trans for d in (-3601, -1, 0, 1, 3600)} | {0}), np.int64)
    got = OT.convert(OT.FROM_UTC, OT.TIMESTAMP_SECONDS, utc, tbl, 0)
    want = np.array([M.from_utc(zone, s) for s in utc], np.int64)
    assert np.array_equal(got, want), [(int(s), int(g), int(w)) for s, g, w in zip(utc, got, want) if g != w][:5]
    # local times on both sides of each transition's wall clocks, and inside its gap or overlap
    local = np.array(sorted({v for s in trans for o in (M.from_utc(zone, s - 1) - (s - 1), M.from_utc(zone, s) - s)
                             for d in (-1, 0, 1, 1799, 3599, 3600) for v in (s + o + d, s + o - d)}), np.int64)
    got = OT.convert(OT.TO_UTC, OT.TIMESTAMP_SECONDS, local, tbl, 0)
    want = np.array([M.to_utc(zone, s) for s in local], np.int64)
    assert np.array_equal(got, want), [(int(s), int(g), int(w)) for s, g, w in zip(local, got, want) if g != w][:5]


@pytest.mark.parametrize("zone", G.ZONES)
def test_table_and_oracle_agree_with_zoneinfo_at_random_instants(zone):
    t, tbl = _system_table([zone])
    rng = np.random.default_rng(zlib.crc32(zone.encode()))
    lo, hi = -2208988800, 10413792000                       # 1900-01-01 .. 2300-01-01
    s = rng.integers(lo, hi, 100_000, dtype=np.int64)
    got = OT.convert(OT.FROM_UTC, OT.TIMESTAMP_SECONDS, s, tbl, 0)
    assert np.array_equal(got, np.array([M.from_utc(zone, v) for v in s], np.int64))
    got = OT.convert(OT.TO_UTC, OT.TIMESTAMP_SECONDS, s, tbl, 0)
    assert np.array_equal(got, np.array([M.to_utc(zone, v) for v in s], np.int64))


def test_posix_footers_become_java_rules():
    from srj_b200.timezone import posix_rules
    # Dublin's footer starts with the October rule (negative DST); the rules come back in calendar order
    assert posix_rules("IST-1GMT0,M10.5.0,M3.5.0/1") == [3, 25, 6, 3600, 0, 3600, 10, 25, 6, 7200, 3600, 0]
    assert posix_rules("PST8PDT,M3.2.0,M11.1.0") == [3, 8, 6, 7200, -28800, -25200, 11, 1, 6, 7200, -25200, -28800]
    # Nuuk's rule times are negative; a last-weekday-of-February rule keeps -1
    assert posix_rules("<-02>2<-01>,M3.5.0/-1,M10.5.0/0")[:6] == [3, 25, 6, -3600, -7200, -3600]
    assert posix_rules("XST3XDT,M2.5.1,M11.1.0")[:3] == [2, -1, 0]
    assert posix_rules("<+0545>-5:45") == [] and posix_rules("UTC0") == []
    for bad in ("EST5EDT,J60,J300", "EST5EDT,60,300", "EST5EDT"):
        with pytest.raises(ValueError):
            posix_rules(bad)


def test_rules_with_a_negative_day_of_month_count_from_the_end():
    # the kernel takes both forms: dom -1 / previous-or-same and minLength - 6 / next-or-same name the same Sunday
    years = np.arange(1900, 2301)
    last = OT.rule_instant(years, (10, -1, 6, 7200, 3600, 0))
    assert np.array_equal(last, OT.rule_instant(years, (10, 25, 6, 7200, 3600, 0)))
    assert np.all(OT.weekday(last // 86400) == 6)


def test_quirks():
    t, tbl = _golden()
    la = t.index("America/Los_Angeles")
    utc, local, off, rules = tbl.zone(la)
    # truncating seconds: a negative sub-second value just below an instant takes the offset at the instant
    neg = [i for i, v in enumerate(utc) if v < 0 and i > 0][-1]
    us = np.array([utc[neg] * 10**6 - 1, utc[neg] * 10**6 - 10**6], np.int64)
    got = OT.convert(OT.FROM_UTC, OT.TIMESTAMP_MICROSECONDS, us, tbl, la)
    assert got[0] - us[0] == int(off[neg]) * 10**6 and got[1] - us[1] == int(off[neg - 1]) * 10**6
    # the micros overflow test at the minimum second: >= 224192 overflows, below wraps
    res, ovf = OT.add_micros(np.array([-(2**63 // 10**6) - 1] * 2, np.int64), np.array([224191, 224192]))
    assert list(ovf) == [False, True]
    # ORC: from the last transition on, the raw offset
    t_ms, o_ms = np.array([0, 1000], np.int64), np.array([3600000, 7200000], np.int32)
    assert list(OT.orc_offset(t_ms, o_ms, 5, np.array([-1, 0, 999, 1000, 5000]))) == [5, 3600000, 3600000, 5, 5]
