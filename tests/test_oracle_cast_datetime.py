"""CPU: the restatement of CastStrings' timestamp and date parses (oracle/cast_datetime.py) against the literal cases of
the reference's CastStringsTest, and against the zone table for the time-alone rows that name a zone."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from golden import cast_datetime_golden as G          # noqa: E402
from golden import timezone_golden as TG              # noqa: E402
from oracle import cast_datetime as OC                # noqa: E402
from oracle import timezone as OTZ                    # noqa: E402

import datetime as dt                                  # noqa: E402

GATES_330 = OC.version_gates(0, 3, 3, 0)


def _table():
    sys.path.insert(0, os.path.join(ROOT, "spark-rapids-jni_b200"))
    from srj_b200.timezone import TimeZoneTable
    return OTZ.Table(*TimeZoneTable(TG.ZONES, TG.ENTRIES, TG.RULES).arrays())


@pytest.mark.parametrize("rows", ["JUST_TIME", "FIRST_PHASE"])
def test_oracle_first_phase_goldens(rows):
    for case in getattr(G, rows):
        s, want = case[0], tuple(case[1:])
        got = OC.parse_timestamp(s.encode(), G.DEFAULT_TZ_INDEX, G.DEFAULT_EPOCH_DAY, G.NAME_MAP, None, 0, *GATES_330)
        assert got == want, s


def test_oracle_to_date_goldens():
    for s, want in G.TO_DATE:
        assert OC.parse_date(None if s is None else s.encode()) == want, s


def test_oracle_date_matches_python_calendar():
    d0 = dt.date(1970, 1, 1)
    for y in (1, 4, 100, 400, 1582, 1900, 1970, 2000, 2024, 9999):
        for m in range(1, 13):
            for d in (1, 15, 28):
                assert OC.parse_date(b"%04d-%02d-%02d" % (y, m, d)) == (dt.date(y, m, d) - d0).days


def test_version_gates():
    assert OC.version_gates(0, 3, 2, 0) == (True, False)
    assert OC.version_gates(0, 3, 5, 1) == (False, False)
    assert OC.version_gates(0, 4, 0, 0) == (False, True)
    assert OC.version_gates(1, 3, 2, 0) == (False, False)
    assert OC.version_gates(1, 14, 3, 0) == (False, True)
    assert OC.version_gates(1, 13, 3, 9) == (False, False)


def test_oracle_spark_320_and_400_gates():
    ok = lambda s, g: OC.parse_timestamp(s, 1, 0, G.NAME_MAP, None, 0, *g)  # noqa: E731
    assert ok(b"2023-11-05 03:04:55+01:02", (True, False))[3:5] == (1, 3720)
    assert ok(b"2023-11-05 03:04:55-01:02", (True, False))[3:5] == (1, 0)       # the sign is read as (b == '+')
    assert ok(b"2023-11-05 03:04:55 +1:2", (True, False))[0] == 1                # 3.2.0 rejects a one-digit minute
    assert ok(b"2023-11-05 03:04:55 +1:2", (False, False))[0] == 0
    assert ok(b" T01:02:03", (False, True))[0] == 1                              # SPARK-52351
    assert ok(b"T01:02:03", (False, True))[0] == 0


def test_oracle_just_time_named_zone_uses_the_table():
    table = _table()
    names = sorted((n.encode(), i) for i, n in enumerate(TG.ZONES))
    for zone in ("America/Los_Angeles", "Asia/Shanghai", "Pacific/Kiritimati"):
        z = TG.ZONES.index(zone)
        for now in (0, 1699153495, 1711846800, 4102444800 + 12345):
            got = OC.parse_timestamp(b"T01:02:03 " + zone.encode(), 0, 0, names, table, now, *GATES_330)
            utc, local, off, rules = table.zone(z)
            loc = now + int(OTZ.zone_offset(OTZ.FROM_UTC, [now], utc, local, off, rules)[0])
            day = abs(loc) // 86400 * (1 if loc >= 0 else -1)          # the reference's day: truncated toward zero
            assert got == (0, day * 86400 + 3723, 0, 2, 0, z)


# ---- the independent model (tests/cast_datetime_model.py) against the restatement and the goldens ----------------------
import random                                          # noqa: E402

import cast_datetime_gen as GEN                        # noqa: E402
import cast_datetime_model as CM                       # noqa: E402
import timezone_model as TZM                           # noqa: E402

GATES = {"320": (0, 3, 2, 0), "330": (0, 3, 3, 0), "400": (0, 4, 0, 0), "db143": (1, 14, 3, 0), "db133": (1, 13, 3, 0)}
NOW = 1_760_000_000


def _agree(model, oracle_row):
    valid, row = model
    if valid or row is not None:
        return row == oracle_row
    return oracle_row[0] == 1


def _names_dict():
    sys.path.insert(0, os.path.join(ROOT, "spark-rapids-jni_b200"))
    from srj_b200.timezone import TimeZoneTable
    return {k.encode(): v for k, v in TimeZoneTable(TG.ZONES, TG.ENTRIES, TG.RULES).name_to_index().items()}


@pytest.mark.parametrize("rows", ["JUST_TIME", "FIRST_PHASE"])
def test_model_first_phase_goldens(rows):
    names = dict(G.NAME_MAP)
    for case in getattr(G, rows):
        got = CM.timestamp(case[0].encode(), G.DEFAULT_TZ_INDEX, G.DEFAULT_EPOCH_DAY, names, None, 0, False, False)
        assert _agree(got, tuple(case[1:])), case[0]


def test_model_to_date_goldens():
    for s, want in G.TO_DATE:
        assert CM.date(None if s is None else s.encode()) == want, s


def test_model_civil_days_match_the_restatement():
    rng = random.Random(3)
    for _ in range(20_000):
        y, m = rng.randint(-10**7, 10**7), rng.randint(1, 12)
        d = rng.randint(1, 28)
        assert CM.days_from_civil(y, m, d) == int(OTZ.epoch_day(y, m, d)), (y, m, d)


@pytest.mark.parametrize("gate", sorted(GATES))
def test_model_oracle_agree_on_generated_strings(gate):
    if not TZM.available("America/Los_Angeles"):
        pytest.skip("no tzdata")
    names = _names_dict()
    table = _table()
    pairs = sorted(names.items())
    g320, g400 = OC.version_gates(*GATES[gate])
    rng = random.Random(sum(gate.encode()) * 7)
    strings = [GEN.timestamp(rng, [k.decode() for k in names]) for _ in range(40_000)]
    strings += [c + s for c in GEN.TRIM for s in (b"2023-11-05 03:04:55", b"T01:02")]       # every trim byte, leading
    strings += [s + c for c in GEN.TRIM for s in (b"2023-11-05 03:04:55", b"1:2")]           # and trailing
    strings += [b"%s-%s-%s %s:%s:%s" % tuple(b"7" * n for n in ns) for ns in
                [(a, b, c, d, e, f) for a in range(1, 8) for b in (1, 2, 3) for c in (1, 2, 3) for d in (1, 2, 3)
                 for e in (1, 2) for f in (1, 2, 3)]]                                          # 1-7 digit segments
    strings += [b"2023-11-05%s03:04:55%s%s" % (sep, sp, z.encode()) for sep in (b" ", b"T") for sp in (b"", b" ")
                for z in GEN.ZONE_FORMS + ["Nowhere/City", "Asia/Tokyo", "PST", "Z"]]         # every zone form
    for s in strings:
        want = OC.parse_timestamp(s, 3, -5, pairs, table, NOW, g320, g400)
        assert _agree(CM.timestamp(s, 3, -5, names, TG.ZONES, NOW, g320, g400), want), (s, want)


def test_model_oracle_agree_on_generated_dates():
    rng = random.Random(11)
    for _ in range(40_000):
        s = GEN.date(rng)
        assert CM.date(s) == OC.parse_date(s), s
