"""Independent model of the time zone conversions: java.time's semantics through Python's zoneinfo, which reads the
system's tzdata.  A local time in a gap is moved forward (converted with the offset before it) and one in an overlap
takes the earlier offset, as ZonedDateTime.of does; zoneinfo gives both with fold=0.  Whole seconds only."""
import datetime as dt

try:
    import zoneinfo
except ImportError:                       # pragma: no cover
    zoneinfo = None

EPOCH = dt.datetime(1970, 1, 1)


def available(name: str) -> bool:
    if zoneinfo is None:
        return False
    try:
        zoneinfo.ZoneInfo(name)
        return True
    except Exception:
        return False


def to_utc(name: str, local_seconds: int) -> int:
    """UTC seconds of a local date-time of the zone, given as seconds since 1970-01-01T00:00 local."""
    z = zoneinfo.ZoneInfo(name)
    local = (EPOCH + dt.timedelta(seconds=int(local_seconds))).replace(tzinfo=z, fold=0)
    return int(local_seconds) - int(local.utcoffset().total_seconds())


def from_utc(name: str, utc_seconds: int) -> int:
    """Local seconds of a UTC instant in the zone."""
    z = zoneinfo.ZoneInfo(name)
    utc = (EPOCH + dt.timedelta(seconds=int(utc_seconds))).replace(tzinfo=dt.timezone.utc)
    return int(utc_seconds) + int(utc.astimezone(z).utcoffset().total_seconds())


def transitions(name: str, first_year: int, last_year: int):
    """Every UTC second in [first_year, last_year] at which the zone's offset changes, found by scanning day by day and
    bisecting each change to the second."""
    z = zoneinfo.ZoneInfo(name)
    off = lambda s: (EPOCH + dt.timedelta(seconds=s)).replace(tzinfo=dt.timezone.utc).astimezone(z).utcoffset()   # noqa: E731
    lo = int((dt.datetime(first_year, 1, 1) - EPOCH).total_seconds())
    hi = int((dt.datetime(last_year, 12, 31) - EPOCH).total_seconds())
    out = []
    step = 86400 * 7
    prev = off(lo)
    s = lo
    while s < hi:
        nxt = min(s + step, hi)
        cur = off(nxt)
        if cur != prev:
            a, b = s, nxt                                   # off(a) == prev != off(b)
            while b - a > 1:
                m = (a + b) // 2
                if off(m) == prev:
                    a = m
                else:
                    b = m
            out.append(b)
            prev = off(b)
            s = b
            continue
        s = nxt
    return out
