"""A grammar-driven generator of timestamp and date strings for the cast tests: every trim byte, 1 to 7 digit segments,
both date-time separators, every zone form (valid and not), names in and out of the map, and random damage."""
import random

TRIM = [bytes([c]) for c in list(range(0, 33)) + [127]]
ZONE_FORMS = ["Z", "+8", "-08", "+0830", "-083015", "+08:30", "+8:3", "-08:30:15", "+18:00", "+18:00:01", "+19:00", "+1:2:3",
              "UT", "UTC", "GMT", "GMT0", "GMT+", "UT+", "UTC-7", "GMT+08:00", "UT-8:1:08", "U", "Ux", "UTx", "UTCx", "Gx", "GMTx",
              "+", "-X", "+07:", "+09:x", "+111", "+11111", "+1x"]


def _num(rng, lo, hi):
    return str(rng.randint(0, 10**rng.randint(lo, hi) - 1)).zfill(rng.randint(lo, hi))


def timestamp(rng: random.Random, names) -> bytes:
    parts = []
    r = rng.random()
    if r < 0.1:
        t = "%s:%s" % (_num(rng, 1, 2), _num(rng, 1, 2))
        if rng.random() < 0.6:
            t += ":" + _num(rng, 1, 3)
        s = ("T" if rng.random() < 0.5 else "") + t
    else:
        y = rng.choice([_num(rng, 4, 4), _num(rng, 1, 7), str(rng.randint(1, 300001))])
        s = rng.choice(["", "", "", "+", "-"]) + y
        if rng.random() < 0.9:
            s += "-" + rng.choice([_num(rng, 1, 2), str(rng.randint(1, 12)), _num(rng, 1, 3)])
            if rng.random() < 0.9:
                s += "-" + rng.choice([str(rng.randint(1, 28)), _num(rng, 1, 2), _num(rng, 1, 3)])
                if rng.random() < 0.85:
                    s += rng.choice([" ", "T", "T", " "])
                    if rng.random() < 0.95:
                        s += "%s:%s:%s" % (rng.randint(0, 24), _num(rng, 1, 2), str(rng.randint(0, 60)).zfill(rng.randint(1, 2)))
                        if rng.random() < 0.5:
                            s += "." + _num(rng, 0, 9)
    if rng.random() < 0.5:
        z = rng.choice(ZONE_FORMS + list(names) + ["Nowhere/City", "America/Los_Angelesx"])
        s += rng.choice(["", " ", "  "]) + z
    b = s.encode()
    if rng.random() < 0.05 and b:
        i = rng.randrange(len(b))
        b = b[:i] + bytes([rng.randrange(256)]) + b[i + 1:]
    if rng.random() < 0.2:
        b = b"".join(rng.choice(TRIM) for _ in range(rng.randint(1, 3))) + b
    if rng.random() < 0.2:
        b = b + b"".join(rng.choice(TRIM) for _ in range(rng.randint(1, 3)))
    return b


def date(rng: random.Random) -> bytes:
    s = rng.choice(["", "", "+", "-"]) + _num(rng, 1, 8)
    if rng.random() < 0.85:
        s += "-" + _num(rng, 0, 3)
        if rng.random() < 0.85:
            s += "-" + _num(rng, 0, 3)
            if rng.random() < 0.3:
                s += rng.choice([" ", "T", "x", ":"]) + rng.choice(["", "12:00", "xyz"])
    b = s.encode()
    if rng.random() < 0.2:
        b = rng.choice(TRIM) + b + rng.choice(TRIM)
    return b
