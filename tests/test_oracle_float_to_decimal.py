"""CPU checks of the floatingPointToDecimal oracles: the Python restatement (oracle/float_to_decimal.py) and the C one
(oracle/float_to_decimal.c) hold the goldens, agree with each other on over 10^6 rows that reach every path of the reference's
shifting, and agree with an independent model of Spark's intent (tests/float_to_decimal_model.py) except on named classes
of rows, each given by a predicate: every class is reached, and no disagreement falls outside them."""
import collections

import numpy as np
import pytest

import float_to_decimal_model as M
from golden import float_to_decimal_golden as G
from oracle import float_to_decimal as D

DEC32, DEC64, DEC128 = D.F2D_DECIMAL32, D.F2D_DECIMAL64, D.F2D_DECIMAL128


def _ints(out, out_type):
    return D.to_ints(out.reshape(-1)) if out_type == DEC128 else [int(v) for v in out]


@pytest.mark.parametrize("case", range(len(G.CASES)), ids=[c[0] for c in G.CASES])
def test_goldens(case):
    name, values, out_type, precision, scale, want, failed = G.CASES[case]
    x = np.array(values, np.float32 if name.startswith("f32") else np.float64)
    vals, ok, first = D.floating_point_to_decimal(x, None, out_type, precision, scale)
    assert [v if o else None for v, o in zip(vals, ok)] == want and (first >= 0) == failed
    cvals, cok, cfirst = D.floating_point_to_decimal_c(x, None, out_type, precision, scale)
    assert _ints(cvals, out_type) == vals and np.array_equal(cok, ok) and cfirst == first


def _inputs(rng, n):
    """Random bit patterns, log-uniform magnitudes, k / 10^d, denormals, whole numbers about 2^53 and 2^63, and the
    DECIMAL128 can_round edge."""
    bits = rng.integers(0, 1 << 64, n, dtype=np.uint64).view(np.float64)
    mags = 10.0 ** rng.uniform(-330, 308, n) * rng.choice([-1.0, 1.0], n)
    small = 10.0 ** rng.uniform(-12, 45, n) * rng.choice([-1.0, 1.0], n)
    kd = np.round(rng.uniform(-1, 1, n) * 10.0 ** rng.integers(0, 17, n)) / 10.0 ** rng.integers(0, 20, n)
    den = rng.integers(1, 1 << 52, n // 8, dtype=np.uint64).view(np.float64)
    whole = np.concatenate([2.0 ** 53 + np.arange(-8, 8), 2.0 ** 63 * np.array([1 - 2 ** -53, 1.0, 1 + 2 ** -52, 2.0])])
    edge = np.concatenate([2.0 ** 127 / 10.0 / 10.0 ** s * np.array([1 - 2 ** -52, 1.0, 1 + 2 ** -52]) for s in range(0, 39, 5)])
    return np.concatenate([bits, mags, small, kd, den, -den, whole, -whole, edge, [0.0, -0.0, np.nan, np.inf, -np.inf]])


def test_c_and_python_oracles_agree_on_every_path(monkeypatch):
    seen = collections.Counter()
    for name in ("_pospow", "_negpow"):
        fn = getattr(D, name)

        def counted(base2, pow2, p, ub, fn=fn, name=name):
            seen[(name, (abs(p) - 1) // 18)] += 1                        # the number of 18-digit steps
            return fn(base2, pow2, p, ub)
        monkeypatch.setattr(D, name, counted)
    ipow = D.ipow10

    def counted_ipow(k, bits):
        r = ipow(k, bits)
        seen["zero_power" if r == 0 else "negative_power" if k < 0 else "power"] += 1
        return r
    monkeypatch.setattr(D, "ipow10", counted_ipow)
    rng = np.random.default_rng(2024)
    rows = 0
    for out_type in (DEC32, DEC64, DEC128):
        p = D.F2D_MAX_PRECISION[out_type]
        for scale in sorted({-p, -(p // 2), -2, 0, 1, 2, 19, 20, 37, 38}):
            for f32 in (False, True):
                x = _inputs(rng, 4000)
                if f32:
                    with np.errstate(over="ignore", invalid="ignore"):
                        x = x.astype(np.float32)
                want, ok, first = D.floating_point_to_decimal(x, None, out_type, p, scale)
                got, cok, cfirst = D.floating_point_to_decimal_c(x, None, out_type, p, scale)
                assert np.array_equal(cok, ok) and cfirst == first, (out_type, scale, f32)
                assert _ints(got, out_type) == want, (out_type, scale, f32)
                rows += len(x)
    assert rows > 10 ** 6
    for key in [("_pospow", 0), ("_pospow", 1), ("_pospow", 2), ("_negpow", 0), ("_negpow", 1), ("_negpow", 2), "zero_power",
                "negative_power"]:
        assert seen[key] > 0, key


# Where the reference (and so the oracle) and Spark's intent part, by class.  g is the oracle's value (None: null), m
# the model's; both are unscaled integers at the Spark scale s.
def _quirk(out_type, spark_scale, g, m):
    if g is not None and m is None:
        # the exact result has more than p digits, but the reference's fixed-width steps wrap it to a value inside the
        # bound (the int64 cast of the magnitude, ipow wrapping to 0 and zeroing it, the 32-bit helper's 0 past 10^9)
        return "wrap_inside_bound"
    if g is not None and m is not None:
        if out_type == DEC32 and spark_scale < 0:
            # a legacy negative scale gives DECIMAL32 a scale factor of 0 (the 32-bit switch), so every row takes the
            # int32 intermediate, which wraps for the larger values
            return "dec32_legacy_int32_wrap"
        big = max(abs(g), abs(m))
        if abs(g - m) <= 10 ** max(len(str(big)) - 15, 0):
            # the reference keeps the binary value's digits past the shortest decimal string, which the model rounds
            # from; they differ from the 16th significant digit on
            return "digits_past_the_shortest_string"
    return None


def test_oracle_and_spark_model_differ_only_in_named_classes():
    rng = np.random.default_rng(3)
    classes = collections.Counter()
    outside = []
    for out_type in (DEC32, DEC64, DEC128):
        p = D.F2D_MAX_PRECISION[out_type]
        for spark_scale in sorted({p, p // 2, 2, 0, -2, -10, -38}):
            for f32 in (False, True):
                x = np.concatenate([10.0 ** rng.uniform(-12, 45, 1500) * rng.choice([-1.0, 1.0], 1500),
                                    np.round(rng.uniform(-1, 1, 1500) * 10.0 ** rng.integers(0, 17, 1500)) / 10.0 ** rng.integers(0, 20, 1500)])
                if f32:
                    with np.errstate(over="ignore"):
                        x = x.astype(np.float32)
                vals, ok, _ = D.floating_point_to_decimal(x, None, out_type, p, -spark_scale)
                for xi, v, o in zip(x.tolist(), vals, ok):
                    g, m = (v if o else None), M.cast(xi, p, spark_scale)
                    if g == m:
                        classes["agree"] += 1
                        continue
                    c = _quirk(out_type, spark_scale, g, m)
                    classes[c] += 1
                    if c is None:
                        outside.append((out_type, f32, spark_scale, xi, g, m))
    assert not outside, outside[:10]
    for c in ("wrap_inside_bound", "dec32_legacy_int32_wrap", "digits_past_the_shortest_string"):
        assert classes[c] > 0, c
    assert classes["agree"] > 10 * sum(v for k, v in classes.items() if k != "agree") / 3
