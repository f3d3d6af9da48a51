"""CPU checks of oracle/decimal.py: the reference's DecimalUtilsTest cases and hand-derived edges; agreement with the
independent decimal-module model on random rows over a scale grid, the reference's quirks enumerated rather than skipped;
and the limb division with host-computed reciprocals (csrc/decimal_arith.cuh, compiled here as plain C++) against
Python's // and % for every power of ten the kernels divide by."""
import os
import shutil
import subprocess
import tempfile
import numpy as np
import pytest

import decimal_model as MD
from golden import decimal_golden as G
from oracle import decimal as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "spark-rapids-jni_b200", "csrc")


def _parse(s):
    """Java BigDecimal string -> (unscaled, cudf scale)"""
    whole, _, frac = s.partition(".")
    return int(whole + frac), -len(frac)


def _golden_rows():
    for op, aa, bb, so, cast, want in G.REFERENCE + G.HAND:
        for i, (x, y) in enumerate(zip(aa, bb if len(bb) == len(aa) else bb * len(aa))):
            yield op, x, y, so, cast, want[i]


@pytest.mark.parametrize("case", list(_golden_rows()), ids=lambda c: f"op{c[0]}:{c[1]}:{c[2]}")
def test_oracle_matches_goldens(case):
    op, x, y, so, cast, (ovf, exp) = case
    (a, sa), (b, sb) = _parse(x), _parse(y)
    got_ovf, got = O.row(op, a, b, sa, sb, so, cast)
    assert got_ovf == ovf
    if exp is None:
        return
    if isinstance(exp, int):
        assert got == exp
    else:
        v, s = _parse(exp)
        assert (got * 10 ** (so - s) == v) if so >= s else (got == v * 10 ** (s - so))


# (a_scale, b_scale, out_scale): Spark's result scales and positive cudf scales
MODEL_GRID = {
    O.MULTIPLY: [(-10, -10, -6), (-2, -2, -4), (0, 0, 0), (-5, -3, -10), (2, 1, 0), (-19, -19, -2), (-1, 0, -30)],
    O.DIVIDE: [(-10, -10, -6), (-2, -5, -10), (0, -38, -38), (-6, -2, -20), (2, -3, 0), (-1, -1, 10), (0, 0, -39), (4, 0, 0)],
    O.INTEGER_DIVIDE: [(-10, -10, 0), (-2, -5, 0), (2, -3, 0), (0, 0, 0)],
    O.REMAINDER: [(-2, -3, -3), (-3, -2, -3), (-10, -10, -10), (0, 3, 0), (2, 0, 0), (0, -20, -20)],
    O.ADD: [(-10, -2, -10), (-2, -10, -6), (0, 0, 0), (3, -3, -5), (-38, 38, -38), (-1, -1, 2)],
}
MODEL_GRID[O.SUBTRACT] = MODEL_GRID[O.ADD]
ROWS_PER_OP = 100_000


def _rand(rng, n):
    digits = rng.integers(1, 39, n)
    mags = [int.from_bytes(rng.bytes(16), "little") % 10 ** int(d) for d in digits]
    return [-m if s else m for m, s in zip(mags, rng.random(n) < 0.5)]


# the quirks each op must reach on its grid, and where oracle and model must then differ
EXPECTED_QUIRKS = {(O.MULTIPLY, True): {"interim", "pow10"}, (O.MULTIPLY, False): {"pow10"}}
CASES = [(op, cast) for op in sorted(MODEL_GRID) for cast in ((True, False) if op == O.MULTIPLY else (True,))]


@pytest.mark.parametrize("op,cast", CASES)
def test_oracle_agrees_with_the_model(op, cast):
    rng = np.random.default_rng(op)
    grid = MODEL_GRID[op]
    per = ROWS_PER_OP // len(grid) + 1
    reached, differs = {}, {}
    for sa, sb, so in grid:
        a, b = _rand(rng, per), _rand(rng, per)
        b[:3] = [0, 1, -1]
        a[:4] = [10**37, -10**37, 10**38 - 1, 0]
        for x, y in zip(a, b):
            q = MD.quirk(op, x, y, sa, sb, so, cast)
            f, v = MD.model(op, x, y, sa, sb, so)
            want = (f, O.s64(v) if op == O.INTEGER_DIVIDE else O.s128(v))   # an overflowing row keeps the low bits
            got = O.row(op, x, y, sa, sb, so, cast)
            if q is None:
                assert got == want, (op, cast, x, y, sa, sb, so)
            else:
                reached[q] = reached.get(q, 0) + 1
                differs[q] = differs.get(q, 0) + (got != want)
    expected = EXPECTED_QUIRKS.get((op, cast), set())
    for q in expected:
        assert reached.get(q, 0) > 0 and differs.get(q, 0) > 0, (q, reached, differs)
    assert set(reached) <= expected | {"wrap"}, reached


def test_interim_cast_quirk_is_the_documented_one():
    a, b = -85334448647530481077706777111312637916, -120000000000
    assert O.multiply(a, b, -10, -10, -6, True) == (False, 102401338377036577293248132533575166)
    assert O.multiply(a, b, -10, -10, -6, False) == MD.model(O.MULTIPLY, a, b, -10, -10, -6) == \
        (False, 102401338377036577293248132533575165)


def test_precision10_power_of_ten_edges():
    for k in range(77):
        assert O.precision10(10**k) == k and O.precision10(-(10**k)) == k
        assert O.precision10(10**k + 1) == k + 1 if k < 76 else O.precision10(10**k + 1) == -1
        if k:
            assert O.precision10(10**k - 1) == k
    assert O.precision10(0) == 0 and O.precision10(1) == 0 and O.precision10(2**255) == -1


HARNESS = r"""
#include <cstdio>
#include <cstring>
#include "decimal_arith.cuh"
using namespace srj::dec;
static uint64_t hex64(const char* s) { uint64_t v = 0; for (int i = 0; i < 16; ++i) v = v * 16 + (s[i] <= '9' ? s[i] - '0' : s[i] - 'a' + 10); return v; }
int main() {
  int k; char a[80];
  while (scanf("%d %64s", &k, a) == 2) {
    u128 d = 1;
    for (int i = 0; i < k; ++i) d *= 10;
    const Div D = make_div(d);                    // the reciprocal the host computes for a call's fixed 10^k
    U256 n;
    for (int i = 0; i < 4; ++i) n.w[i] = hex64(a + 48 - 16 * i);
    u128 r;
    const U256 q = udivrem(n, D, &r);
    printf("%016llx%016llx%016llx%016llx %016llx%016llx\n", (unsigned long long)q.w[3], (unsigned long long)q.w[2], (unsigned long long)q.w[1],
           (unsigned long long)q.w[0], (unsigned long long)(uint64_t)(r >> 64), (unsigned long long)(uint64_t)r);
  }
}
"""


def test_host_reciprocals_divide_exactly():
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    rng = np.random.default_rng(38)
    with tempfile.TemporaryDirectory() as td:
        src, exe = os.path.join(td, "h.cpp"), os.path.join(td, "h")
        open(src, "w").write(HARNESS)
        r = subprocess.run([gxx, "-std=c++17", "-O2", "-I", CSRC, src, "-o", exe], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        for k in range(39):
            ns = [int.from_bytes(rng.bytes(32), "little") >> int(s) for s in rng.integers(0, 256, 100_000)]
            ns[:4] = [0, 10**k - 1, 10**k, (1 << 256) - 1]
            out = subprocess.run([exe], input="".join(f"{k} {n:064x}\n" for n in ns), capture_output=True, text=True).stdout.split()
            d = 10**k
            for i, n in enumerate(ns):
                assert (int(out[2 * i], 16), int(out[2 * i + 1], 16)) == (n // d, n % d), (k, n)
