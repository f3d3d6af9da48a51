"""GPU checks of Histogram.percentileFromHistogram at group-by scale and at the radix select's rank edges, against
tests/histogram_scale_model.py (pinned to oracle/histogram.py by tests/test_histogram_scale_model.py):

  * each tier's persistent grid just short of, at and past the rows of one sweep;
  * a million histograms of 1 to 16 elements, with P = 1, 3, 5, 7 and 101;
  * rows of all three tiers, null rows and empty rows in one call, and a slice of it;
  * one set of elements padded with nulls onto each tier, which must answer bit for bit alike;
  * ranks placed exactly on a cumulative-count boundary and one unit either side, with keys that differ only in their
    lowest or highest byte, keys in bins 0x00 and 0xff, and each type's extreme keys.

Both output shapes are checked: values bit for bit (a NaN matches any NaN), masks, list offsets and null counts."""
import numpy as np
import pytest

import histogram_scale_model as M
from test_gpu_histogram import BOOL8, FLOAT64, INT32, INT64, K, NP, _bits, _hist_view, _s, _same, _values

pytestmark = pytest.mark.gpu

INT8, INT16, UINT8, UINT16, UINT32, UINT64, FLOAT32 = 1, 2, 5, 6, 7, 8, 9
NAME = {INT8: "int8", INT16: "int16", INT32: "int32", INT64: "int64", UINT8: "uint8", UINT16: "uint16", UINT32: "uint32",
        UINT64: "uint64", FLOAT32: "float32", FLOAT64: "float64", BOOL8: "bool8"}
WARP_CAP = 256                                # kWarpCap: the longest row of the warp tier; longer rows up to K take a CTA


def _check(S, Hs, t, offsets, vals, valid, counts, pct, slice_from=0, want=None):
    """Both output shapes of one call against the model (or `want` = (values [rows, P], row_valid)); -> flat [rows, P]."""
    offs = np.asarray(offsets, np.int64)[slice_from:]
    rows, P = len(offs) - 1, len(pct)
    want, ok = want if want is not None else M.percentile(offs, vals, valid, counts, pct, bool8=t == BOOL8)
    nulls = rows - int(ok.sum())
    view = _hist_view(S, t, offsets, vals, valid, counts, slice_from)
    flat = Hs.percentileFromHistogram(view, pct, False)
    assert flat.size == rows * P and flat.getNullCount() == nulls * P
    assert np.array_equal(_bits(flat, rows * P), np.repeat(ok, P))
    got = flat.data.cpu().numpy().view(np.float64).reshape(rows, P)
    del flat
    assert _same(got, want)                                     # 0.0 under the null rows on both sides
    lists = Hs.percentileFromHistogram(view, pct, True)
    assert lists.size == rows and lists.getNullCount() == nulls
    assert np.array_equal(_bits(lists, rows), ok)
    assert np.array_equal(lists.offsets.cpu().numpy(), np.concatenate([[0], np.cumsum(ok)]) * P)
    assert _same(lists.child.data.cpu().numpy().view(np.float64), want[ok].reshape(-1))
    return got


def _column(rng, t, lens, null_rows, null_share=0.1, max_count=5):
    """Rows of the given lengths; rows flagged in null_rows hold only nulls, every other non-empty row at least one value."""
    lens = np.asarray(lens, np.int64)
    offsets = np.concatenate([[0], np.cumsum(lens)])
    n = int(offsets[-1])
    vals = _values(rng, t, n)
    valid = rng.random(n) >= null_share
    valid[np.repeat(null_rows, lens)] = False
    live = (lens > 0) & ~null_rows
    valid[offsets[:-1][live] + rng.integers(0, lens[live])] = True
    counts = rng.integers(0, max_count, n).astype(np.int64)
    return offsets, vals, valid, counts


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# The tiers' grids (launch_pct_fill in csrc/histogram.cu): pct_group_kernel<32> runs min(ceil(rows / kWarpRows),
# sm_count() * 8) CTAs of kWarpRows = 8 warps, a row per warp, so one sweep covers W = sms * 8 * 8 rows;
# pct_group_kernel<kCtaThreads> runs min(rows, sm_count()) CTAs, a row per CTA, so one sweep covers C = sms rows.  The
# counts are of rows in the tier's list (rows with a value); null and empty rows are added beside them.
CYCLES = [("warp", "w_minus_1", 1, -1, INT16), ("warp", "w", 1, 0, FLOAT32), ("warp", "w_plus_1", 1, 1, UINT64),
          ("warp", "3w_plus_5", 3, 5, FLOAT64), ("cta", "c", 1, 0, INT32), ("cta", "c_plus_1", 1, 1, INT8),
          ("cta", "2c_plus_3", 2, 3, FLOAT64)]


@pytest.mark.parametrize("case", CYCLES, ids=[f"{c[0]}-{c[1]}" for c in CYCLES])
def test_grid_cycles_past_its_first_sweep(case):
    S, Hs = _s()
    tier, _, a, b, t = case
    sweep = _sms() * 8 * 8 if tier == "warp" else _sms()
    lo, hi = (1, WARP_CAP) if tier == "warp" else (WARP_CAP + 1, K)
    n_valid = a * sweep + b
    rng = np.random.default_rng(CYCLES.index(case))
    n_null, n_empty = n_valid // 40 + 1, n_valid // 40 + 1
    kind = rng.permutation(np.repeat([0, 1, 2], [n_valid, n_null, n_empty]))      # 0 valid, 1 all-null, 2 empty
    lens = np.where(kind == 2, 0, rng.integers(lo, hi + 1, len(kind)))
    offsets, vals, valid, counts = _column(rng, t, lens, kind == 1)
    _check(S, Hs, t, offsets, vals, valid, counts, [0.0, 0.25, 0.5, 0.9, 1.0])


@pytest.mark.parametrize("t", [INT64, FLOAT64], ids=["int64", "float64"])
def test_a_million_short_histograms(t):
    """Spark's percentile after a group-by: many short rows.  P = 3, 5 and 7 do not divide 32, so the flat output's mask
    words span row boundaries."""
    S, Hs = _s()
    rng = np.random.default_rng(t)
    rows = 1_000_000
    lens = rng.integers(1, 17, rows)
    offsets, vals, valid, counts = _column(rng, t, lens, rng.random(rows) < 0.02, max_count=100)
    want, ok = M.percentile(offsets, vals, valid, counts, [i / 100 for i in range(101)])
    for hundredths in ([50], [10, 50, 90], [0, 25, 50, 75, 100], [5, 15, 30, 45, 60, 80, 95], range(101)):
        pct = [i / 100 for i in hundredths]
        _check(S, Hs, t, offsets, vals, valid, counts, pct, want=(np.ascontiguousarray(want[:, list(hundredths)]), ok))


PCT9 = [0.0, 0.1, 0.25, 1 / 3, 0.5, 0.75, 0.9, 0.999, 1.0]     # 18 select targets: two groups of kSelGroup = 16


@pytest.mark.parametrize("t", [INT8, INT64, UINT64, FLOAT32, FLOAT64], ids=lambda t: NAME[t])
def test_every_tier_in_one_call(t):
    """Each tier writes its rows' outputs at pos[row], and the select state starts afresh for each long row."""
    S, Hs = _s()
    rng = np.random.default_rng(100 + t)
    spec = [(rng.integers(1, WARP_CAP + 1, 3000), False), (rng.integers(WARP_CAP + 1, K + 1, 300), False),
            (np.array([K + 1, K + 2, 3 * K, 40_000, 150_000]), False),
            (rng.integers(1, WARP_CAP + 1, 40), True), (rng.integers(WARP_CAP + 1, K + 1, 10), True), (np.array([K + 1, 20_000]), True),
            (np.zeros(60, np.int64), False)]
    lens = np.concatenate([s[0] for s in spec])
    null_rows = np.concatenate([np.full(len(s[0]), s[1]) for s in spec])
    order = rng.permutation(len(lens))
    lens, null_rows = lens[order], null_rows[order]
    offsets, vals, valid, counts = _column(rng, t, lens, null_rows)
    _check(S, Hs, t, offsets, vals, valid, counts, PCT9)
    select = np.nonzero((lens > K) & ~null_rows)[0]
    start = max(int(select[len(select) // 2]) - 7, 1)           # offsets[0] > 0, and select-tier rows follow
    assert offsets[start] > 0 and (select >= start).any()
    _check(S, Hs, t, offsets, vals, valid, counts, PCT9, slice_from=start)


PAD = (200, 5000, 9000)                       # e - s, nulls included, picks the tier: warp (<= 256), CTA (<= K), select


def _on_every_tier(rng, t, histograms):
    """Each (values, counts) as three rows, padded with nulls to each PAD length at random positions.  The null
    elements carry large counts, so one that leaked into a sum would show."""
    lens, vals, valid, counts = [], [], [], []
    for v, c in histograms:
        for L in PAD:
            at = np.sort(rng.choice(L, len(v), replace=False))
            perm = rng.permutation(len(v))
            rv, rc = _values(rng, t, L), rng.integers(1, 2**40, L).astype(np.int64)
            rv[at], rc[at] = v[perm], c[perm]
            rvalid = np.zeros(L, bool)
            rvalid[at] = True
            lens.append(L), vals.append(rv), valid.append(rvalid), counts.append(rc)
    offsets = np.concatenate([[0], np.cumsum(lens)])
    return offsets, np.concatenate(vals), np.concatenate(valid), np.concatenate(counts)


def _alike_on_every_tier(got, n):
    bits = got.view(np.uint64).reshape(n, len(PAD), -1)
    for i in range(n):
        for j in range(1, len(PAD)):
            assert np.array_equal(bits[i, 0], bits[i, j]), (i, PAD[j], got.reshape(n, len(PAD), -1)[i])


def _equal_keys(t, n):
    """n values of one key: distinct NaN payloads for floats, distinct nonzero bytes for BOOL8, the maximum otherwise."""
    if t == FLOAT64:
        pool = np.array([0x7ff8000000000000, 0xfff8000000000001, 0x7ff0000000000123], np.uint64).view(np.float64)
    elif t == FLOAT32:
        pool = np.array([0x7fc00000, 0xffc00001, 0x7f800123], np.uint32).view(np.float32)
    elif t == BOOL8:
        pool = np.array([1, 2, 255], np.uint8)
    else:
        pool = np.array([np.iinfo(NP[t]).max], NP[t])
    return np.resize(pool, n)


@pytest.mark.parametrize("t", sorted(NAME), ids=lambda t: NAME[t])
def test_every_tier_gives_one_answer(t):
    S, Hs = _s()
    rng = np.random.default_rng(200 + t)
    v = _values(rng, t, 120)
    c = rng.integers(0, 4, 120).astype(np.int64)
    k = M.sort_keys(v, t == BOOL8)
    c[(k == k.min()) | (k == k.max())] = 0                     # zero counts at either end
    histograms = [(v, c),
                  (_values(rng, t, 60), np.zeros(60, np.int64)),                        # total count 0
                  (_values(rng, t, 1), np.array([7], np.int64)),                        # one valid element
                  (_equal_keys(t, 80), rng.integers(0, 4, 80).astype(np.int64)),        # every key equal
                  (_values(rng, t, 150), rng.integers(1, 1000, 150).astype(np.int64))]
    offsets, vals, valid, counts = _on_every_tier(rng, t, histograms)
    got = _check(S, Hs, t, offsets, vals, valid, counts, PCT9)
    _alike_on_every_tier(got, len(histograms))


def _int64_with_key(key):
    """The INT64 value whose key (the value with its sign bit flipped) is `key`."""
    return (np.array([key], np.uint64) ^ np.uint64(1 << 63)).view(np.int64)


def _floats(dt, xs, nan_bits):
    nans = np.array(nan_bits, np.uint64 if dt == np.float64 else np.uint32).view(dt)
    return [np.array([x], dt) for x in xs] + [nans]


F64_NAN = [0x7ff8000000000000, 0xfff8000000000001, 0x7ff0000000000001]
F32_NAN = [0x7fc00000, 0xffc00001, 0x7f800001]
# name -> (type, groups of values in ascending key order; the values of a group share one key)
EDGES = {
    # below 2^53, so values one apart stay apart as doubles
    "int64_lowest_byte": (INT64, [_int64_with_key(0x8012_3456_789a_bc00 | d) for d in (0x00, 0x01, 0x02, 0x7f, 0x80, 0xfe, 0xff)]),
    "int64_highest_byte": (INT64, [_int64_with_key((h << 56) | 0x00a5_5a00_ff00_01) for h in (0x00, 0x01, 0x7f, 0x80, 0xfe, 0xff)]),
    "int64_extremes": (INT64, [np.array([x], np.int64) for x in (-2**63, -2**63 + 1, -1, 0, 2**63 - 2, 2**63 - 1)]),
    "uint64_extremes": (UINT64, [np.array([x], np.uint64) for x in (0, 1, 0xff, 2**63, 2**64 - 0x100, 2**64 - 2, 2**64 - 1)]),
    "uint32_middle_bytes": (UINT32, [np.array([x], np.uint32) for x in (0x00000000, 0x0000ff00, 0x00ff0000, 0x00ffff00, 0xff000000, 0xffffffff)]),
    "float64_specials": (FLOAT64, _floats(np.float64, [-np.inf, -1.7976931348623157e308, -1.0, -5e-324, -0.0, 0.0, 5e-324, 1.0,
                                                       1.7976931348623157e308, np.inf], F64_NAN)),
    "float32_specials": (FLOAT32, _floats(np.float32, [-np.inf, -3.4028235e38, -1.0, -1e-45, -0.0, 0.0, 1e-45, 1.0, 3.4028235e38, np.inf],
                                          F32_NAN)),
    "int8": (INT8, [np.array([x], np.int8) for x in (-128, -127, -1, 0, 1, 126, 127)]),
    "uint8": (UINT8, [np.array([x], np.uint8) for x in (0, 1, 127, 128, 254, 255)]),
    "bool8": (BOOL8, [np.array([0], np.uint8), np.array([1, 2, 255], np.uint8)]),
}


def _edge_histogram(rng, groups, zero_ends):
    """Values and counts of the groups, whose total T is 2^k + 1, and percentages p = m / 2^k (position (T - 1) * p = m
    exactly) that put a rank on each cumulative-count boundary B between groups, at B - 1 and B + 1, halfway across it
    (ranks B and B + 1), and at p = 0 and p = 1.  zero_ends: the first and last groups (the first only, with two) count 0."""
    m = len(groups)
    c = rng.integers(1, 1000, m)
    if zero_ends:
        c[0] = 0
        c[-1] = 0 if m > 2 else c[-1]
    k = int(c.sum() - 1).bit_length()
    c[m // 2] += 2**k + 1 - c.sum()
    T = 2**k + 1
    vals, counts = [], []
    for g, total in zip(groups, c):                          # each group as several elements, some with count 0
        n = len(g) + int(rng.integers(0, 4))
        vals.append(np.resize(g, n))
        counts.append(rng.multinomial(total, np.full(n, 1 / n)))
    vals, counts = np.concatenate(vals), np.concatenate(counts).astype(np.int64)
    if (len(vals) & (len(vals) - 1)) == 0:                      # the sort pads the row to a power of two: keep padding
        vals, counts = np.append(vals, groups[m // 2][:1]), np.append(counts, 0)
    bounds = np.cumsum(c)[:-1]
    ranks = {1, T} | {int(b) + d for b in bounds for d in (-1, 0, 1) if 1 <= b + d <= T}
    pct = {(r - 1) / 2**k for r in ranks} | {(2 * int(b) - 1) / 2**(k + 1) for b in bounds if 1 <= b < T}
    return vals, counts, sorted(pct | {0.1, 0.25, 0.5, 0.75, 0.9, 1 / 3, 2 / 3, 0.999})


@pytest.mark.parametrize("zero_ends", [False, True], ids=["counted_ends", "zero_count_ends"])
@pytest.mark.parametrize("name", sorted(EDGES))
def test_ranks_on_count_boundaries(name, zero_ends):
    """The radix select's pick (the first bin whose running weight reaches the rank) and rank (lower + 1) at the exact
    boundary; the same rows on the warp and CTA tiers, whose sort pads with the key ~0 that INT64 and UINT64 maxima have."""
    S, Hs = _s()
    t, groups = EDGES[name]
    rng = np.random.default_rng(sorted(EDGES).index(name) * 2 + zero_ends)
    vals, counts, pct = _edge_histogram(rng, groups, zero_ends)
    assert 2 * len(pct) > 16                                    # several target groups
    offsets, v, valid, c = _on_every_tier(rng, t, [(vals, counts)])
    got = _check(S, Hs, t, offsets, v, valid, c, pct)
    _alike_on_every_tier(got, 1)
