"""Inputs where Arithmetic.round goes wrong first, and a float32 reference of the round recipe that runs on the device.

FLOAT32: round_float32 restates oracle/arithmetic.py's round_float (the reference's round_float.cu:54-97) in torch, every
float32 operation computed in float64 and rounded to float32.  That is exact for + - * /: float64 carries 53 >= 2 * 24 + 2
bits, so rounding its correctly rounded result to float32 gives the correctly rounded float32 result.  trunc, round and
rint are exact in either type.  The divisor n is a device tensor: PyTorch's CUDA division by a CPU scalar multiplies by
the reciprocal, which is not correctly rounded.

FLOAT64: a division e / n by n = pow(10, k) is hardest to round right where the exact quotient lies close to a midpoint
between two adjacent doubles.  near_midpoints finds numerators m whose m / D sits at the smallest distance from such a
midpoint that integers of that range can reach.  f64_positive_dp and f64_negative_dp build inputs from them for the two
branches of the recipe.

Integers and decimals: rounding by 10^k turns on the remainder's comparison with h = 10^k / 2, so int_ties gives
q * 10^k + {h - 1, h, h + 1} for even and odd q, both signs, up to the largest q of the storage range.
"""
from __future__ import annotations

import math
from fractions import Fraction

import numpy as np

from oracle import arithmetic as A

HALF_UP, HALF_EVEN = 0, 1

F32_DPS = list(range(-39, 40)) + [40, -40, 45, -45, 300, -300]
F64_DPS = [s * d for d in list(range(1, 24)) + [100] + list(range(300, 310)) + [323] for s in (1, -1)]


# ---- FLOAT32 ------------------------------------------------------------------------------------------------------------
def f32_pow10(dp: int) -> float:
    """n of the recipe: float32(pow(10, |dp|)), inf from |dp| = 39."""
    with np.errstate(over="ignore"):
        return float(np.float32(A.pow10(abs(int(dp)))))


def _half_up(t):
    """C's round(): halves away from zero (t - trunc(t) is exact)."""
    import torch
    tr = torch.trunc(t)
    return torch.where((t - tr).abs() >= 0.5, tr + torch.sign(t), tr)


def round_float32(x, dp: int) -> dict:
    """{HALF_UP: round(x, dp), HALF_EVEN: bround(x, dp)} for a float32 tensor x, on x's device."""
    import torch
    rnd = {HALF_UP: _half_up, HALF_EVEN: torch.round}
    if dp == 0:
        return {m: f(x) for m, f in rnd.items()}
    n = torch.tensor(f32_pow10(dp), dtype=torch.float64, device=x.device)
    xd = x.double()
    if dp > 0:
        ip = torch.trunc(xd)
        # modf: the fraction carries x's sign (so -0.0 and -2.0 give -0.0), and +-inf give +-0
        frac = torch.copysign(torch.nan_to_num(xd - ip, nan=0.0), xd)
        p = (frac * n).float()
        return {m: (ip + (f(p).double() / n).float().double()).float() for m, f in rnd.items()}
    q = (xd / n).float()
    return {m: (f(q).double() * n).float() for m, f in rnd.items()}


# ---- FLOAT64 ------------------------------------------------------------------------------------------------------------
def f64_pow10(dp: int) -> float:
    """n of the recipe in float64: pow(10, |dp|), inf from |dp| = 309."""
    return A.pow10(abs(int(dp)))


def ulp_exp(E: int) -> int:
    """log2 of the spacing of doubles in [2^E, 2^(E+1)), subnormals included."""
    return max(E, -1022) - 52


def midpoint_distance(q: Fraction) -> Fraction:
    """Distance of q > 0 from the nearest midpoint between adjacent doubles, in units of q's ulp (0 .. 1/2)."""
    E = q.numerator.bit_length() - q.denominator.bit_length()
    if Fraction(2) ** E > q:
        E -= 1
    t = q / Fraction(2) ** ulp_exp(E)
    f = t - math.floor(t)
    return abs(f - Fraction(1, 2))


def near_midpoints(D: Fraction, lo: int, hi: int, E: int, count: int, tries: int = 20000) -> list:
    """Up to `count` integers m in [lo, hi), with m / D in [2^E, 2^(E+1)), closest to a midpoint between doubles.

    m / D in ulps is m * a / P with a / P = 1 / (D * ulp) reduced, so its distance from a midpoint is |c - P / 2| / P
    for c = m * a mod P.  Walking c outward from P / 2 and solving m = c * a^-1 mod P gives the nearest reachable ones."""
    F = 1 / (D * Fraction(2) ** ulp_exp(E))
    a, P = F.numerator, F.denominator
    if P < 3:
        return []
    inv = pow(a, -1, P)
    out = []
    c0 = P // 2
    for j in range(tries):
        c = c0 + (j + 1) // 2 * (1 if j % 2 else -1)
        r = c * inv % P
        m = lo + (r - lo) % P
        while m < hi and len(out) < count:
            out.append(m)
            m += P
            if m - lo > 4 * P:                      # a few per residue class are enough
                break
        if len(out) >= count:
            break
    return out


def _binades(lo_q: Fraction, hi_q: Fraction, keep: int):
    """Exponents E with [2^E, 2^(E+1)) meeting [lo_q, hi_q): the top and bottom `keep` ones and a few between."""
    Elo = lo_q.numerator.bit_length() - lo_q.denominator.bit_length() - 1
    Ehi = hi_q.numerator.bit_length() - hi_q.denominator.bit_length() + 1
    Es = [E for E in range(Elo, Ehi + 1) if Fraction(2) ** (E + 1) > lo_q and Fraction(2) ** E < hi_q]
    if len(Es) <= 3 * keep:
        return Es
    mid = Es[keep:-keep]
    return Es[:keep] + mid[:: max(1, len(mid) // keep)] + Es[-keep:]


def f64_positive_dp(k: int) -> dict:
    """dp = k > 0 on FLOAT64.  -> {"mid": e = +-m / 10^k with m / n near a midpoint and round(e * n) == m (the recipe's
    quotient is m / n), "small": every m < min(10^k, 10^6), "sub": m / n subnormal, each as float64 arrays}."""
    n = f64_pow10(k)
    if math.isinf(n):
        return {"mid": np.zeros(0), "small": np.zeros(0), "sub": np.zeros(0)}
    D = Fraction(n)
    mmax = min(int(D), 2 ** 53)                     # m < n (a fraction) and exactly representable
    ms = []
    for E in _binades(1 / D, Fraction(mmax) / D, 4):
        lo = max(1, math.ceil(Fraction(2) ** E * D))
        hi = min(mmax, math.ceil(Fraction(2) ** (E + 1) * D))
        ms += near_midpoints(D, lo, hi, E, 48)
    ms = np.array(sorted(set(ms)), np.float64)
    e = ms / np.float64(10.0 ** k) if k <= 22 else np.array([float(Fraction(int(m), 10 ** k)) for m in ms])
    with np.errstate(all="ignore"):
        keep = np.round(e * n) == ms                 # the kernel's round(frac * n) reproduces m
    e = e[keep]
    small = np.arange(1, min(10 ** k, 10 ** 6), dtype=np.float64) / np.float64(10.0 ** k) if k <= 22 else \
        np.array([float(Fraction(m, 10 ** k)) for m in range(1, 4096)])
    sub = np.array([float(Fraction(m, 10 ** k)) for m in range(1, 64)]) if k >= 300 else np.zeros(0)
    return {"mid": np.concatenate([e, -e]), "small": np.concatenate([small, -small]), "sub": np.concatenate([sub, -sub])}


def f64_negative_dp(k: int) -> dict:
    """dp = -k < 0 on FLOAT64.  -> {"half": e within a few ulps of (h + 0.5) * n, "mid": e / n near a midpoint between
    doubles, each as float64 arrays with both signs}."""
    n = f64_pow10(k)
    if math.isinf(n):
        return {"half": np.zeros(0), "mid": np.zeros(0)}
    D = Fraction(n)
    hmax = min(Fraction(np.finfo(np.float64).max) / D - 1, Fraction(2 ** 52))
    hs = sorted({h for h in list(range(0, 16)) + [2 ** j + d for j in range(4, 53) for d in (-1, 0, 1)] if h <= hmax})
    half = []
    for h in hs:
        e0 = float(Fraction(2 * h + 1, 2) * D)
        if math.isinf(e0):
            continue
        lo, hi = e0, e0
        half.append(e0)
        for _ in range(3):
            lo, hi = np.nextafter(lo, -np.inf), np.nextafter(hi, np.inf)
            half += [float(lo), float(hi)]
    half = np.array([v for v in half if np.isfinite(v)], np.float64)
    mids = []
    # e = M * 2^f with M in [2^52, 2^53): f puts e / n near 2^qexp, and E picks the binade of the quotient
    for qexp in (0, 3, 10, 20):
        f = qexp + int(math.floor(math.log2(n))) - 52
        if f + 53 > 1024:
            continue
        Dm = D / Fraction(2) ** f
        for E in (qexp - 1, qexp):
            lo = max(2 ** 52, math.ceil(Fraction(2) ** E * Dm))
            hi = min(2 ** 53, math.ceil(Fraction(2) ** (E + 1) * Dm))
            if lo < hi:
                mids += [float(Fraction(M) * Fraction(2) ** f) for M in near_midpoints(Dm, lo, hi, E, 32)]
    mids = np.array([v for v in mids if np.isfinite(v)], np.float64)
    return {"half": np.concatenate([half, -half]), "mid": np.concatenate([mids, -mids])}


F64_SPECIALS = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 5e-324, -5e-324, 1.5e-323, 2.2250738585072014e-308,
                         np.finfo(np.float64).max, -np.finfo(np.float64).max, 0.5, -0.5, 1.5, -1.5, 2.5, -2.5, 1.25, 0.125,
                         12345.675, -12345.675, 1.234, 25.66, 154.9, 2346.0, 1e308, -1e308, 1e-308, 0.1, 2.0 ** 52 + 0.5,
                         2.0 ** 53, 4503599627370497.0], np.float64)


# ---- integers and decimals ----------------------------------------------------------------------------------------------
def int_ties(k: int, lo: int, hi: int, seed: int = 0) -> list:
    """Python ints in [lo, hi]: q * 10^k + {h - 1, h, h + 1} (h = 10^k / 2) for q even and odd, small, random and up to
    the largest that fits, both signs; and the range's ends."""
    d = 10 ** k
    h = d // 2
    rng = np.random.default_rng(seed * 1000 + k)
    qmax = max(0, (hi - h - 1) // d)
    qs = {0, 1, 2, 3, 4, 5}
    qs |= {max(0, qmax - i) for i in range(6)}
    qs |= {int(x) for x in rng.integers(0, qmax + 1, 24, dtype=np.uint64)} if qmax < 2 ** 64 else \
        {int(x) * int(y) % (qmax + 1) for x, y in zip(rng.integers(0, 2 ** 62, 24), rng.integers(0, 2 ** 62, 24))}
    out = set()
    for q in qs:
        for r in (h - 1, h, h + 1):
            v = q * d + r
            for s in (v, -v):
                if lo <= s <= hi:
                    out.add(s)
    ends = {lo, lo + 1, lo + 2, hi, hi - 1, hi - 2, 0, 1, -1}
    return sorted(out | {v for v in ends if lo <= v <= hi})
