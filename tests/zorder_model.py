"""An independent per-row model of ZOrder.interleaveBits and ZOrder.hilbertIndex in Python integers.

It shares no code with oracle/zorder.py or the package.  interleave: each value becomes an 8W-character string of '0' /
'1' (MSB first) and the row's stream reads those strings column-wise, one character from each column per step.
hilbert: Skilling's AxesToTranspose on a list of Python ints, then the same column-wise read of num_bits-character
strings, taken as a binary number.
"""
from __future__ import annotations

from typing import List, Optional, Sequence


def value_bits(v: Optional[int], nbits: int) -> str:
    """v (any Python int, possibly negative) as its low nbits two's-complement bits, MSB first; None counts as 0."""
    return format((v or 0) & ((1 << nbits) - 1), f"0{nbits}b")


def interleave_row(values: Sequence[Optional[int]], width: int) -> bytes:
    """One row of interleaveBits: values are the row's N raw values (ints of 8W bits, or None for a null)."""
    strs = [value_bits(v, 8 * width) for v in values]
    stream = "".join(s[j] for j in range(8 * width) for s in strs)
    return bytes(int(stream[i:i + 8], 2) for i in range(0, len(stream), 8))


def hilbert_row(values: Sequence[Optional[int]], num_bits: int) -> int:
    """One row of hilbertIndex (the unsigned index; the column stores it as int64 bits)."""
    n = len(values)
    x: List[int] = [(v or 0) & ((1 << num_bits) - 1) for v in values]
    m = 1 << (num_bits - 1)
    q = m
    while q > 1:                                  # inverse undo
        p = q - 1
        for i in range(n):
            if x[i] & q:
                x[0] ^= p
            else:
                t = (x[0] ^ x[i]) & p
                x[0] ^= t
                x[i] ^= t
        q >>= 1
    for i in range(1, n):                         # Gray encode
        x[i] ^= x[i - 1]
    t = 0
    q = m
    while q > 1:
        if x[n - 1] & q:
            t ^= q - 1
        q >>= 1
    x = [xi ^ t for xi in x]
    strs = [value_bits(xi, num_bits) for xi in x]
    return int("".join(s[j] for j in range(num_bits) for s in strs), 2)


def to_int64(u: int) -> int:
    return u - (1 << 64) if u >= 1 << 63 else u
