"""Row-by-row restatement, in Python integers, of the radix casts (srj_b200.radix / cast, csrc/radix.cu):

  conv(inputs, from_bases, to_bases)  NumberConverter.convert: reference number_converter.cu:148-243 (Spark 3.5's
                                      NumberConverter), one row at a time at the widths of its C++ types
  conv_overflow(...)                  NumberConverter.isConvertOverflow: the same parse under its ANSI rule
  long_to_binary(values, valid)       CastStrings.fromLongToBinary (cast_long_to_binary_string.cu)
  integers_to_string(values, valid, bits, signed, base)   CastStrings.fromIntegersWithBase (cudf from_integers /
                                      integers_to_hex, then CastStringJni.cpp's extract ^0?([0-9a-fA-F]+)$)
  bytes_to_hex(data, offsets)         CastStrings.bytesToHex (hex.cu)

Rows are bytes (None: null); bases are ints or per-row lists with None for a null base.  Each function returns the
rows as bytes / None; to_column() turns them into the (offsets, chars, valid) of a STRING column.
"""
M64 = (1 << 64) - 1


def _trim(s: bytes):
    """number_converter.cu:65-76: (first, last) after skipping ASCII 32 at both ends"""
    first, last = 0, len(s) - 1
    while first < len(s) and s[first] == 0x20:
        first += 1
    while last > first and s[last] == 0x20:
        last -= 1
    return first, last


def _char_to_byte(c: int, base: int) -> int:
    """number_converter.cu:117-128 over a signed char: bytes >= 0x80 match no range"""
    if 0x30 <= c <= 0x39 and c - 0x30 < base:
        return c - 0x30
    if 0x41 <= c <= 0x5A and c - 0x41 + 10 < base:
        return c - 0x41 + 10
    if 0x61 <= c <= 0x7A and c - 0x61 + 10 < base:
        return c - 0x61 + 10
    return -1


def _s64(u: int) -> int:
    u &= M64
    return u - (1 << 64) if u >> 63 else u


def _digits(u: int, base: int) -> bytes:
    out = []
    while True:
        out.append(b"0123456789ABCDEFGHIJKLMNOPQRSTUVWXYZ"[u % base])
        u //= base
        if u == 0:
            return bytes(reversed(out))


SUCCESS, OVERFLOW, NULL_VALUE = 0, 1, 2


def convert_row(s: bytes, from_base: int, to_base: int, ansi: bool):
    """number_converter.cu:148-243: (result_type, bytes or None)"""
    first, last = _trim(s)
    if last - first < 0:
        return NULL_VALUE, None
    negative = False
    if s[first] == 0x2D:
        negative = True
        first += 1
    v = 0                                                   # int64_t
    bound = ((-1 - from_base) & M64) // from_base           # static_cast<unsigned long>(-1L - from_base) / from_base
    for i in range(first, last + 1):
        b = _char_to_byte(s[i], from_base)
        if b < 0:
            break
        if v < 0:
            if ansi:
                return OVERFLOW, None
            v = -1
            break
        if (v & M64) >= bound:                              # int64 against unsigned long: v read as unsigned
            if ((-1 - b) & M64) // from_base < (v & M64):
                if ansi:
                    return OVERFLOW, None
                v = -1
                break
        v = _s64(v * from_base + b)
    if negative and to_base > 0:
        v = -1 if v < 0 else _s64(-v)
    if to_base < 0 and v < 0:
        v = _s64(-v)
        negative = True
    out = _digits(v & M64, abs(to_base))
    if negative and to_base < 0:
        out = b"-" + out
    return SUCCESS, out


def _valid_bases(f, t) -> bool:
    return 2 <= f <= 36 and 2 <= abs(t) <= 36


def _rows(inputs, from_bases, to_bases):
    """the row count and a per-row view of each argument (a scalar repeats)"""
    n = next(len(a) for a in (inputs, from_bases, to_bases) if isinstance(a, list))
    rep = lambda a: a if isinstance(a, list) else [a] * n
    return n, rep(inputs), rep(from_bases), rep(to_bases)


def conv(inputs, from_bases, to_bases):
    """NumberConverter.convert: inputs a list of bytes / None or one bytes scalar; bases lists (None: null) or ints"""
    n, ins, fbs, tbs = _rows(inputs, from_bases, to_bases)
    if not isinstance(from_bases, list) and not isinstance(to_bases, list) and not _valid_bases(from_bases, to_bases):
        return [None] * n
    out = []
    for s, f, t in zip(ins, fbs, tbs):
        if s is None or f is None or t is None or not _valid_bases(f, t):
            out.append(None)
        else:
            out.append(convert_row(s, f, t, False)[1])
    return out


def conv_overflow(inputs, from_bases, to_bases) -> bool:
    """NumberConverter.isConvertOverflow (number_converter.cu:419-474)"""
    n, ins, fbs, tbs = _rows(inputs, from_bases, to_bases)
    if not isinstance(from_bases, list) and not isinstance(to_bases, list) and not _valid_bases(from_bases, to_bases):
        return False
    return any(s is not None and f is not None and t is not None and _valid_bases(f, t) and convert_row(s, f, t, True)[0] == OVERFLOW
               for s, f, t in zip(ins, fbs, tbs))


def long_to_binary(values, valid=None):
    """cast_long_to_binary_string.cu:41-76: max(1, 64 - clz(v)) bits of the two's complement"""
    out = []
    for i, v in enumerate(values):
        if valid is not None and not valid[i]:
            out.append(None)
            continue
        u = int(v) & M64
        out.append(bytes(b"01"[(u >> k) & 1] for k in range(max(1, u.bit_length()) - 1, -1, -1)))
    return out


def integers_to_string(values, valid, bits: int, signed: bool, base: int):
    """base 10: cudf's from_integers (digits, '-' for negative); base 16: integers_to_hex's fewest bytes of the value's
    width (at least one), two upper-case digits each, most significant first, then one leading '0' dropped"""
    out = []
    for i, v in enumerate(values):
        if valid is not None and not valid[i]:
            out.append(None)
            continue
        v = int(v)
        if base == 10:
            out.append((b"-" if v < 0 else b"") + _digits(abs(v), 10))
            continue
        u = v & ((1 << bits) - 1)
        nbytes = bits // 8
        while nbytes > 1 and (u >> (8 * (nbytes - 1))) & 0xFF == 0:
            nbytes -= 1
        hexs = b"".join(b"%02X" % ((u >> (8 * k)) & 0xFF) for k in range(nbytes - 1, -1, -1))
        out.append(hexs[1:] if hexs[:1] == b"0" else hexs)
    return out


def bytes_to_hex(data: bytes, offsets):
    """hex.cu: (output offsets, output chars): each byte of the chars span [offsets[0], offsets[n]) as two upper-case
    digits, the offsets twice the input's rebased to 0"""
    base = int(offsets[0])
    offs = [2 * (int(o) - base) for o in offsets]
    return offs, bytes(data[base:int(offsets[-1])]).hex().upper().encode()


def to_column(rows):
    """(offsets list, chars bytes, valid list) of a STRING column holding `rows` (None: null, length 0)"""
    offs, acc = [0], 0
    for r in rows:
        acc += 0 if r is None else len(r)
        offs.append(acc)
    return offs, b"".join(r for r in rows if r is not None), [r is not None for r in rows]
