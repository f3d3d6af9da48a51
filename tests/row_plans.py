"""The planning rules of the row-conversion kernels, restated in Python so that tests can size their tables from them.

Each function below mirrors one host-side decision of csrc/ (file and function named in its docstring): which kernel a
schema and a row count take, the tile height, the ring depth, the super-tile.  The GPU tests derive the row counts at
which a persistent CTA wraps its ring or takes a second tile from these, with the SM count read from the device.  The
constants are checked against the sources by tests/test_jcudf_model.py, so a retuned planner fails there first instead
of silently moving the tests off the edges they were written for."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional, Sequence

import jcudf_model as M

SMEM_BUDGET = 232448          # dynamic shared memory a CTA may request on sm_90 (227 KB)

# csrc/from_rows.cu, capi.cu srj_plan_create
FR_NARROW_MAX = 128           # fixed_row_size <= this: three 64 KB stages; wider: two 100 KB stages
FR_NARROW_STAGE = 64 * 1024
FR_WIDE_STAGE = 100 * 1024
FR_MAX_TILE = 512
FR_MAX_STAGES = 4             # kMaxStages
FR_STAGE_SLACK = 32           # kStageSlack
FR_STAGE_HDR = 32             # sizeof(StageHdr)
FR_SUPER_FIXED = 2            # super-tile = 2 tiles (fixed stride) ...
FR_SUPER_VAR = 8              # ... or 8 tiles (variable width)

# csrc/from_rows_wide.cu
W_MAX_COLS = 448              # kWMaxCols
W_SLAB_CAP = 3200             # slab_cap
W_MAX_SLABS = 16
W_MAX_G = 4                   # kWMaxG: row groups of 32 per tile
W_MAX_STAGES = 4              # kWMaxStages
W_SLACK = 32                  # kWSlack
W_DESC, W_HDR, W_SLAB = 16, 32, 36   # sizeof(WDesc), sizeof(WHdr), sizeof(WideSlab)
W_TABLES_MAX = 64 * 1024
GS_THREADS, GS_PER = 256, 16  # wide_group_scan_kernel: kGsThreads x kGsPer groups per CTA
GS_CHUNK_GROUPS = GS_THREADS * GS_PER

# csrc/strings.cu
SW_NG = 3                     # kSwNG: 32-row tiles in flight per CTA; the ring has 2 * kSwNG stages
SW_STAGES = 2 * SW_NG
SW_MAX_WPT, SW_MAX_CPW = 8, 8  # warps per tile, STRING columns per warp
SW_MIN_STRINGS = 8

# csrc/to_rows.cu, to_rows_var.cu
T2_SUPER = 4                  # kT2Super: consecutive tiles a to_rows2 CTA takes before the round-robin moves on
T2_BUDGET = 225 * 1024
TW_WARPS = 24                 # kTwWarps: to_rows_w_kernel warps (one 32-row group each)
T3_MAX_BLOCKS = 48            # kT3MaxBlocks
T3_MAX_ITEMS = 1024           # kT3MaxItems
RS_CHUNK = 4096               # kRsChunk: rows per CTA of the row-size scan
STR_SCAN_CHUNK = 4 * 256 * 4  # strings.cu kScanChunk (kScanIter * 4): offsets per CTA of the from_rows string scan


def _class_of(sz: int) -> int:
    return {1: 0, 2: 1, 4: 2, 8: 3, 16: 4}[sz]


@dataclass
class FromRowsTiling:
    tile_rows: int
    rows_per_item: int
    stage_bytes: int
    num_stages: int


def _tile_rows(stage_bytes: int, S: int) -> int:
    fit = stage_bytes // S
    R = min(fit // 32 * 32, FR_MAX_TILE)
    if R >= 128:
        R = R // 128 * 128
    if R < 32:
        R = 16 if fit >= 16 else 8
    return R


def from_rows_entries(types: Sequence[int]) -> int:
    """Fields the whole-row from_rows kernel moves: one per fixed-width column, one (the length word) per STRING."""
    return len(types)


def from_rows_smem_bytes(tl: FromRowsTiling, nent: int, ncols: int, nstr: int) -> int:
    """from_rows.cu from_rows_smem_bytes."""
    b = tl.num_stages * (tl.stage_bytes + FR_STAGE_SLACK)
    b += tl.num_stages * ((tl.tile_rows + 4) & ~3) * 4
    b += tl.num_stages * FR_STAGE_HDR
    b += 2 * FR_MAX_STAGES * 8
    b += ((nent + 1) & ~1) * 4
    b += nent * 8 + ncols * 8 + ((ncols + 3) & ~3) * 4
    b += ((tl.tile_rows + 4) & ~3) * 4
    b += (nstr + 4) * 4
    return (b + 127) & ~127


def from_rows_tiling(types: Sequence[int]) -> FromRowsTiling:
    """capi.cu srj_plan_create: the tile of the whole-row from_rows kernel, stages shrunk by 3/4 while the kernel's
    shared-memory request (stages + per-schema tables) exceeds the budget."""
    lay = M.layout(types)
    S = lay.fixed_row_size
    nstr = sum(t == M.STRING for t in types)
    stage, ns = (FR_NARROW_STAGE, 3) if S <= FR_NARROW_MAX else (FR_WIDE_STAGE, 2)
    R = _tile_rows(stage, S)
    tl = FromRowsTiling(R, R if R < 32 else 32, stage, ns)
    nent = from_rows_entries(types)
    while from_rows_smem_bytes(tl, nent, len(types), nstr) > SMEM_BUDGET and tl.stage_bytes > 8 * 1024:
        tl.stage_bytes = (tl.stage_bytes * 3 // 4) & ~127
        tl.tile_rows = _tile_rows(tl.stage_bytes, S)
        tl.rows_per_item = tl.tile_rows if tl.tile_rows < 32 else 32
    if from_rows_smem_bytes(tl, nent, len(types), nstr) > SMEM_BUDGET:
        raise ValueError("schema too wide for the from_rows kernel")
    return tl


def from_rows_super_rows(types: Sequence[int]) -> int:
    """from_rows.cu launch_from_rows: rows of a super-tile, the unit dealt round-robin to the CTAs."""
    var = any(t == M.STRING for t in types)
    return from_rows_tiling(types).tile_rows * (FR_SUPER_VAR if var else FR_SUPER_FIXED)


def from_rows_kernel_name(types: Sequence[int]) -> str:
    """The from_rows_kernel<NCW, RPL, VAR, ONEG> instantiation launch_variant picks (11 consumer warps)."""
    tl = from_rows_tiling(types)
    var = any(t == M.STRING for t in types)
    oneg = var and _from_rows_gpu(types, tl) == 1
    b = lambda x: "true" if x else "false"   # noqa: E731
    return f"from_rows_kernel<11, {tl.rows_per_item}, {b(var)}, {b(oneg)}>"


def _from_rows_gpu(types, tl: FromRowsTiling) -> int:
    """Row groups per unit of the static schedule (launch_from_rows): ONEG = a variable-width tile of one group."""
    rpl = tl.rows_per_item
    cpi = 32 // rpl
    ngroups = (tl.tile_rows + rpl - 1) // rpl
    counts = [0] * 5
    for t in types:
        counts[2 if t == M.STRING else _class_of(M.SIZE[t])] += 1
    slots = sum((k + cpi - 1) // cpi for k in counts)
    cs = 0
    while (slots << cs) < 96 and ngroups % (8 << cs) == 0:
        cs += 1
    return (ngroups + (1 << cs) - 1) >> cs


# ---------------------------------------------------------------------------- wide from_rows (from_rows_wide.cu)
@dataclass
class WidePlan:
    R: int
    G: int
    pitch: int
    nstages: int
    nslabs: int
    slabs: list           # [(begin, end)]


def wide_refusal(types: Sequence[int]) -> Optional[str]:
    """Why plan_wide does not take a schema, or None when it does."""
    try:
        plan_wide(types)
        return None
    except _Refused as e:
        return str(e)


class _Refused(Exception):
    pass


def plan_wide(types: Sequence[int]) -> WidePlan:
    """from_rows_wide.cu plan_wide.  Raises _Refused (via wide_refusal) for the schemas the whole-row kernel serves."""
    lay = M.layout(types)
    nc = len(types)
    strs = [c for c, t in enumerate(types) if t == M.STRING]
    nstr, spr = len(strs), lay.size_per_row
    if nstr < 8:
        raise _Refused("fewer than 8 STRING columns")
    if spr < 512:
        raise _Refused("size_per_row below 512")
    if nc > W_MAX_COLS:
        raise _Refused("more than kWMaxCols columns")
    nslabs = max(1, min((spr + W_SLAB_CAP - 1) // W_SLAB_CAP, W_MAX_SLABS))
    first = [0] + [nc] * nslabs
    c = 0
    for i in range(1, nslabs):
        target = i * spr // nslabs
        while c < nc and lay.starts[c] < target:
            c += 1
        first[i] = c
    sidx = {col: s for s, col in enumerate(strs)}
    slabs, nent, maxlen = [], 0, 0
    for i in range(nslabs):
        c0, c1 = first[i], first[i + 1]
        begin = lay.starts[c0] if c0 < nc else lay.validity_offset
        end = begin
        for cc in range(c0, c1):
            end = max(end, lay.starts[cc] + lay.sizes[cc])
        for cc in range(c0, c1):
            if sidx.get(cc, 0) > 0:
                begin = min(begin, lay.starts[strs[sidx[cc] - 1]])
                break
        if i == nslabs - 1:
            end = spr
        nominal = lay.starts[c0] if c0 < nc else lay.validity_offset
        if nominal - begin > 128:
            raise _Refused("a slab's previous STRING pair lies more than 128 bytes back")
        b, e = begin & ~7, (end + 7) & ~7
        slabs.append((b, e))
        maxlen = max(maxlen, e - b)
        nent += c1 - c0
    pitch = (maxlen + 16 + 15) & ~15
    if ((pitch >> 4) & 1) == 0:
        pitch += 16
    tables = (nent * W_DESC + W_MAX_STAGES * W_HDR + 2 * W_MAX_STAGES * 8 + nc * 12 + nslabs * W_SLAB + nstr * 4
              + nslabs * 6 * 16 * 2 + 256)
    if tables > W_TABLES_MAX:
        raise _Refused("descriptor tables above 64 KB")
    ns = 3
    while True:
        R = ((SMEM_BUDGET - tables) // ns - W_SLACK) // (pitch + 4) // 32 * 32
        if R >= 64 or ns == 2:
            break
        ns -= 1
    R = min(R, 32 * W_MAX_G)
    if R < 32:
        raise _Refused("no 32-row tile fits")
    return WidePlan(R, R // 32, pitch, ns, nslabs, slabs)


def wide_kernel_name(types: Sequence[int]) -> str:
    return f"from_rows_wide_kernel<12, {plan_wide(types).G}>"


# ---------------------------------------------------------------------------- chars gather (strings.cu)
def strings_wide_eligible(types: Sequence[int]) -> bool:
    """strings_wide_eligible: the fast gather takes 8..64 STRING columns; others take strings_from_rows_kernel."""
    nstr = sum(t == M.STRING for t in types)
    return SW_MIN_STRINGS <= nstr <= SW_MAX_WPT * SW_MAX_CPW


def strings_wide_split(nstr: int) -> tuple:
    """(warps per tile, STRING columns per warp) of launch_strings_from_rows."""
    wpt = min(SW_MAX_WPT, (nstr + 3) // 4)
    return wpt, (nstr + wpt - 1) // wpt


# ---------------------------------------------------------------------------- to_rows (to_rows.cu, to_rows_var.cu)
def to_rows2_R(types: Sequence[int]) -> int:
    """to_rows.cu launch_to_rows: tile height of to_rows2_kernel (fixed-width tables); 0 = the generic kernel only.
    The kernel also wants >= R rows, 16-byte aligned columns and output, and a batch starting on a 32-row boundary."""
    if any(t == M.STRING for t in types):
        return 0
    lay = M.layout(types)
    S, D = lay.fixed_row_size, sum(lay.sizes)
    tables = len(types) * 28 + len(types) * 8 + 1024
    budget = T2_BUDGET - tables
    R = budget // (3 * D + 2 * S) // 128 * 128
    if R < 128:
        R = budget // (2 * D + 2 * S) // 32 * 32
    R = min(R, 512)
    if R >= 128:
        R = R // 128 * 128
    return R if R >= 128 else 0


def _to_rows3_stage(types: Sequence[int]) -> int:
    """Payload bytes of a to_rows3_kernel stage (what shared memory leaves after the tables and the chars slots), or 0
    when the schema has too many work items for the kernel."""
    lay = M.layout(types)
    nstr = sum(t == M.STRING for t in types)
    nc = len(types)
    nfixed = nc - nstr
    sb = max(4, (nstr + T3_MAX_BLOCKS - 1) // T3_MAX_BLOCKS)
    nblocks = (nstr + sb - 1) // sb
    counts = [0] * 5
    for t in types:
        if t != M.STRING:
            counts[_class_of(M.SIZE[t])] += 1
    nitems = nblocks + (nc + 31) // 32 + sum((k + 7) // 8 for k in counts)
    if nitems > T3_MAX_ITEMS:
        return 0
    tables = (8 * (nfixed + nc + 2 * nstr) + 4 * (nfixed + nstr + 32 * nblocks + nstr + 2 * nitems)
              + ((nitems + 15) & ~15) + 32 + 128)
    budget = SMEM_BUDGET - 1024 - 64
    slot = min((budget - tables) // 4, 1024 * nstr) // nstr // 16 * 16
    if slot < 128:
        slot = 0
    stage = (budget - tables - slot * nstr) // 16 * 16
    return 0 if stage < 32 * 1024 or stage < 8 * (lay.fixed_row_size + 64) else stage


def to_rows_var_kernel(types: Sequence[int], batch_bytes: int, nrows: int) -> Optional[str]:
    """to_rows_var.cu launch_to_rows_var: which kernel a batch with STRING columns (aligned buffers) takes before the
    generic kernel behind it: "to_rows_w_kernel", "to_rows3_kernel" or None (the generic kernel alone)."""
    lay = M.layout(types)
    nstr = sum(t == M.STRING for t in types)
    if nstr == 0 or nrows == 0:
        return None
    nc = len(types)
    avg = max(lay.fixed_row_size, batch_bytes // nrows)
    tables = 8 * (nc - nstr + nc + 2 * nstr) + 4 * (nc - nstr + nstr) + 128
    wbuf = ((SMEM_BUDGET - 1024 - 64 - tables) // TW_WARPS - 32) // 16 * 16
    if not (wbuf < 1024 or wbuf < lay.fixed_row_size + 64 or avg * 16 > wbuf):
        return "to_rows_w_kernel"
    stage = _to_rows3_stage(types)
    if not stage or min(32, stage // avg // 8 * 8) < 8 or stage // avg >= 64:
        return None
    return "to_rows3_kernel"


def to_rows3_super_rows(types: Sequence[int], batch_bytes: int, nrows: int) -> int:
    """Rows a to_rows3_kernel CTA takes at a time: two tiles of up to 32 rows, as many as a stage holds."""
    avg = max(M.layout(types).fixed_row_size, batch_bytes // nrows)
    return 2 * min(32, _to_rows3_stage(types) // avg // 8 * 8)
