"""strings_wide_kernel against the independent JCUDF model (tests/jcudf_model.py) at the cases its producer split
creates.

kSwProducers producer warps share the row copies of a 32-row tile: producer q issues the copies of the rows whose lane
index is congruent to q, and arrives on the stage's full barrier with the bytes of its own copies (without a byte
count when its rows carry none).  The producers load the row offsets one tile ahead, and each consumer warp loads its
columns' offsets entries one tile ahead.  The cases here are the ones random tables do not build on purpose: every
row of one producer with an empty variable section, a table with no chars at all, last tiles of 1, P - 1, P and P + 1
rows, and tables of more than 2 x kSwStages x SMs tiles, so that every CTA goes round its ring with prefetched offsets.
Each runs phase 1 and phase 2 through the C ABI, compares every output with the model, and checks through
torch.profiler that strings_wide_kernel ran."""
import os
import re

import numpy as np
import pytest

import row_plans as P
from oracle import oracle as O
from test_gpu_rows_scale import _from_rows_case, _sms
from util import random_table

pytestmark = pytest.mark.gpu

S_, I32, I64 = O.STRING, O.INT32, O.INT64


def _producers() -> int:
    src = os.path.join(os.path.dirname(__file__), "..", "spark-rapids-jni_b200", "csrc", "strings.cu")
    with open(src) as f:
        return int(re.search(r"constexpr int kSwProducers\s*=\s*(\d+);", f.read()).group(1))


PW = _producers()
# Only the gather is required in the profiler's records: after many multi-gigabyte profiled calls in one process,
# torch.profiler was seen to drop the phase-1 kernels' records while the outputs matched the model.
GATHER = ["strings_wide_kernel"]

# (STRING columns, phase-1 kernel in front of the gather): the wide plan leaves group-local offsets sums and
# per-group bases, the whole-row kernel finished offsets.  15 columns is nvbench_var's split (4 warps per tile).
SCHEMAS = {
    "8_wide": [S_] * 8 + [I64] * 60,
    "8_whole_row": [I32, I32] + [S_] * 8,
    "15_wide": [S_] * 15 + [I64] * 60,
    "15_whole_row": [I32, I32] + [S_] * 15,
    "64_wide": [S_] * 64,
}


def _schema(name):
    types = SCHEMAS[name]
    assert P.strings_wide_eligible(types)
    assert (P.wide_refusal(types) is None) == name.endswith("_wide")
    return types


def _tiles() -> int:
    """More than 2 x kSwStages x SMs tiles, and not a multiple of the grid: every CTA wraps its ring at least twice."""
    return 2 * P.SW_STAGES * _sms() + 3


def _set_lengths(col: O.HCol, keep: np.ndarray) -> O.HCol:
    """col with the strings of the rows where keep is False emptied (nulls stay null)."""
    lens = np.diff(col.offsets.astype(np.int64))
    new = np.zeros(len(lens) + 1, dtype=np.int32)
    np.cumsum(lens * keep, out=new[1:])
    chars = col.data[np.repeat(keep, lens)]
    return O.HCol(col.type_id, chars, col.mask, new, col.scale, col.size)


def _table(types, n, seed, keep=None):
    cols = random_table(types, n, seed=seed, max_str=24)
    if keep is not None:
        cols = [_set_lengths(c, keep) if c.type_id == S_ else c for c in cols]
    return cols


@pytest.mark.parametrize("schema", list(SCHEMAS))
@pytest.mark.parametrize("q", list(range(PW)))
def test_one_producer_without_bytes(schema, q):
    """Every row owned by producer q (lane index congruent to q) has an empty variable section -- null or empty
    strings -- in every tile, the short last tile included: q arrives without a byte count while the others stage."""
    types = _schema(schema)
    n = _tiles() * 32 + 17
    keep = (np.arange(n) % 32) % PW != q
    cols = _table(types, n, seed=100 + q, keep=keep)
    _from_rows_case(types, cols, GATHER)


@pytest.mark.parametrize("schema", list(SCHEMAS))
def test_no_chars_at_all(schema):
    """Every string of the table null or empty: no producer has bytes to copy, and no column any chars."""
    types = _schema(schema)
    n = _tiles() * 32 + PW + 1
    cols = _table(types, n, seed=7, keep=np.zeros(n, bool))
    assert all(c.offsets[-1] == 0 for c in cols if c.type_id == S_)
    _from_rows_case(types, cols, GATHER)


@pytest.mark.parametrize("schema", list(SCHEMAS))
@pytest.mark.parametrize("tail", ["1", "P-1", "P", "P+1"])
def test_short_last_tile(schema, tail):
    """A last tile of 1, P - 1, P or P + 1 rows (P = kSwProducers): some producers own none of its rows."""
    types = _schema(schema)
    extra = {"1": 1, "P-1": PW - 1, "P": PW, "P+1": PW + 1}[tail]
    n = _tiles() * 32 + extra
    _from_rows_case(types, _table(types, n, seed=200 + extra), GATHER)
