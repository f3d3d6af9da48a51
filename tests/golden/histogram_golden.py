"""Histogram test data (data only): the two cases of the reference's HistogramTest.java, and answers derived by hand
from Spark's Percentile.

ROUND_TRIPS: (name, values (None = null), frequencies, percentages, expected percentile per row (None = null)).  The
values go through createHistogramIfValid(values, frequencies, outputAsLists=True), then percentileFromHistogram(...,
outputAsLists=False); the values are INT32.
PERCENTILES: (name, one histogram as (value, count) pairs with INT32 values, percentages, expected results).
  - p = 0.3 over {0, 10}: position 0.3, 0.7 * 0 + 0.3 * 10 = 3.0
  - {0.25, 0.75} over {0, 10}: 2.5 and 7.5; the median of {0, 10} is 5.0
  - weighted {1 x 3, 2 x 1, 10 x 4}: acc 3, 4, 8, max position 7.  p = 0.5: position 3.5, ranks 4 and 5 read 2 and 10,
    0.5 * 2 + 0.5 * 10 = 6.0; p = 0.25: position 1.75, ranks 2 and 3 both read 1, so 1.0; p = 1: rank 8 reads 10.
"""

ROUND_TRIPS = [
    ("testZeroFrequency", [5, 10, 30], [1, 0, 1], [1.0], [5.0, None, 30.0]),
    ("testAllNulls", [None, None, None], [1, 2, 3], [0.5], [None, None, None]),
]

PERCENTILES = [
    ("p30_of_0_10", [(0, 1), (10, 1)], [0.3], [3.0]),
    ("quartiles_of_0_10", [(0, 1), (10, 1)], [0.25, 0.75], [2.5, 7.5]),
    ("median_of_0_10", [(10, 1), (0, 1)], [0.5], [5.0]),
    ("weighted", [(10, 4), (1, 3), (2, 1)], [0.5, 0.25, 1.0, 0.0], [6.0, 1.0, 10.0, 1.0]),
]
