"""Golden vector of the Unique aggregate, transcribed from the reference's end-to-end test.

Source: query/engine_test.go TestUniqueAggregation.  One record of two REQUIRED int64 columns, aggregated with
`Unique(example)` grouped by `timestamp`: group 1 holds two different values and is NULL, group 3 holds one.
"""

SCHEMA = [("example", "int64"), ("timestamp", "int64")]
ROWS = {"example": [1, 2, 3], "timestamp": [1, 1, 3]}
AGGREGATE = ("unique", "example")
GROUP_BY = ["timestamp"]
EXPECTED = {"timestamp": [1, 3], "unique(example)": [None, 3]}
