"""The string GROUP BY reference (agg_string_reference.py) pinned to the reference's own collator key table
(TestUTF8CollatorKey, pkg/util/collate/collate_test.go:86: its binary, utf8mb4_bin and utf8mb4_0900_bin columns) and to
hand-worked cases of firstRow4String's earliest-row rule."""
import numpy as np
import pytest

import agg_string_reference as S
from tidb_b200 import abi
from tidb_b200.chunk import Chunk, Column
from tidb_b200.plan import AggFunc, AggPlan, FieldType

# value -> (binary, utf8mb4_bin, utf8mb4_0900_bin) keys, from TestUTF8CollatorKey
KEYS = [
    ("a", b"\x61", b"\x61", b"\x61"),
    ("A", b"\x41", b"\x41", b"\x41"),
    ("Foo © bar 𝌆 baz ☃ qux", "Foo © bar 𝌆 baz ☃ qux".encode(), "Foo © bar 𝌆 baz ☃ qux".encode(), "Foo © bar 𝌆 baz ☃ qux".encode()),
    ("a ", b"\x61\x20", b"\x61", b"\x61\x20"),
    ("ﷻ", b"\xef\xb7\xbb", b"\xef\xb7\xbb", b"\xef\xb7\xbb"),
    ("中文", b"\xe4\xb8\xad\xe6\x96\x87", b"\xe4\xb8\xad\xe6\x96\x87", b"\xe4\xb8\xad\xe6\x96\x87"),
    ("갟감1", b"\xea\xb0\x9f\xea\xb0\x90\x31", b"\xea\xb0\x9f\xea\xb0\x90\x31", b"\xea\xb0\x9f\xea\xb0\x90\x31"),
]


@pytest.mark.parametrize("value,binary,mb4_bin,mb4_0900_bin", KEYS)
def test_collator_keys(value, binary, mb4_bin, mb4_0900_bin):
    b = value.encode()
    assert S.collation_key(b, 63) == binary
    assert S.collation_key(b, 46) == mb4_bin
    assert S.collation_key(b, 309) == mb4_0900_bin
    for pad in (83, 65, 47):   # the other binPaddingCollator ids
        assert S.collation_key(b, pad) == mb4_bin


def test_pad_rules():
    assert S.collation_key(b"a  ", 46) == b"a" and S.collation_key(b"a\t", 46) == b"a\t"
    assert S.collation_key(b"", 46) == b"" == S.collation_key(b" ", 46)
    assert S.collation_key(b" ", 63) == b" " and S.collation_key(None, 46) is None
    with pytest.raises(ValueError):
        S.collation_key(b"a", 45)   # utf8mb4_general_ci is not offloaded


def _plan(coll, extra=()):
    t = FieldType(abi.TYPE_VARCHAR, 0, collation=coll)
    return AggPlan([t, FieldType(abi.TYPE_LONGLONG, 0)], [0], [AggFunc(abi.AGG_FIRSTROW, 0), AggFunc(abi.AGG_COUNT, -1), *extra])


def test_firstrow_earliest_in_sel_order():
    # physical order puts "a  " last, but sel visits it first: it is the earliest row of the group
    col = Column.strings([b"a", b"a ", b"a  "])
    ch = Chunk([col, Column(np.arange(3, dtype=np.int64))], sel=np.array([2, 0, 1]))
    exp = S.expected(_plan(46), [ch])
    assert list(exp) == [(b"a",)] and exp[(b"a",)][0].value == b"a  " and exp[(b"a",)][1].value == 3
    # under binary the three are three groups, each its own FIRSTROW
    exp = S.expected(_plan(63), [ch])
    assert {k: e[0].value for k, e in exp.items()} == {(b"a",): b"a", (b"a ",): b"a ", (b"a  ",): b"a  "}


def test_firstrow_earliest_push_wins():
    first = Chunk([Column.strings([b"x ", None]), Column(np.zeros(2, dtype=np.int64))])
    second = Chunk([Column.strings([b"x", b"", b" "]), Column(np.zeros(3, dtype=np.int64))])
    exp = S.expected(_plan(46), [first, second])
    assert exp[(b"x",)][0].value == b"x " and exp[(b"x",)][1].value == 2
    assert exp[(None,)][0].value is None and exp[(None,)][1].value == 1     # NULL is its own group, apart from ''
    assert exp[(b"",)][0].value == b"" and exp[(b"",)][1].value == 2        # '' and ' ' are one group under PAD
    exp = S.expected(_plan(309), [first, second])
    assert exp[(b"",)][1].value == 1 and exp[(b" ",)][1].value == 1


def test_numeric_aggregates_reuse_agg_reference():
    vals = [b"k", b"k ", None, b"m", b"k"]
    x = np.array([1.0, 2.0, 4.0, 8.0, 16.0])
    ch = Chunk([Column.strings(vals), Column(x), Column(np.arange(5, dtype=np.int64))])
    t = FieldType(abi.TYPE_VARCHAR, 0, collation=46)
    plan = AggPlan([t, FieldType(abi.TYPE_DOUBLE, 0), FieldType(abi.TYPE_LONGLONG, 0)], [0],
                   [AggFunc(abi.AGG_FIRSTROW, 0), AggFunc(abi.AGG_SUM, 1, abi.TYPE_DOUBLE), AggFunc(abi.AGG_COUNT, 0)])
    exp = S.expected(plan, [ch])
    assert exp[(b"k",)][1].value == 19.0 and exp[(b"k",)][2].value == 3
    assert exp[(None,)][2].value == 0 and exp[(b"m",)][1].value == 8.0
    # and the checker accepts exactly these rows
    rows = [(b"k", 19.0, 3), (None, 4.0, 0), (b"m", 8.0, 1)]
    assert S.check(plan, [ch], rows) == 3
    with pytest.raises(AssertionError):
        S.check(plan, [ch], [(b"k ", 19.0, 3), (None, 4.0, 0), (b"m", 8.0, 1)])   # not the earliest row's bytes
