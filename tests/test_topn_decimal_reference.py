"""The DECIMAL order of tests/topn_decimal.py (cmpMyDecimal -> MyDecimal.Compare) on known answers and hand cases, the agreement of
its comparator and numpy forms, and the argument checks tg_topn makes for DECIMAL columns before it looks for a device."""
import ctypes as C
import struct

import numpy as np
import pytest

import mydecimal_args as A
import topn_decimal as TD
from tidb_b200 import abi
from tidb_b200.chunk import DECIMAL_DTYPE, Chunk, Column, MutChunk


def dec(text: str, digits_int=None, frac=None, result_frac=0, neg_zero=False, tail=()) -> bytes:
    """a stored cell of the literal: digitsInt defaults to the integer digits written, digitsFrac to the fraction digits
    written (frac > that pads trailing zeros); `tail` fills the words after the used ones (never looked at)"""
    neg = text.startswith("-")
    ip, _, fp = text.lstrip("-").partition(".")
    s = len(fp) if frac is None else frac
    fp = fp.ljust(s, "0")
    scaled = int((ip or "0") + fp)
    di = len(ip.lstrip("0")) if digits_int is None else digits_int
    c = bytearray(A.cell(-scaled if neg else scaled, max(di + s, 1), s, di, result_frac, neg_zero=neg_zero and scaled == 0))
    used = (di + 8) // 9 + (s + 8) // 9
    for j, w in enumerate(tail):
        struct.pack_into("<i", c, 4 + 4 * (used + j), w)
    return bytes(c)


def raw(di, df, neg, words, rf=0) -> bytes:
    words = list(words) + [0] * (9 - len(words))
    return struct.pack("<bbbB9i", di, df, rf, neg, *words)


# TestCompareMyDecimal (pkg/types/mydecimal_test.go:520), copied as data
COMPARE_KAT = [("12", "13", -1), ("13", "12", 1), ("-10", "10", -1), ("10", "-10", 1), ("-12", "-13", 1), ("0", "12", -1),
               ("-10", "0", -1), ("4", "4", 0), ("-1.1", "-1.2", 1), ("1.2", "1.1", 1), ("1.1", "1.2", -1)]


@pytest.mark.parametrize("a,b,want", COMPARE_KAT)
def test_compare_known_answers(a, b, want):
    assert TD.cmp_decimal(dec(a), dec(b)) == want
    # the same values in other stored forms: FromBin-style leading zero words, padded fraction digits, any resultFrac
    assert TD.cmp_decimal(dec(a, digits_int=20, frac=4, result_frac=7), dec(b, digits_int=30, frac=11)) == want


# value classes in ascending order; every cell of a class equals every other cell of it
ORDERED_CLASSES = [
    [dec("-" + "9" * 81), raw(81, 0, 1, [10 ** 9 - 1] * 9)],
    [dec("-1.5"), dec("-1.50"), dec("-0000000001.5", digits_int=10)],
    [dec("-1.000000000000000000000000000002")],
    [dec("-1.000000000000000000000000000001")],                 # differ only in the 30th fraction digit
    [dec("-0.0001"), dec("-0.000100", digits_int=0)],
    # negative zeros: after every negative value, before +0, all equal
    [dec("-0", neg_zero=True), dec("0.00", neg_zero=True, digits_int=0), raw(0, 0, 1, []), raw(18, 30, 1, [0] * 6, rf=3)],
    [dec("0"), raw(0, 0, 0, []), dec("0.000", digits_int=27), raw(9, 9, 0, [0, 0])],
    [dec("0." + "0" * 80 + "1"), raw(0, 81, 0, [0] * 8 + [1])],   # 10^-81, the smallest magnitude 9 words hold
    [dec("1.000000000000000000000000000001")],
    [dec("1.000000000000000000000000000002")],
    [dec("1.000000001")],
    [dec("1.000000002")],
    [dec("1.5"), dec("1.50"), dec("0000000001.5", digits_int=10), dec("1.5", result_frac=30, tail=(123, 10 ** 9 + 5)),
     raw(1, 2, 0, [1, 500000000]), raw(10, 1, 0, [0, 1, 500000000])],
    [dec("123456789012345678901234567890123456.123456789012345678901234567890")],
    [raw(45, 36, 0, [1, 2, 3, 4, 5, 6, 7, 8, 9])],              # 9 words: 5 integer, 4 fraction
    [raw(81, 0, 0, [10 ** 9 - 1] * 9), dec("9" * 81)],
]


def test_hand_cases_order():
    flat = [(i, c) for i, cls in enumerate(ORDERED_CLASSES) for c in cls]
    for i, a in flat:
        for j, b in flat:
            want = -1 if i < j else (1 if i > j else 0)
            assert TD.cmp_decimal(a, b) == want, (i, j)


def _edge_table(rng, n):
    cells = [c for cls in ORDERED_CLASSES for c in cls]
    pick = rng.integers(0, len(cells), n)
    d = np.frombuffer(b"".join(cells[k] for k in pick), np.uint8).reshape(n, 40).copy()
    nulls = rng.random(n) < 0.15
    d[nulls] = rng.integers(0, 256, (int(nulls.sum()), 40), dtype=np.uint8)   # garbage under NULL
    second = rng.integers(-3, 4, n).astype(np.int64)
    d2 = np.frombuffer(b"".join(cells[k] for k in rng.integers(0, len(cells), n)), np.uint8).reshape(n, 40).copy()
    return [(d, nulls), (second, rng.random(n) < 0.1), (d2, np.zeros(n, bool)), (np.arange(n, dtype=np.int64), np.zeros(n, bool))]


@pytest.mark.parametrize("items", [[(0, False)], [(0, True)], [(0, False), (1, True)], [(1, False), (0, True), (2, False)],
                                   [(2, True), (0, False), (3, False)]])
def test_comparator_and_numpy_forms_agree(items):
    rng = np.random.default_rng(len(items) * 7 + int(items[0][1]))
    n = 400
    cols = _edge_table(rng, n)
    kinds = ["decimal", "int", "decimal", "int"]
    rows = [tuple(None if nl[r] else (bytes(v[r]) if v.ndim == 2 else int(v[r])) for v, nl in cols) for r in range(n)]
    exp = TD.topn_rows(rows, kinds, items, 0, n)
    got = TD.topn_order(cols, kinds, items, 0, n)
    assert [r[3] for r in exp] == got.tolist()   # both sort stably: the same rows in the same order
    # item_keys: equal keys exactly on equal ORDER BY values, in any row subset
    k = TD.item_keys(cols, kinds, items, got)
    for x in range(n - 1):
        a, b = rows[got[x]], rows[got[x + 1]]
        same = all((a[c] is None and b[c] is None) or (a[c] is not None and b[c] is not None and TD.cmp_value(a[c], b[c], kinds[c]) == 0)
                   for c, _ in items)
        assert same == bool((k[x] == k[x + 1]).all())
    sub = got[::3]
    assert np.array_equal(TD.item_keys(cols, kinds, items, sub), k[::3])


# ---- tg_topn argument checks (no device needed) ------------------------------------------------------------------
def _call(cols, tps, items, out_elem=None):
    lib = abi.load_lib()
    chk = Chunk(cols)
    cs = chk.to_struct()
    elem = out_elem or [c.elem_len for c in cols]
    out = MutChunk(elem, 16, [DECIMAL_DTYPE if e == 40 else np.int64 for e in elem])
    its = (abi.TgSortItem * len(items))(*[abi.TgSortItem(c, d) for c, d in items])
    ta = (C.c_int32 * len(tps))(*tps)
    fa = (C.c_uint32 * len(tps))(*([0] * len(tps)))
    nr = C.c_int64(-1)
    rc = lib.tg_topn(0, 0, C.byref(cs), ta, fa, its, len(items), C.c_int64(0), C.c_int64(5), C.byref(out.struct), C.byref(nr), None)
    return rc, nr.value


def test_topn_decimal_gate():
    n = 16
    cells = np.frombuffer(b"".join(dec(str(i) + ".25") for i in range(n)), np.uint8).reshape(n, 40).copy()
    ints = np.arange(n, dtype=np.int64)
    L, D = abi.TYPE_LONGLONG, abi.TYPE_NEWDECIMAL
    # a 40-byte column of any type but DECIMAL, as an item or as payload
    assert _call([Column(cells), Column(ints)], [L, L], [(1, 0)])[0] == abi.TG_ERR_UNSUPPORTED
    assert _call([Column(ints), Column(cells)], [L, abi.TYPE_DOUBLE], [(0, 0)])[0] == abi.TG_ERR_UNSUPPORTED
    # an 8-byte column typed DECIMAL is no ORDER BY item
    assert _call([Column(ints), Column(cells)], [D, D], [(0, 0)])[0] == abi.TG_ERR_UNSUPPORTED
    # DECIMAL cells pass the argument checks as an item, a later item and payload: without a device the call stops at
    # the device check; with one it runs
    want = abi.TG_OK if abi.load_lib().tg_device_count() > 0 else abi.TG_ERR_CUDA
    for items in ([(0, 0)], [(1, 1), (0, 0)], [(1, 0)]):
        assert _call([Column(cells), Column(ints)], [D, L], items)[0] == want
