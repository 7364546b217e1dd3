"""CPU-side checks of the DECIMAL VecEval boundary (tg_vec_compare_decimal, tg_vec_filter_ex, tg_decimal_normalize): the
exports and enum values, the argument checks answered before the device is looked for, and the comparison form of a
constant cell against the reference order of tests/topn_decimal.py (cmp_decimal, pinned to TestCompareMyDecimal)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import test_topn_decimal_reference as TR
import topn_decimal as TD
from tidb_b200 import abi
from tidb_b200.chunk import Chunk, Column
from tidb_b200.plan import FilterItem, dec_const_array, filter_array

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L, DBL, DATE, D = abi.TYPE_LONGLONG, abi.TYPE_DOUBLE, abi.TYPE_DATE, abi.TYPE_NEWDECIMAL
U, I = abi.TG_ERR_UNSUPPORTED, abi.TG_ERR_INVALID
BAD_CELLS = [TR.raw(-1, 2, 0, [1, 2]), TR.raw(2, -3, 0, [1]), TR.raw(45, 45, 0, [1] * 9),
             TR.raw(9, 2, 0, [10 ** 9, 0]), TR.raw(9, 2, 0, [5, 10 ** 9])]


@pytest.fixture(scope="module")
def lib():
    from tidb_b200 import build
    build.build()
    return abi.load_lib()


def test_exports_and_enum_values(lib):
    for name in ("tg_vec_compare_decimal", "tg_vec_filter_ex", "tg_decimal_normalize"):
        assert name in abi.EXPORTED_SYMBOLS and hasattr(lib, name), name
    hdr = open(os.path.join(ROOT, "include", "tidbgpu.h")).read()
    m = re.search(r"enum \{ TG_FILTER_INT = (\d+), TG_FILTER_REAL = (\d+), TG_FILTER_DECIMAL = (\d+) \};", hdr)
    assert m and tuple(int(x) for x in m.groups()) == (abi.FILTER_INT, abi.FILTER_REAL, abi.FILTER_DECIMAL) == (0, 1, 2)
    # a DECIMAL FilterItem renders as is_real = TG_FILTER_DECIMAL; the others keep their tg_vec_filter encoding
    arr = filter_array([FilterItem(abi.CMP_LT, 0), FilterItem(abi.CMP_LT, 0, is_real=True),
                        FilterItem(abi.CMP_LT, 0, is_decimal=True, const_cell=TR.dec("1.5"))])
    assert [arr[i].is_real for i in range(3)] == [0, 1, 2]


def test_dec_const_array_layout():
    a, b = TR.dec("0.05"), TR.dec("-7.125")
    items = [FilterItem(abi.CMP_GT, 0), FilterItem(abi.CMP_GE, 1, is_decimal=True, const_cell=a),
             FilterItem(abi.CMP_LE, 1, rhs_col=2, is_decimal=True), FilterItem(abi.CMP_LT, 2, is_decimal=True, const_cell=b)]
    buf = bytes(dec_const_array(items))
    assert len(buf) == 160 and buf[40:80] == a and buf[120:160] == b and buf[:40] == buf[80:120] == bytes(40)
    assert dec_const_array(items[:1] + items[2:3]) is None


def _normalize(lib, cell):
    out = (C.c_uint8 * 40)(*([0xEE] * 40))
    rc = lib.tg_decimal_normalize((C.c_uint8 * 40).from_buffer_copy(bytes(cell)), out)
    return rc, bytes(out)


def test_normalized_constant_keeps_the_order(lib):
    # every hand case of the TopN reference: its comparison form compares with every other hand case as the cell does,
    # and equal values in different forms share one comparison form
    cells = [c for cls in TR.ORDERED_CLASSES for c in cls]
    for i, cls in enumerate(TR.ORDERED_CLASSES):
        forms = set()
        for c in cls:
            rc, nc = _normalize(lib, c)
            assert rc == abi.TG_OK
            forms.add(nc)
            di, df, rf, neg = nc[0], nc[1], nc[2], nc[3]
            assert di % 9 == 0 and df % 9 == 0 and rf == 0 and neg == c[3]
            words = np.frombuffer(nc[4:], np.int32)
            used = di // 9 + df // 9
            assert not words[used:].any()                                      # unused words are 0
            assert used == 0 or (di == 0 or words[0] != 0) and (df == 0 or words[used - 1] != 0)
            assert TD.cmp_decimal(nc, c) == 0
            for other in cells:
                assert TD.cmp_decimal(nc, other) == TD.cmp_decimal(c, other)
                assert TD.cmp_decimal(other, nc) == TD.cmp_decimal(other, c)
        assert len(forms) == 1, i


def test_normalize_rejects_malformed_cells(lib):
    for c in BAD_CELLS:
        rc, out = _normalize(lib, c)
        assert rc == I and out == bytes([0xEE] * 40), c
    assert lib.tg_decimal_normalize(None, (C.c_uint8 * 40)()) == I


# ---- argument checks (no device needed) ---------------------------------------------------------------------------
def _cells(vals):
    return np.frombuffer(b"".join(TR.dec(v) for v in vals), np.uint8).reshape(len(vals), 40).copy()


def _filter_ex(lib, cols, types, items, consts="auto", sel=None):
    chk = Chunk(cols, sel)
    cs = chk.to_struct()
    n = cols[0].length
    out = np.full(max(n, 1), 7, np.uint8)
    cnt = C.c_int64(-5)
    tps = (C.c_int32 * len(types))(*types)
    dc = dec_const_array(items) if consts == "auto" else consts
    rc = lib.tg_vec_filter_ex(0, 0, C.byref(cs), tps, filter_array(items), len(items), dc, out.ctypes.data_as(C.c_void_p), C.byref(cnt), None)
    return rc, out, cnt.value


def _want_ok(lib):
    return abi.TG_OK if lib.tg_device_count() > 0 else abi.TG_ERR_CUDA


def test_filter_ex_argument_checks(lib):
    n = 12
    dec = Column(_cells([f"{i}.25" for i in range(n)]))
    ints = Column(np.arange(n, dtype=np.int64))
    reals = Column(np.arange(n, dtype=np.float64))
    cols, types = [ints, dec, reals, Column(_cells(["-1"] * n))], [L, D, DBL, D]
    k = TR.dec("3.5")
    ok = _want_ok(lib)
    # valid mixes pass the checks: without a device the call stops at the device check
    assert _filter_ex(lib, cols, types, [FilterItem(abi.CMP_GT, 1, is_decimal=True, const_cell=k)])[0] == ok
    assert _filter_ex(lib, cols, types, [FilterItem(abi.CMP_GT, 0, const_i64=3), FilterItem(abi.CMP_LE, 1, rhs_col=3, is_decimal=True),
                                         FilterItem(abi.CMP_NE, 2, is_real=True, const_f64=1.0)])[0] == ok
    assert _filter_ex(lib, cols, types, [FilterItem(abi.CMP_GT, 0, const_i64=3)])[0] == ok          # no DECIMAL item
    # a DECIMAL column in an INT or REAL item, an 8-byte column in a DECIMAL item: UNSUPPORTED
    assert _filter_ex(lib, cols, types, [FilterItem(abi.CMP_GT, 1, const_i64=3)])[0] == U
    assert _filter_ex(lib, cols, types, [FilterItem(abi.CMP_GT, 0, rhs_col=1)])[0] == U
    assert _filter_ex(lib, cols, types, [FilterItem(abi.CMP_GT, 1, is_real=True, const_f64=3.0)])[0] == U
    assert _filter_ex(lib, cols, types, [FilterItem(abi.CMP_GT, 0, is_decimal=True, const_cell=k)])[0] == U
    assert _filter_ex(lib, cols, types, [FilterItem(abi.CMP_GT, 2, is_decimal=True, const_cell=k)])[0] == U
    assert _filter_ex(lib, cols, types, [FilterItem(abi.CMP_GT, 1, rhs_col=0, is_decimal=True)])[0] == U
    # a DATE column typed as such is no DECIMAL operand either
    assert _filter_ex(lib, [Column(np.arange(n, dtype=np.int64)), dec], [DATE, D], [FilterItem(abi.CMP_GT, 0, is_decimal=True, const_cell=k)])[0] == U
    # wrong elem_len: an 8-byte column typed DECIMAL in a DECIMAL item
    assert _filter_ex(lib, [ints, dec], [D, D], [FilterItem(abi.CMP_GT, 0, is_decimal=True, const_cell=k)])[0] == I
    assert _filter_ex(lib, [ints, dec], [D, D], [FilterItem(abi.CMP_GT, 1, rhs_col=0, is_decimal=True)])[0] == I
    # a missing or malformed constant cell
    assert _filter_ex(lib, cols, types, [FilterItem(abi.CMP_GT, 1, is_decimal=True)], consts=None)[0] == I
    for bad in BAD_CELLS:
        assert _filter_ex(lib, cols, types, [FilterItem(abi.CMP_GT, 0, const_i64=3), FilterItem(abi.CMP_GT, 1, is_decimal=True, const_cell=bad)])[0] == I
    # columns out of range, unknown op / item kind
    assert _filter_ex(lib, cols, types, [FilterItem(abi.CMP_GT, 4, is_decimal=True, const_cell=k)])[0] == I
    assert _filter_ex(lib, cols, types, [FilterItem(abi.CMP_GT, -1, is_decimal=True, const_cell=k)])[0] == I
    assert _filter_ex(lib, cols, types, [FilterItem(abi.CMP_GT, 1, rhs_col=4, is_decimal=True)])[0] == I
    assert _filter_ex(lib, cols, types, [FilterItem(6, 1, is_decimal=True, const_cell=k)])[0] == I
    item = FilterItem(abi.CMP_GT, 1, is_decimal=True, const_cell=k)
    arr = filter_array([item]); arr[0].is_real = 3
    cs = Chunk(cols).to_struct()
    out, cnt = np.zeros(n, np.uint8), C.c_int64(0)
    assert lib.tg_vec_filter_ex(0, 0, C.byref(cs), (C.c_int32 * 4)(*types), arr, 1, dec_const_array([item]), out.ctypes.data_as(C.c_void_p), C.byref(cnt), None) == I
    # more than 8 items, NULL col_types
    assert _filter_ex(lib, cols, types, [item] * 9)[0] == U
    assert lib.tg_vec_filter_ex(0, 0, C.byref(cs), None, filter_array([item]), 1, dec_const_array([item]), out.ctypes.data_as(C.c_void_p), C.byref(cnt), None) == I
    # a rejected call writes nothing
    rc, got, c = _filter_ex(lib, cols, types, [FilterItem(abi.CMP_GT, 1, is_decimal=True)], consts=None)
    assert rc == I and (got == 7).all() and c == -5


def _compare(lib, a, b, cell, op=abi.CMP_LT, on_device=0):
    n = a.length
    sa = a.to_struct()
    sb = None if b is None else b.to_struct()
    res = np.full(max(n, 1), 0x5A, np.int64)
    bm = np.full(max((n + 7) // 8, 1), 0xA5, np.uint8)
    k = None if cell is None else (C.c_uint8 * 40).from_buffer_copy(cell)
    rc = lib.tg_vec_compare_decimal(0, on_device, op, C.byref(sa), None if sb is None else C.byref(sb), k,
                                    res.ctypes.data_as(C.c_void_p), bm.ctypes.data_as(C.c_void_p), None)
    assert (res == 0x5A).all() and (bm == 0xA5).all() or rc == abi.TG_OK
    return rc


def test_compare_decimal_argument_checks(lib):
    n = 9
    dec, dec2 = Column(_cells([f"-{i}.5" for i in range(n)])), Column(_cells(["0"] * n))
    ints = Column(np.arange(n, dtype=np.int64))
    ok = _want_ok(lib)
    assert _compare(lib, dec, None, TR.dec("1")) == ok
    assert _compare(lib, dec, dec2, None) == ok
    assert _compare(lib, ints, None, TR.dec("1")) == I                      # elem_len 8
    assert _compare(lib, dec, ints, None) == I
    assert _compare(lib, dec, None, None) == I                              # no constant cell
    for bad in BAD_CELLS:
        assert _compare(lib, dec, None, bad) == I
    assert _compare(lib, dec, Column(_cells(["0"] * (n - 1))), None) == I  # lengths differ
    assert _compare(lib, dec, None, TR.dec("1"), op=7) == I
