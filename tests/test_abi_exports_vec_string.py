"""CPU-side checks of the string VecEval boundary (tg_vec_filter_ex2, tg_vec_compare_string, tg_vec_like): the exports
and enum values, the Python renderings of STRING items, and the argument checks answered before the device is looked
for (each answer below is the one a machine with a GPU gives too)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from tidb_b200 import abi
from tidb_b200.chunk import Chunk, Column
from tidb_b200.plan import FilterItem, filter_array, str_arg_array

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U, I = abi.TG_ERR_UNSUPPORTED, abi.TG_ERR_INVALID
VC, L, DEC = abi.TYPE_VARCHAR, abi.TYPE_LONGLONG, abi.TYPE_NEWDECIMAL


@pytest.fixture(scope="module")
def lib():
    from tidb_b200 import build
    build.build()
    return abi.load_lib()


def test_exports_and_enum_values(lib):
    for name in ("tg_vec_filter_ex2", "tg_vec_compare_string", "tg_vec_like"):
        assert name in abi.EXPORTED_SYMBOLS and hasattr(lib, name), name
    hdr = open(os.path.join(ROOT, "include", "tidbgpu.h")).read()
    assert re.search(r"enum \{ TG_FILTER_STRING = 3 \};", hdr) and abi.FILTER_STRING == 3
    m = re.search(r"enum \{ TG_STR_CMP = (\d+), TG_STR_LIKE = (\d+), TG_STR_NOT_LIKE = (\d+) \};", hdr)
    assert m and tuple(int(x) for x in m.groups()) == (abi.STR_CMP, abi.STR_LIKE, abi.STR_NOT_LIKE) == (0, 1, 2)
    # pkg/parser/mysql/type.go
    for name, val in (("VARCHAR", 15), ("BIT", 16), ("JSON", 0xF5), ("ENUM", 0xF7), ("SET", 0xF8), ("TINY_BLOB", 0xF9),
                      ("MEDIUM_BLOB", 0xFA), ("LONG_BLOB", 0xFB), ("BLOB", 0xFC), ("VARSTRING", 0xFD), ("STRING", 0xFE)):
        assert re.search(rf"TG_TYPE_{name} = {val:#x}\b" if val > 99 else rf"TG_TYPE_{name} = {val}\b", hdr), name
        assert getattr(abi, "TYPE_" + name) == val
    assert C.sizeof(abi.TgStrArg) == 32


def test_str_arg_array_layout():
    items = [FilterItem(abi.CMP_GT, 0), FilterItem(abi.CMP_EQ, 1, is_string=True, const_bytes=b"BUILDING", collation=46),
             FilterItem(abi.CMP_EQ, 1, is_string=True, str_kind=abi.STR_NOT_LIKE, const_bytes=b"%special%requests%", escape=0x2B),
             FilterItem(abi.CMP_LT, 1, 2, is_string=True, collation=63)]
    arr = filter_array(items)
    assert [arr[i].is_real for i in range(4)] == [0, 3, 3, 3]
    sa = str_arg_array(items)
    assert sa[0].bytes is None and sa[0].len == 0
    assert C.string_at(sa[1].bytes, sa[1].len) == b"BUILDING" and sa[1].collation == 46 and sa[1].kind == abi.STR_CMP
    assert C.string_at(sa[2].bytes, sa[2].len) == b"%special%requests%" and sa[2].kind == abi.STR_NOT_LIKE and sa[2].escape == 0x2B
    assert sa[3].bytes is None and sa[3].len == 0 and sa[3].collation == 63
    assert str_arg_array(items[:1]) is None


def test_column_strings_roundtrip():
    vals = [b"a", None, b"", b"\xff\x00 ", b"BUILDING"]
    c = Column.strings(vals)
    assert c.elem_len == -1 and c.length == 5 and list(c.offsets) == [0, 1, 1, 1, 4, 12]
    assert c.values() == vals
    assert c.slice(2, 5).values() == vals[2:5] and c.take(np.array([4, 1, 0])).values() == [vals[4], None, vals[0]]
    s = c.to_struct()
    assert s.elem_len == -1 and s.offsets == c.offsets.ctypes.data and s.length == 5


def _chunk(cols):
    return Chunk(cols)


def _filter(lib, chk, types, items, on_device=0):
    cs = chk.to_struct()
    sel = np.zeros(max(chk.columns[0].length, 1), np.uint8)
    n = C.c_int64(-7)
    tps = (C.c_int32 * len(types))(*types)
    rc = lib.tg_vec_filter_ex2(0, on_device, C.byref(cs), tps, filter_array(items), len(items), None, str_arg_array(items),
                               sel.ctypes.data_as(C.c_void_p), C.byref(n), None)
    return rc, n.value


def _cols():
    return [Column.strings([b"a", b"bb", None]), Column(np.arange(3, dtype=np.int64)), Column(np.zeros((3, 40), np.uint8))]


@pytest.mark.parametrize("collation", [33, 45, 224, 255, 28, 87, 248, 0, 8, -1])
def test_unsupported_collation(lib, collation):
    it = FilterItem(abi.CMP_EQ, 0, is_string=True, const_bytes=b"a", collation=collation)
    assert _filter(lib, _chunk(_cols()), [VC, L, DEC], [it]) == (U, -7)
    a = _cols()[0].to_struct()
    res, nl = np.zeros(3, np.int64), np.zeros(1, np.uint8)
    assert lib.tg_vec_compare_string(0, 0, abi.CMP_EQ, collation, C.byref(a), None, b"a", C.c_int64(1),
                                     res.ctypes.data_as(C.c_void_p), nl.ctypes.data_as(C.c_void_p), None) == U
    assert lib.tg_vec_like(0, 0, collation, C.byref(a), b"a%", C.c_int64(2), ord("\\"),
                           res.ctypes.data_as(C.c_void_p), nl.ctypes.data_as(C.c_void_p), None) == U


@pytest.mark.parametrize("escape", [-1, 256, 1000])
def test_bad_escape(lib, escape):
    it = FilterItem(abi.CMP_EQ, 0, is_string=True, str_kind=abi.STR_LIKE, const_bytes=b"a%", escape=escape)
    assert _filter(lib, _chunk(_cols()), [VC, L, DEC], [it]) == (I, -7)
    a = _cols()[0].to_struct()
    res, nl = np.zeros(3, np.int64), np.zeros(1, np.uint8)
    assert lib.tg_vec_like(0, 0, 46, C.byref(a), b"a%", C.c_int64(2), escape,
                           res.ctypes.data_as(C.c_void_p), nl.ctypes.data_as(C.c_void_p), None) == I


@pytest.mark.parametrize("tp", [abi.TYPE_ENUM, abi.TYPE_SET, abi.TYPE_JSON, abi.TYPE_BIT, L])
def test_non_string_column_in_string_item(lib, tp):
    it = FilterItem(abi.CMP_EQ, 0, is_string=True, const_bytes=b"a")
    assert _filter(lib, _chunk(_cols()), [tp, L, DEC], [it]) == (U, -7)
    it = FilterItem(abi.CMP_EQ, 1, is_string=True, const_bytes=b"a")      # an 8-byte column typed as a string
    assert _filter(lib, _chunk(_cols()), [VC, VC, DEC], [it])[0] == I


@pytest.mark.parametrize("tp", abi.STRING_TYPES)
def test_string_column_in_other_items(lib, tp):
    for it in (FilterItem(abi.CMP_EQ, 0, is_decimal=True, rhs_col=2), FilterItem(abi.CMP_EQ, 0, const_i64=1),
               FilterItem(abi.CMP_EQ, 0, is_real=True)):
        assert _filter(lib, _chunk(_cols()), [tp, L, DEC], [it]) == (U, -7)
    it = FilterItem(abi.CMP_EQ, 0, 1, is_string=True)                    # string against an integer column
    assert _filter(lib, _chunk(_cols()), [tp, L, DEC], [it]) == (U, -7)


@pytest.mark.parametrize("tp", abi.STRING_TYPES)
def test_string_typed_fixed_column_in_other_items(lib, tp):
    # an 8-byte column whose type says string: refused in an INT / REAL item by its type, with or without a STRING item
    cols = _cols()
    for it in (FilterItem(abi.CMP_EQ, 1, const_i64=1), FilterItem(abi.CMP_EQ, 1, is_real=True), FilterItem(abi.CMP_LT, 1, 1)):
        assert _filter(lib, _chunk(cols), [VC, tp, DEC], [it]) == (U, -7)
        assert _filter(lib, _chunk(cols), [VC, tp, DEC], [FilterItem(abi.CMP_EQ, 0, is_string=True, const_bytes=b"a"), it]) == (U, -7)


def test_host_offsets_end_before_start(lib):
    c = Column(np.frombuffer(b"abcdef", np.uint8), None, np.array([4, 5, 6, 2], np.int64))
    it = FilterItem(abi.CMP_EQ, 0, is_string=True, const_bytes=b"a")
    assert _filter(lib, _chunk([c]), [VC], [it]) == (I, -7)
    a = c.to_struct()
    res, nl = np.full(3, 9, np.int64), np.full(1, 0xAB, np.uint8)
    assert lib.tg_vec_compare_string(0, 0, abi.CMP_EQ, 46, C.byref(a), None, b"a", C.c_int64(1),
                                     res.ctypes.data_as(C.c_void_p), nl.ctypes.data_as(C.c_void_p), None) == I
    assert list(res) == [9, 9, 9] and nl[0] == 0xAB


def test_other_argument_checks(lib):
    cols = _cols()
    # unknown kind, unknown op, a NULL constant with a length, too many items, a string item without str_args
    assert _filter(lib, _chunk(cols), [VC, L, DEC], [FilterItem(abi.CMP_EQ, 0, is_string=True, str_kind=3, const_bytes=b"a")])[0] == I
    assert _filter(lib, _chunk(cols), [VC, L, DEC], [FilterItem(9, 0, is_string=True, const_bytes=b"a")])[0] == I
    assert _filter(lib, _chunk(cols), [VC, L, DEC], [FilterItem(abi.CMP_EQ, 0, is_string=True)] * 9)[0] == U
    cs = _chunk(cols).to_struct()
    sel, n = np.zeros(3, np.uint8), C.c_int64(0)
    tps = (C.c_int32 * 3)(VC, L, DEC)
    rc = lib.tg_vec_filter_ex2(0, 0, C.byref(cs), tps, filter_array([FilterItem(abi.CMP_EQ, 0, is_string=True)]), 1, None, None,
                               sel.ctypes.data_as(C.c_void_p), C.byref(n), None)
    assert rc == I
    bad = (abi.TgStrArg * 1)()
    bad[0].bytes, bad[0].len, bad[0].collation = None, 4, 46
    rc = lib.tg_vec_filter_ex2(0, 0, C.byref(cs), tps, filter_array([FilterItem(abi.CMP_EQ, 0, is_string=True)]), 1, None, bad,
                               sel.ctypes.data_as(C.c_void_p), C.byref(n), None)
    assert rc == I
