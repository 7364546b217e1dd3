"""The string VecEval calls (csrc/vec_string.cu: tg_vec_compare_string, tg_vec_like, tg_vec_filter_ex2) and the
SelectionExec / ProjectionExec shims over var-length columns, exact against tests/string_reference.py (pinned to the
reference's tables by tests/test_string_reference.py).

Rows are drawn from a pool of strings: empty and all-space strings, strings equal up to trailing spaces, tabs, bytes
>= 0x80 and embedded 0x00, valid 2-4 byte runes and every class of invalid sequence, TPC-H-like values, random strings
over {a, b, é, 0xff, %, _, \\, +, space}, and rows longer than a warp's shared-memory tile (a few KiB, and one of
about 100 KiB) among short ones.  The pool's results are computed once; a row's expected value is its pool entry's.
Results are checked bit for bit: 0/1 values (0 under NULL), NULL bitmaps, `selected` bytes and counts."""
import ctypes as C

import numpy as np
import pytest

import mydecimal_args as A
import string_reference as S
from tidb_b200 import abi
from tidb_b200.chunk import Chunk, Column
from tidb_b200.executor import HashAggExec, MockDataSource, ProjectionExec, SelectionExec, drain
from tidb_b200.plan import (AggFunc, AggPlan, ColRef, Const, FieldType, FilterItem, ScalarFunc, dec_const_array,
                            filter_array, str_arg_array)

pytestmark = pytest.mark.gpu
CMP_OPS = [abi.CMP_LT, abi.CMP_LE, abi.CMP_GT, abi.CMP_GE, abi.CMP_EQ, abi.CMP_NE]
SIZES = [1, 31, 33, 1061, 70_001, 4_200_001]
COLLS = [63, 46, 309]            # binary, utf8mb4_bin, utf8mb4_0900_bin: one id per collator behaviour
ALL_BIN_IDS = [63, 46, 83, 65, 47, 309]
VC, L, DBL, DEC = abi.TYPE_VARCHAR, abi.TYPE_LONGLONG, abi.TYPE_DOUBLE, abi.TYPE_NEWDECIMAL
BS = ord("\\")
GUARD = 8


# ---- the string pool -------------------------------------------------------------------------------------------------
SEGMENTS = [b"AUTOMOBILE", b"BUILDING", b"FURNITURE", b"HOUSEHOLD", b"MACHINERY"]
TYPES = [b"PROMO BURNISHED COPPER", b"PROMO PLATED BRASS", b"STANDARD POLISHED BRASS", b"LARGE BRUSHED STEEL",
         b"ECONOMY ANODIZED TIN", b"PROMO", b"promo x"]
COMMENTS = [b"carefully final deposits detect slyly agai", b"special requests sleep", b"pending special packages requests",
            b"the special, bold requests", b"requests special", b"forest green almond", b"blush forest thistle",
            b"ironic green foxes", b"quickly special deposits. regular requests haggle"]
HAND = [b"", b" ", b"   ", b"a", b"a ", b"a  ", b"a\t", b"a\t ", b"a\x00", b"\x00", b"\x00 ", b"ab", b"abc", b"abc ", b"A",
        b"b", b"\x7f", b"\x80", b"\x80\x7f", b"\xff", b"\xff\xfe", b"\xfe", b"\xe9", b"\xc3\xa9", b"\xc3\xa9e", "ée".encode(),
        b"\xe2\x82", b"\xe2\x82\xac", b"\xe2\x82\xac ", b"\xc0\xaf", b"\xe0\x80\xaf", b"\xed\xa0\x80", b"\xf4\x90\x80\x80",
        b"\xf0\x9f\x98", b"\xf0\x9f\x98\x9c", b"\xf0\x9f\x98\x83", "�".encode(), b"\xef\xbf\xbd\xff", b"%", b"_",
        b"\\", b"a%", b"a_b", "À".encode(), "中文".encode(), "汉字".encode(), b"MAIL", b"SHIP", b"AIR", b"MAIL ", b"RAIL"]


def _random_strings(rng, k, alphabet, maxlen):
    return [b"".join(alphabet[j] for j in rng.integers(0, len(alphabet), int(rng.integers(0, maxlen + 1)))) for _ in range(k)]


RAND_ALPHA = [b"a", b"b", "é".encode(), b"\xff", b"%", b"_", b"\\", b"+", b" "]


def _build_pool(seed=11, huge=True):
    rng = np.random.default_rng(seed)
    pool = HAND + SEGMENTS + TYPES + COMMENTS + [s + b" " * int(k) for s, k in zip(SEGMENTS, rng.integers(1, 4, 5))]
    pool += _random_strings(rng, 150, RAND_ALPHA, 8)
    longs = [b"x" * 2100, (b"special " * 400) + b"requests", bytes(rng.integers(0, 256, 3000, dtype=np.uint8)),
             "é".encode() * 2500 + b"%"]
    if huge:
        longs.append(b"".join(COMMENTS[i % len(COMMENTS)] + b" " for i in range(2400))[:100_000])
    pool += longs
    seen, out = set(), []
    for s in pool:
        if s not in seen:
            seen.add(s); out.append(s)
    long_ids = [i for i, s in enumerate(out) if len(s) > 1024]
    return out, long_ids


POOL, LONG_IDS = _build_pool()
SMALL_POOL, SMALL_LONG = _build_pool(huge=False)


def _cmp_matrix(pool, coll):
    return np.array([[S.compare(a, b, coll) for b in pool] for a in pool], dtype=np.int8)


_CACHE = {}


def cmp_matrix(coll):
    if coll not in _CACHE:
        _CACHE[coll] = _cmp_matrix(POOL, coll)
    return _CACHE[coll]


def draw(rng, n, pool_len, long_ids, null_p=0.1):
    """row -> pool index, long rows rare but present; NULL mask"""
    p = np.ones(pool_len)
    p[long_ids] = 1e-6 * pool_len
    idx = rng.choice(pool_len, n, p=p / p.sum())
    if n > 40:
        for k, li in enumerate(long_ids):
            idx[(k * 7919 + 13) % n] = li
    nl = rng.random(n) < null_p
    return idx.astype(np.int64), nl


def make_col(pool, idx, nl, lead=0):
    """the var-length column of pool rows idx (NULL rows keep their bytes), with `lead` bytes before the first row"""
    blob = b"".join(pool)
    po = np.zeros(len(pool) + 1, np.int64)
    np.cumsum([len(s) for s in pool], out=po[1:])
    pb = np.frombuffer(blob, np.uint8)
    base = Column(pb, None, po).take(idx)
    data = np.concatenate([np.full(lead, 0x5A, np.uint8), base.data])
    return Column(data, nl if nl.any() else None, base.offsets + lead)


def _bitmap(nulls):
    return np.packbits(~nulls, bitorder="little")


class Dev:
    """device copies of columns; `shift` moves the data base 1..15 bytes off 16-byte alignment"""

    def __init__(self):
        import torch
        self.torch, self.keep = torch, []

    def col(self, c: Column, shift=0):
        t = self.torch
        s = c.to_struct()
        d = t.zeros(c.data.size + 16 + shift, dtype=t.uint8, device="cuda")
        if c.data.size:
            d[shift:shift + c.data.size] = t.from_numpy(c.data).cuda()
        o = t.from_numpy(c.offsets.copy()).cuda()
        self.keep += [d, o]
        s.data, s.offsets = d.data_ptr() + shift, o.data_ptr()
        if c.null_bitmap is not None:
            m = t.from_numpy(c.null_bitmap.copy()).cuda(); self.keep.append(m); s.null_bitmap = m.data_ptr()
        return s

    def fixed(self, c: Column):
        t = self.torch
        s = c.to_struct()
        d = t.from_numpy(np.ascontiguousarray(c.data).view(np.uint8).reshape(-1).copy()).cuda(); self.keep.append(d)
        s.data = d.data_ptr()
        if c.null_bitmap is not None:
            m = t.from_numpy(c.null_bitmap.copy()).cuda(); self.keep.append(m); s.null_bitmap = m.data_ptr()
        return s


def call_column(fn, a: Column, b=None, const=None, on_device=False, shift=0, **kw):
    """tg_vec_compare_string (fn 'cmp', kw op, coll) or tg_vec_like (fn 'like', kw coll, escape) -> (rc, values, nulls)"""
    lib = abi.load_lib()
    n = a.length
    kb = (C.c_uint8 * max(len(const or b""), 1)).from_buffer_copy((const or b"").ljust(1, b"\0"))
    kp = C.cast(kb, C.c_void_p) if const else None
    if on_device:
        import torch
        dv = Dev()
        sa = dv.col(a, shift)
        sb = dv.col(b, (shift * 7) % 16) if b is not None else None
        res_t = torch.full((max(n, 1),), 0x5A5A5A5A, dtype=torch.int64, device="cuda")
        bm_t = torch.full(((n + 7) // 8 + GUARD,), 0xA5, dtype=torch.uint8, device="cuda")
        rp, bp = C.c_void_p(res_t.data_ptr()), C.c_void_p(bm_t.data_ptr())
    else:
        sa, sb = a.to_struct(), (b.to_struct() if b is not None else None)
        res = np.full(max(n, 1), 0x5A5A5A5A, np.int64)
        bm = np.full((n + 7) // 8 + GUARD, 0xA5, np.uint8)
        rp, bp = res.ctypes.data_as(C.c_void_p), bm.ctypes.data_as(C.c_void_p)
    if fn == "cmp":
        rc = lib.tg_vec_compare_string(0, int(on_device), kw["op"], kw["coll"], C.byref(sa), C.byref(sb) if sb is not None else None,
                                       kp, C.c_int64(len(const or b"")), rp, bp, None)
    else:
        rc = lib.tg_vec_like(0, int(on_device), kw["coll"], C.byref(sa), kp, C.c_int64(len(const or b"")), kw.get("escape", BS), rp, bp, None)
    if on_device:
        torch.cuda.synchronize()
        res, bm = res_t.cpu().numpy(), bm_t.cpu().numpy()
    nb = (n + 7) // 8
    assert (bm[nb:] == 0xA5).all(), "bitmap written past its end"
    return rc, res[:n], bm[:nb]


def check_column(got, expect, nulls):
    rc, res, bm = got
    assert rc == 0, abi.load_lib().tg_last_error()
    exp = np.where(nulls, 0, expect.astype(np.int64))
    bad = np.flatnonzero(res != exp)
    assert bad.size == 0, (bad[:10], res[bad[:10]], exp[bad[:10]])
    assert np.array_equal(bm, _bitmap(nulls)), "NULL bitmap"


# ---- comparisons ------------------------------------------------------------------------------------------------------
CONSTS = [b"BUILDING", b"a", b"a  ", b"\xff", b"", b"\x80", "é".encode(), b"MAIL"]


@pytest.mark.parametrize("n", SIZES)
def test_compare_with_constant(n):
    rng = np.random.default_rng(n)
    idx, nl = draw(rng, n, len(POOL), LONG_IDS)
    col = make_col(POOL, idx, nl)
    consts = CONSTS if n < 100_000 else CONSTS[:1]
    for coll in COLLS:
        for k in consts:
            vec = np.array([S.compare(s, k, coll) for s in POOL])[idx]
            for op in CMP_OPS:
                check_column(call_column("cmp", col, const=k, op=op, coll=coll), S.apply_cmp(op, vec), nl)


@pytest.mark.parametrize("n", SIZES)
def test_compare_column_against_column(n):
    rng = np.random.default_rng(100 + n)
    ia, na = draw(rng, n, len(POOL), LONG_IDS)
    ib, nb_ = draw(rng, n, len(POOL), LONG_IDS)
    eq = rng.random(n) < 0.3                         # many equal and equal-up-to-spaces pairs
    ib[eq] = ia[eq]
    a, b = make_col(POOL, ia, na), make_col(POOL, ib, nb_, lead=5)
    nulls = na | nb_
    for coll in COLLS:
        vec = cmp_matrix(coll)[ia, ib]
        for op in (CMP_OPS if n < 100_000 else [abi.CMP_LT, abi.CMP_EQ]):
            check_column(call_column("cmp", a, b, op=op, coll=coll), S.apply_cmp(op, vec), nulls)


@pytest.mark.parametrize("n", [1, 33, 1061, 70_001])
def test_compare_device_buffers_unaligned_views(n):
    rng = np.random.default_rng(200 + n)
    for shift in (1, 7, 15):
        ia, na = draw(rng, n, len(POOL), LONG_IDS)
        ib, nb_ = draw(rng, n, len(POOL), LONG_IDS)
        a, b = make_col(POOL, ia, na, lead=3 + shift), make_col(POOL, ib, nb_, lead=17)
        for coll in COLLS:
            k = CONSTS[shift % len(CONSTS)]
            vec = np.array([S.compare(s, k, coll) for s in POOL])[ia]
            op = CMP_OPS[shift % 6]
            check_column(call_column("cmp", a, const=k, on_device=True, shift=shift, op=op, coll=coll), S.apply_cmp(op, vec), na)
            check_column(call_column("cmp", a, b, on_device=True, shift=shift, op=op, coll=coll),
                         S.apply_cmp(op, cmp_matrix(coll)[ia, ib]), na | nb_)
            check_column(call_column("cmp", a, const=k, shift=shift, op=op, coll=coll), S.apply_cmp(op, vec), na)


def test_every_bin_collation_id():
    rng = np.random.default_rng(3)
    idx, nl = draw(rng, 5000, len(POOL), LONG_IDS)
    col = make_col(POOL, idx, nl)
    for coll in ALL_BIN_IDS:
        vec = np.array([S.compare(s, b"a ", coll) for s in POOL])[idx]
        check_column(call_column("cmp", col, const=b"a ", op=abi.CMP_EQ, coll=coll), S.apply_cmp(abi.CMP_EQ, vec), nl)
        m = np.array([S.like(s, "%é_%".encode(), BS, coll) for s in POOL])[idx]
        check_column(call_column("like", col, const="%é_%".encode(), coll=coll), m, nl)


# ---- LIKE ---------------------------------------------------------------------------------------------------------------
TPCH_PATTERNS = [b"%special%requests%", b"PROMO%", b"%BRASS", b"%green%", b"forest%", b"%MAIL%", b"BUILDING"]
TRANSCRIBED = [b"", b"a", b"b", b"Aa", b"Aa%", b"aA_", b"b_%b", b"b%_b", b"b_%b%", b"\\a", b"_", b"__", b"%", b"%b", b"%a%",
               b"a%", b"\\%a", b"\\_a", b"\\\\_a", b"%%_", b"%_%_aA", "___Հ".encode(), "%é%".encode(), b"%\xff%", "_�".encode(),
               b"a\\", b"% ", b"%\t"]


_LIKE_CACHE, _RUNES = {}, {}


def _like_vec(pool, pattern, escape, coll):
    """S.like of every pool entry (the pattern compiled once, each entry decoded once)"""
    key = (tuple(pool), pattern, escape, coll)
    if key not in _LIKE_CACHE:
        over = S.collator_of(coll) != S.BINARY
        w, t = S.compile_pattern(pattern, escape, over)
        for x in pool:
            if over and x not in _RUNES:
                _RUNES[x] = S.runes(x)
        _LIKE_CACHE[key] = np.array([S.do_match(_RUNES[x] if over else x, w, t) for x in pool], dtype=bool)
    return _LIKE_CACHE[key]


@pytest.mark.parametrize("n", [1, 33, 1061, 70_001, 4_200_001])
def test_like_tpch_and_transcribed_patterns(n):
    rng = np.random.default_rng(300 + n)
    idx, nl = draw(rng, n, len(POOL), LONG_IDS)
    col = make_col(POOL, idx, nl, lead=n % 9)
    pats = TPCH_PATTERNS + (TRANSCRIBED if n < 100_000 else [])
    for coll in COLLS:
        for pat in pats:
            check_column(call_column("like", col, const=pat, coll=coll), _like_vec(POOL, pat, BS, coll)[idx], nl)


def test_like_random_patterns_and_escapes():
    rng = np.random.default_rng(17)
    n = 4000
    idx, nl = draw(rng, n, len(SMALL_POOL), SMALL_LONG)
    col = make_col(SMALL_POOL, idx, nl)
    for t in range(60):
        pat = b"".join(RAND_ALPHA[j] for j in rng.integers(0, len(RAND_ALPHA), int(rng.integers(0, 7))))
        esc = [BS, ord("%"), ord("_"), ord("+"), 0xE9, 0xFF, ord("a")][t % 7]
        coll = COLLS[t % 3]
        on_device = t % 4 == 3
        check_column(call_column("like", col, const=pat, coll=coll, escape=esc, on_device=on_device, shift=t % 16),
                     _like_vec(SMALL_POOL, pat, esc, coll)[idx], nl)


def test_like_fast_path_both_sides():
    # ASCII literals and '%' only match over bytes in the rune collations; '_' and non-ASCII need the rune walk.  Each
    # pattern here sits on one side of that choice, over strings where the two walks would differ.
    strs = [b"\xe2\x82\xac", b"a\xe2\x82\xacb", b"ab", b"a\xffb", "aéb".encode(), b"a\xc3b", b"", b"a", b"\xff"]
    col = Column.strings(strs * 40)
    nl = np.zeros(len(strs) * 40, bool)
    for pat in (b"a%b", b"%", b"a_b", b"_", b"___", "a%é%".encode(), b"a\xffb", b"%\xff"):
        for coll in COLLS:
            check_column(call_column("like", col, const=pat, coll=coll), _like_vec(strs * 40, pat, BS, coll), nl)


# ---- Selection: mixed CNF -----------------------------------------------------------------------------------------------
def call_filter(cols, types, items, sel=None, on_device=False, shift=0):
    lib = abi.load_lib()
    chk = Chunk(cols, sel)
    cs = chk.to_struct()
    nphys = cols[0].length
    keep = None
    if on_device:
        import torch
        dv = Dev()
        for i, c in enumerate(cols):
            cs.cols[i] = dv.col(c, shift) if c.is_varlen else dv.fixed(c)
        if sel is not None:
            s = torch.from_numpy(chk.sel.copy()).cuda(); dv.keep.append(s); cs.sel = s.data_ptr()
        out_t = torch.full((max(nphys, 1),), 7, dtype=torch.uint8, device="cuda")
        outp = C.c_void_p(out_t.data_ptr())
        keep = dv
    else:
        out = np.full(max(nphys, 1), 7, np.uint8)
        outp = out.ctypes.data_as(C.c_void_p)
    n = C.c_int64(-1)
    tps = (C.c_int32 * len(types))(*types)
    rc = lib.tg_vec_filter_ex2(0, int(on_device), C.byref(cs), tps, filter_array(items), len(items), dec_const_array(items),
                               str_arg_array(items), outp, C.byref(n), None)
    if on_device:
        torch.cuda.synchronize()
        out = out_t.cpu().numpy()
    del keep
    return rc, out[:nphys], n.value


def _mixed_table(n, seed):
    rng = np.random.default_rng(seed)
    ia, na = draw(rng, n, len(POOL), LONG_IDS)
    ib, nb_ = draw(rng, n, len(POOL), LONG_IDS)
    eq = rng.random(n) < 0.3
    ib[eq] = ia[eq]
    iv = rng.integers(-50, 50, n).astype(np.int64)
    inl = rng.random(n) < 0.1
    rv = np.floor(rng.random(n) * 100) / 10
    dv = rng.integers(-500, 500, n)
    dn = rng.random(n) < 0.1
    cells = np.frombuffer(b"".join(A.cell(int(v), 15, 2) for v in dv), np.uint8).reshape(n, 40).copy()
    cols = [make_col(POOL, ia, na), Column(iv, inl if inl.any() else None), make_col(POOL, ib, nb_, lead=2),
            Column(rv), Column(cells, dn if dn.any() else None)]
    return cols, (ia, na, ib, nb_, iv, inl, rv, dv, dn)


TYPES_MIXED = [VC, L, abi.TYPE_BLOB, DBL, DEC]


def _mixed_items():
    return [
        [FilterItem(abi.CMP_NE, 0, is_string=True, const_bytes=b"BUILDING", collation=46), FilterItem(abi.CMP_GT, 1, const_i64=-20)],
        [FilterItem(abi.CMP_EQ, 0, is_string=True, str_kind=abi.STR_NOT_LIKE, const_bytes=b"%special%requests%", collation=309),
         FilterItem(abi.CMP_LE, 3, is_real=True, const_f64=7.5), FilterItem(abi.CMP_GE, 4, is_decimal=True, const_cell=A.cell(-100, 15, 2))],
        [FilterItem(abi.CMP_LT, 0, 2, is_string=True, collation=63), FilterItem(abi.CMP_EQ, 2, is_string=True, str_kind=abi.STR_LIKE,
                                                                              const_bytes=b"%a%", collation=46),
         FilterItem(abi.CMP_LT, 4, is_decimal=True, const_cell=A.cell(250, 15, 2)), FilterItem(abi.CMP_NE, 1, const_i64=0)],
        [FilterItem(abi.CMP_GE, 2, 0, is_string=True, collation=46), FilterItem(abi.CMP_EQ, 0, is_string=True, str_kind=abi.STR_NOT_LIKE,
                                                                              const_bytes=b"_%", collation=309)],
    ]


def filter_reference(tab, items, sel, nphys):
    ia, na, ib, nb_, iv, inl, rv, dv, dn = tab
    s = np.ones(nphys, bool)
    for it in items:
        if it.is_string:
            sides = {0: (ia, na), 2: (ib, nb_)}
            xa, xn = sides[it.lhs_col]
            if it.str_kind == abi.STR_CMP:
                if it.rhs_col >= 0:
                    ya, yn = sides[it.rhs_col]
                    v = S.apply_cmp(it.op, cmp_matrix(it.collation)[xa, ya]) & ~yn
                else:
                    v = S.apply_cmp(it.op, np.array([S.compare(t, it.const_bytes, it.collation) for t in POOL])[xa])
            else:
                m = _like_vec(POOL, it.const_bytes, it.escape, it.collation)[xa]
                v = ~m if it.str_kind == abi.STR_NOT_LIKE else m
            s &= v & ~xn
        elif it.is_decimal:
            s &= S.apply_cmp(it.op, np.sign(dv - CELL_VALUE[it.const_cell])) & ~dn
        elif it.is_real:
            s &= S.apply_cmp(it.op, np.sign(rv - it.const_f64))
        else:
            s &= S.apply_cmp(it.op, np.sign(iv - it.const_i64)) & ~inl
    out = np.zeros(nphys, bool)
    rows = np.arange(nphys) if sel is None else sel
    out[rows] = s[rows]
    return out


CELL_VALUE = {A.cell(v, 15, 2): v for v in (-100, 250)}   # the DECIMAL(15,2) constants of _mixed_items, scaled by 100


@pytest.mark.parametrize("n", [1, 33, 1061, 70_001, 1_000_003])
def test_filter_mixed_cnf(n):
    cols, tab = _mixed_table(n, 400 + n)
    rng = np.random.default_rng(n)
    for k, items in enumerate(_mixed_items()):
        for sel in (None, np.sort(rng.choice(n, max(n // 3, 1), replace=False)).astype(np.int64)):
            for on_device in (False, True):
                rc, got, cnt = call_filter(cols, TYPES_MIXED, items, sel, on_device, shift=k + 1)
                assert rc == 0, abi.load_lib().tg_last_error()
                exp = filter_reference(tab, items, sel, n)
                assert np.array_equal(got, exp.astype(np.uint8)), (k, sel is None, on_device)
                assert cnt == int(exp.sum())


def test_without_string_items_equals_filter_ex():
    n = 70_001
    cols, tab = _mixed_table(n, 9)
    lib = abi.load_lib()
    items = [FilterItem(abi.CMP_GT, 1, const_i64=-20), FilterItem(abi.CMP_LE, 3, is_real=True, const_f64=7.5),
             FilterItem(abi.CMP_GE, 4, is_decimal=True, const_cell=A.cell(-100, 15, 2))]
    for its in (items, items[:2]):
        rc, got, cnt = call_filter(cols, TYPES_MIXED, its)
        assert rc == 0
        cs = Chunk(cols).to_struct()
        out, m = np.full(n, 7, np.uint8), C.c_int64(-1)
        tps = (C.c_int32 * 5)(*TYPES_MIXED)
        assert lib.tg_vec_filter_ex(0, 0, C.byref(cs), tps, filter_array(its), len(its), dec_const_array(its),
                                    out.ctypes.data_as(C.c_void_p), C.byref(m), None) == 0
        assert np.array_equal(got, out) and cnt == m.value


# ---- malformed offsets -----------------------------------------------------------------------------------------------------
def test_malformed_offsets_fail_and_write_nothing():
    n = 3000
    col = Column.strings([b"abcdef"[: i % 7] for i in range(n)])
    bad = col.offsets.copy()
    bad[1500] = bad[1501] + 1              # offsets[1500] > offsets[1501]: row 1500 is bad
    assert bad[1500] <= bad[-1]            # every offset stays inside the buffer
    bcol = Column(col.data, None, bad)
    it = [FilterItem(abi.CMP_EQ, 0, is_string=True, const_bytes=b"ab")]
    for on_device in (False, True):
        rc, out, cnt = call_filter([bcol], [VC], it, None, on_device)
        assert rc == abi.TG_ERR_INVALID
        if not on_device:
            assert (out == 7).all() and cnt == -1
        sel_bad = np.array([0, 5, 1500, 2000], np.int64)
        rc, out, cnt = call_filter([bcol], [VC], it, sel_bad, on_device)
        assert rc == abi.TG_ERR_INVALID
        if not on_device:
            assert (out == 7).all() and cnt == -1
        sel_ok = np.array([0, 2, 5, 1400, 2000, 2999], np.int64)          # the bad rows are outside sel
        rc, out, cnt = call_filter([bcol], [VC], it, sel_ok, on_device)
        assert rc == 0
        exp = np.zeros(n, np.uint8)
        exp[sel_ok] = [col.get_bytes(int(r)) == b"ab" for r in sel_ok]
        assert np.array_equal(out, exp) and cnt == int(exp.sum())
    rc, res, bm = call_column("cmp", bcol, const=b"ab", op=abi.CMP_EQ, coll=46)
    assert rc == abi.TG_ERR_INVALID and (res == 0x5A5A5A5A).all() and (bm == 0xA5).all()
    rc, res, bm = call_column("like", bcol, const=b"a%", coll=46)
    assert rc == abi.TG_ERR_INVALID and (res == 0x5A5A5A5A).all() and (bm == 0xA5).all()
    rc, res, bm = call_column("like", bcol, const=b"a%", coll=46, on_device=True)
    assert rc == abi.TG_ERR_INVALID
    # a row end below offsets[0] in a view
    view = Column(col.data, None, col.offsets[10:21].copy())
    view.offsets[4] = view.offsets[0] - 1
    assert call_column("cmp", view, const=b"a", op=abi.CMP_LT, coll=63)[0] == abi.TG_ERR_INVALID


# ---- the wire codec route ---------------------------------------------------------------------------------------------------
def test_wire_codec_route():
    lib = abi.load_lib()
    rng = np.random.default_rng(21)
    n = 5000
    idx, nl = draw(rng, n, len(SMALL_POOL), SMALL_LONG)
    chk = Chunk([make_col(SMALL_POOL, idx, nl), Column(np.arange(n, dtype=np.int64))])
    cs = chk.to_struct()
    size = C.c_size_t(0)
    assert lib.tg_chunk_wire_size(C.byref(cs), C.byref(size)) == 0
    buf = np.zeros(size.value + 8, np.uint8)
    written = C.c_size_t(0)
    assert lib.tg_chunk_encode(C.byref(cs), buf.ctypes.data_as(C.c_void_p), C.c_size_t(buf.size), C.byref(written)) == 0
    tps = (C.c_int32 * 2)(VC, L)
    dec = (abi.TgColumn * 2)()
    used = C.c_size_t(0)
    assert lib.tg_chunk_decode(buf.ctypes.data_as(C.c_void_p), C.c_size_t(written.value), 2, tps, dec, C.byref(used)) == 0
    assert dec[0].elem_len == -1 and dec[0].offsets
    wire = abi.TgChunk(); wire.ncols = 2; wire.cols = C.cast(dec, C.POINTER(abi.TgColumn)); wire.sel = None; wire.nsel = 0
    items = [FilterItem(abi.CMP_EQ, 0, is_string=True, str_kind=abi.STR_LIKE, const_bytes=b"%a%", collation=46),
             FilterItem(abi.CMP_LT, 1, const_i64=4000)]
    out, m = np.full(n, 7, np.uint8), C.c_int64(-1)
    assert lib.tg_vec_filter_ex2(0, 0, C.byref(wire), tps, filter_array(items), 2, None, str_arg_array(items),
                                 out.ctypes.data_as(C.c_void_p), C.byref(m), None) == 0
    exp = _like_vec(SMALL_POOL, b"%a%", BS, 46)[idx] & ~nl & (np.arange(n) < 4000)
    assert np.array_equal(out, exp.astype(np.uint8)) and m.value == int(exp.sum())


# ---- executors ----------------------------------------------------------------------------------------------------------------
def _sel_chunks(rng, cols, rows_per_chunk=1024):
    out, n = [], cols[0].length
    for lo in range(0, n, rows_per_chunk):
        hi = min(n, lo + rows_per_chunk)
        part = [c.slice(lo, hi) for c in cols]
        sel = np.sort(rng.choice(hi - lo, int((hi - lo) * 0.7), replace=False)).astype(np.int64)
        out.append(Chunk(part, sel))
    return out


@pytest.mark.parametrize("required_rows", [1, 7, 1024])
def test_selection_and_projection_over_strings(required_rows):
    rng = np.random.default_rng(required_rows)
    n = 20_000
    ia, na = draw(rng, n, len(SMALL_POOL), SMALL_LONG)
    ib, nb_ = draw(rng, n, len(SMALL_POOL), SMALL_LONG)
    iv = rng.integers(0, 100, n).astype(np.int64)
    cols = [make_col(SMALL_POOL, ia, na), Column(iv), make_col(SMALL_POOL, ib, nb_)]
    chunks = _sel_chunks(rng, cols)
    logical = np.concatenate([lo * 1024 + c.sel for lo, c in enumerate(chunks)])
    schema = [FieldType(VC, 0), FieldType(L, 0), FieldType(abi.TYPE_STRING, 0)]
    items = [FilterItem(abi.CMP_EQ, 0, is_string=True, str_kind=abi.STR_NOT_LIKE, const_bytes=b"%b%", collation=46),
             FilterItem(abi.CMP_LT, 1, const_i64=70)]
    got = drain(SelectionExec(MockDataSource(schema, chunks), items), required_rows)
    assert all(c.num_rows() <= required_rows for c in got)
    m = ~_like_vec(SMALL_POOL, b"%b%", BS, 46)[ia] & ~na & (iv < 70)
    keep = logical[m[logical]]
    vals_a = [v for c in got for v in c.columns[0].values()]
    vals_b = [v for c in got for v in c.columns[2].values()]
    assert vals_a == [SMALL_POOL[i] for i in ia[keep]]
    assert vals_b == [None if nb_[r] else SMALL_POOL[ib[r]] for r in keep]
    assert np.array_equal(np.concatenate([c.columns[1].data for c in got]), iv[keep])
    # projection: pass the string columns through, compare them and match a pattern
    exprs = [ColRef(0), ScalarFunc("cmp", abi.CMP_LE, (ColRef(0), ColRef(2)), is_string=True, collation=46),
             ScalarFunc("cmp", abi.CMP_GT, (ColRef(2), Const(bytes_value=b"b")), is_string=True, collation=63),
             ScalarFunc("like", 0, (ColRef(0), Const(bytes_value="%é%".encode())), collation=309), ColRef(2)]
    got = drain(ProjectionExec(MockDataSource(schema, chunks), exprs), required_rows)
    assert all(c.num_rows() <= required_rows for c in got)
    assert [v for c in got for v in c.columns[0].values()] == [None if na[r] else SMALL_POOL[ia[r]] for r in logical]
    assert [v for c in got for v in c.columns[4].values()] == [None if nb_[r] else SMALL_POOL[ib[r]] for r in logical]
    cm = np.array([[S.compare(x, y, 46) for y in SMALL_POOL] for x in SMALL_POOL])
    for k, exp, nulls in ((1, cm[ia, ib] <= 0, na | nb_),
                          (2, np.array([S.compare(x, b"b", 63) for x in SMALL_POOL])[ib] > 0, nb_),
                          (3, _like_vec(SMALL_POOL, "%é%".encode(), BS, 309)[ia], na)):
        v = np.concatenate([c.columns[k].data for c in got])
        nl = np.concatenate([c.columns[k].nulls() for c in got])
        assert np.array_equal(nl, nulls[logical]), k
        assert np.array_equal(v, np.where(nulls, 0, exp)[logical].astype(np.int64)), k


def test_q13_shape_end_to_end():
    # select c_custkey, count(o_orderkey) from orders where o_comment not like '%special%requests%' group by o_custkey
    rng = np.random.default_rng(13)
    n = 300_000
    words = [b"carefully", b"final", b"special", b"pending", b"requests", b"deposits", b"ironic", b"packages", b"slyly"]
    vocab = [b" ".join(words[j] for j in rng.integers(0, len(words), int(rng.integers(3, 9)))) for _ in range(2000)]
    ci = rng.integers(0, len(vocab), n)
    cust = rng.integers(0, 5000, n).astype(np.int64)
    comment = make_col(vocab, ci, np.zeros(n, bool))
    chunks = Chunk([Column(cust), Column(np.arange(n, dtype=np.int64)), comment]).split(1024)
    schema = [FieldType(L, abi.FLAG_NOT_NULL), FieldType(L, abi.FLAG_NOT_NULL), FieldType(VC, abi.FLAG_NOT_NULL)]
    sel = SelectionExec(MockDataSource(schema, chunks),
                        [FilterItem(abi.CMP_EQ, 2, is_string=True, str_kind=abi.STR_NOT_LIKE, const_bytes=b"%special%requests%")])
    proj = ProjectionExec(sel, [ColRef(0), ColRef(1)])
    plan = AggPlan([schema[0], schema[1]], [0], [AggFunc(abi.AGG_FIRSTROW, 0), AggFunc(abi.AGG_COUNT, 1, L)])
    out = drain(HashAggExec(plan, proj))
    keys = np.concatenate([c.columns[0].data for c in out])
    cnts = np.concatenate([c.columns[1].data for c in out])
    keep = np.array([not (b"special" in v and v.find(b"requests", v.find(b"special") + 7) >= 0) for v in vocab])[ci]
    exp = np.bincount(cust[keep], minlength=5000)
    assert len(keys) == int((exp > 0).sum())
    assert np.array_equal(cnts, exp[keys])
