"""The string VecEval kernel (csrc/vec_string.cu, k_vec_string) at the edges of its warp staging, rune decoding, byte
fast path and `sel` handling, against like_dp_reference.py (tokens and a DP table, not the kernel's walk).

Every STRING item here runs through tg_vec_compare_string or tg_vec_like with host and device columns, and through
tg_vec_filter_ex2 with and without a sel vector (a sel vector sends every row down the global-memory path, so each case
compares the staged and the unstaged read of the same rows).  A warp stages its 32-row tile into shared memory when the
tile's bytes fit 2048; the staging copy keeps the source's alignment mod 16, so the cases place tiles at every
alignment with short spacer tiles ahead of them."""
import ctypes as C

import numpy as np
import pytest

import like_dp_reference as P
import mydecimal_args as A
from test_gpu_vec_string import call_column, call_filter, check_column
from tidb_b200 import abi
from tidb_b200.chunk import Column
from tidb_b200.plan import FilterItem

pytestmark = pytest.mark.gpu

VC, L, DBL, DEC = abi.TYPE_VARCHAR, abi.TYPE_LONGLONG, abi.TYPE_DOUBLE, abi.TYPE_NEWDECIMAL
LT, LE, GT, GE, EQ, NE = abi.CMP_LT, abi.CMP_LE, abi.CMP_GT, abi.CMP_GE, abi.CMP_EQ, abi.CMP_NE
CMP, LIKE, NOT_LIKE = abi.STR_CMP, abi.STR_LIKE, abi.STR_NOT_LIKE
BS = ord("\\")
COLLS = (63, 46, 309)
STAGE_CAP = 2048
FFFD = "�".encode()


def apply_cmp(op, c):
    return (c < 0, c <= 0, c > 0, c >= 0, c == 0, c != 0)[op]


# ---- columns -----------------------------------------------------------------------------------------------------------
def column(rows, nulls=None, lead=0):
    """a var-length column of `rows` (bytes; NULL rows keep their bytes) whose data starts `lead` junk bytes before
    row 0, so offsets[0] == lead"""
    lens = np.array([len(r) for r in rows], np.int64)
    offs = np.full(len(rows) + 1, lead, np.int64)
    np.cumsum(lens, out=offs[1:])
    offs[1:] += lead
    data = np.frombuffer(b"\x5a" * lead + b"".join(rows), np.uint8).copy()
    nl = None if nulls is None or not np.any(nulls) else np.asarray(nulls, bool)
    return Column(data, nl, offs)


TILE_ALPHA = [b"a", b"b", b"x", b"y", b" ", b"%", b"_", b"\xc3", b"\xa9", b"\xe2", b"\x82", b"\xac", b"\xff", b"\xe0",
              b"\xa0", b"\x80", b"\x9f"]


def tile_rows(rng, total, last_nonempty=True):
    """32 rows whose bytes total `total`: random bytes (valid, truncated and overlong UTF-8 among ASCII) cut at random
    points, so runes are split across rows"""
    blob = b"".join(TILE_ALPHA[i] for i in rng.integers(0, len(TILE_ALPHA), total))
    cuts = np.sort(rng.integers(0, total + 1, 31))
    if last_nonempty:
        cuts = np.minimum(cuts, total - 1)
    bounds = [0] + cuts.tolist() + [total]
    return [blob[bounds[i]:bounds[i + 1]] for i in range(32)]


def aligned_tiles(rng, total, phase=0):
    """16 tiles of `total` bytes, tile k starting at byte offset == k + phase (mod 16) of the column, each after a
    32-row spacer tile whose one non-empty row sets that offset -> rows, and the row index of each test tile"""
    rows, at, starts = [], 0, []
    for k in range(16):
        gap = (k + phase - at) % 16
        rows += [b"s" * gap] + [b""] * 31
        at += gap
        starts.append(len(rows))
        rows += tile_rows(rng, total)
        at += total
    return rows, starts


# ---- one STRING item through every call -----------------------------------------------------------------------------------
def expected(kind, a_rows, b_rows=None, const=None, op=EQ, coll=46, escape=BS):
    if kind == CMP:
        other = b_rows if b_rows is not None else [const] * len(a_rows)
        return np.array([apply_cmp(op, P.compare(x, y, coll)) for x, y in zip(a_rows, other)], bool)
    m = np.array([P.like(x, const, escape, coll) for x in a_rows], bool)
    return ~m if kind == NOT_LIKE else m


def run_item(kind, a_rows, a_nulls=None, b_rows=None, b_nulls=None, const=None, op=EQ, coll=46, escape=BS, lead=0,
             shifts=(0, 5), sels=("all", "sparse"), exp=None):
    """the item over column a (and b) through the column call (host, device at each shift), and through
    tg_vec_filter_ex2 (host and device, without and with sel vectors); every result checked against the DP reference"""
    n = len(a_rows)
    an = np.zeros(n, bool) if a_nulls is None else np.asarray(a_nulls, bool)
    bn = np.zeros(n, bool) if b_nulls is None else np.asarray(b_nulls, bool)
    a = column(a_rows, an, lead)
    b = column(b_rows, bn, lead=(lead * 3 + 7) % 19) if b_rows is not None else None
    nulls = an | (bn if b is not None else False)
    if exp is None:
        exp = expected(kind, a_rows, b_rows, const, op, coll, escape)
    tag = (kind, op, coll, escape, const[:40] if const else None)
    if kind == CMP:
        kw = dict(op=op, coll=coll)
        fn = "cmp"
    else:
        kw = dict(coll=coll, escape=escape)
        fn = "like"
    if kind != NOT_LIKE:   # the column calls have no NOT LIKE
        check_column(call_column(fn, a, b, const=const if b is None else None, **kw), exp, nulls)
        for s in shifts:
            check_column(call_column(fn, a, b, const=const if b is None else None, on_device=True, shift=s, **kw), exp, nulls)
    item = FilterItem(op, 0, 1 if b is not None else -1, is_string=True, const_bytes=const if b is None else None,
                      collation=coll, str_kind=kind, escape=escape)
    cols, types = ([a, b], [VC, VC]) if b is not None else ([a], [VC])
    want = exp & ~nulls
    rng = np.random.default_rng(n)
    variants = [(None, False, 0), (None, True, 3)]
    for s in sels:
        if s == "all":
            variants.append((np.arange(n, dtype=np.int64), False, 0))
        elif s == "sparse" and n:
            variants.append((np.sort(rng.choice(n, max(n // 5, 1), replace=False)).astype(np.int64), True, 9))
    for sel, dev, shift in variants:
        rc, got, cnt = call_filter(cols, types, [item], sel, dev, shift)
        assert rc == 0, (tag, abi.load_lib().tg_last_error())
        w = np.zeros(n, bool)
        rows = np.arange(n) if sel is None else sel
        w[rows] = want[rows]
        bad = np.flatnonzero(got != w)
        assert bad.size == 0, (tag, sel is not None, dev, bad[:8], [a_rows[i][:40] for i in bad[:4]])
        assert cnt == int(w.sum()), tag
    return exp


# ---- staging boundary ---------------------------------------------------------------------------------------------------
TILE_PATTERNS = [b"%", b"%b", b"%\xff", "%é".encode(), b"%_", b"_%", b"%__", b"a%", b"%a%b%", b"x__", b"%\xe2\x82\xac%",
                 b"%" + FFFD, b"___", b"%b_", b"%y", b"%\\%%"]


@pytest.mark.parametrize("total", [STAGE_CAP, STAGE_CAP + 1])
def test_staging_boundary_every_alignment(total):
    rng = np.random.default_rng(total)
    rows, starts = aligned_tiles(rng, total)
    n = len(rows)
    for s in starts:
        assert sum(len(r) for r in rows[s:s + 32]) == total
    nl = np.zeros(n, bool)
    nl[starts[3] + 5] = nl[starts[9] + 31] = True   # NULL rows inside staged tiles keep their bytes
    for coll in COLLS:
        for pat in TILE_PATTERNS:
            run_item(LIKE, rows, nl, const=pat, coll=coll, lead=coll % 13, shifts=(0, 7), sels=("all",))
        # constants: the last row of a few tiles, exactly and with its last byte changed
        for s in starts[::5]:
            last = rows[s + 31]
            for k in (last, last[:-1], last[:-1] + bytes([last[-1] ^ 1])):
                for op in (LT, EQ, GT):
                    run_item(CMP, rows, nl, const=k, op=op, coll=coll, lead=1, shifts=(0,), sels=("all",))
    # column against column: b holds the same rows at other alignments, a few changed in their last byte
    b_rows, b_starts = aligned_tiles(np.random.default_rng(total), total, phase=5)
    assert b_starts == starts and [b_rows[s:s + 32] for s in b_starts] == [rows[s:s + 32] for s in starts]
    for k in range(0, 16, 3):
        r = b_starts[k] + 31
        b_rows[r] = b_rows[r][:-1] + bytes([b_rows[r][-1] ^ 2])
    for coll in COLLS:
        for op in (LT, EQ, GT, NE):
            run_item(CMP, rows, nl, b_rows=b_rows, op=op, coll=coll, lead=4, shifts=(0, 11), sels=("all", "sparse"))


# ---- row shapes ---------------------------------------------------------------------------------------------------------
def shapes_column(rng):
    """tiles: one row over 2048 bytes among short ones; one row of exactly 2048 bytes and 31 empty rows; a 2048-byte
    row with short ones (over the cap); only empty rows; all NULL; NULL rows that own bytes"""
    short = lambda: tile_rows(rng, 200)
    long_row = b"xa" * 1100 + "é".encode() + b"b"
    t1 = short(); t1[13] = long_row
    exact = b"a" + b"\xe2\x82\xac" * 682 + b"b"
    assert len(exact) == STAGE_CAP
    t2 = [exact] + [b""] * 31
    t3 = short(); t3[31] = exact
    t4 = [b""] * 32
    t5 = short()
    t6 = short()
    rows = t1 + t2 + t3 + t4 + t5 + t6 + short()
    nulls = np.zeros(len(rows), bool)
    nulls[128:160] = True                      # t5: all NULL (bytes kept)
    nulls[160:192:3] = True                    # t6: every third row NULL, with bytes
    return rows, nulls


SHAPE_PATTERNS = [b"%", b"", b"%b", b"a%", b"_", b"%\xe2\x82\xac_", b"%a_", "%é%".encode(), b"%\xe2%"]


def test_row_shapes():
    rng = np.random.default_rng(1)
    rows, nulls = shapes_column(rng)
    for coll in COLLS:
        for pat in SHAPE_PATTERNS:
            run_item(LIKE, rows, nulls, const=pat, coll=coll, lead=3)
        for k in (b"", rows[32], rows[13], b"a"):
            for op in (LT, EQ, GE):
                run_item(CMP, rows, nulls, const=k, op=op, coll=coll, shifts=(9,))
        other = rows[32:] + rows[:32]
        run_item(CMP, rows, nulls, b_rows=other, b_nulls=np.roll(nulls, -32), op=LE, coll=coll)
        run_item(NOT_LIKE, rows, nulls, const=b"%b", coll=coll)


@pytest.mark.parametrize("long_last", [False, True], ids=["staged", "over_cap"])
def test_partial_last_tile(long_last):
    rng = np.random.default_rng(int(long_last))
    last = (b"xy" * 1050 if long_last else b"xy" * 50) + "é".encode() + b"\xe2\x82" + b"b"
    for r in range(1, 32):
        rows = tile_rows(rng, 500) + tile_rows(rng, 300)[:r - 1] + [last]
        assert len(rows) == 32 + r
        for coll in (46, 63):
            for pat in (b"%b", b"%\xe2\x82_", "%é%".encode(), b"x%y%"):
                run_item(LIKE, rows, const=pat, coll=coll, lead=r, shifts=(r % 16,), sels=("all",))
            run_item(CMP, rows, const=last, op=EQ, coll=coll, shifts=(r % 16,), sels=())
            run_item(CMP, rows, const=last[:-1], op=GT, coll=coll, shifts=(), sels=())


# ---- rune decoding at row ends ------------------------------------------------------------------------------------------
def test_runes_split_across_rows():
    # a truncated sequence at a row's end whose continuation bytes begin the next row: each stray byte is one U+FFFD
    base = [b"x\xe2\x82", b"\xacy", b"x\xe2", b"\x82\xacy", b"x\xf0\x9f", b"\x98\x9cy", b"x\xc3", b"\xa9y", b"x\xe0\x80",
            b"\x80y", b"x\xe0\x9f\xbf", b"x\xe0\xa0\x80", b"\xe0\x80\x80", b"x\xed\xa0\x80", b"x\xe2\x82\xac", b"\xac"]
    rows = base * 40 + base[:7]
    cases = [b"x__", b"x___", b"x_", b"_y", b"__y", b"___y", b"%_", b"x%", b"%y", b"x_%", b"_", b"___", b"x____", b"%\xac%"]
    for coll in COLLS:
        for pat in cases:
            run_item(LIKE, rows, const=pat, coll=coll, lead=1)
    # the 2-rune and 3-rune counts the DP reference gives, written out for the staged rows
    assert P.like(b"x\xe2\x82", b"x__", BS, 46) and not P.like(b"x\xe2\x82", b"x_", BS, 46)
    assert P.like(b"\xacy", b"__", BS, 46) and P.like(b"x\xe0\x80", b"x__", BS, 46)
    assert P.like(b"x\xe0\xa0\x80", b"x_", BS, 46) and P.like(b"\xe0\x80\x80", b"___", BS, 309)


def test_fffd_literal_against_invalid_bytes():
    rows = [b"\xff", b"\xe2\x82", b"\xc0\xaf", FFFD, b"a\xffb", b"a" + FFFD + b"b", b"ab", b"\xe0\x80\x80", b"", b"\xed\xa0\x80"]
    rows = rows * 7
    for pat in (FFFD, b"a" + FFFD + b"b", b"%" + FFFD + b"%", FFFD * 2, FFFD * 3, b"_" + FFFD):
        m46 = run_item(LIKE, rows, const=pat, coll=46)
        m309 = run_item(LIKE, rows, const=pat, coll=309)
        m63 = run_item(LIKE, rows, const=pat, coll=63)
        assert np.array_equal(m46, m309)
        if pat in (FFFD, b"a" + FFFD + b"b"):
            assert m46[0] if pat == FFFD else m46[4]          # an invalid byte matches U+FFFD over runes
            assert not m63[0] and not m63[4]                  # over bytes it does not
            assert m63[3] if pat == FFFD else m63[5]          # the encoded U+FFFD matches itself either way


# ---- byte fast path against the rune walk --------------------------------------------------------------------------------
FAST_ROWS_ALPHA = [b"a", b"b", b"c", b"%", b"\xc3\xa9", b"\xe2\x82\xac", b"\xe2\x82", b"\xff", b"\xc3", b"\xa9", b"\xf0\x9f\x98\x9c",
                   b"\xe0\x80\xaf", b"\xed\xa0\x80", b" "]


def test_fast_path_against_rune_walk():
    rng = np.random.default_rng(8)
    rows = [b"".join(FAST_ROWS_ALPHA[i] for i in rng.integers(0, len(FAST_ROWS_ALPHA), int(rng.integers(0, 12))))
            for _ in range(3000)]
    fast = [b"%a%", b"a%b", b"%a%b%c%", b"%ab", b"b%", b"%\\%%", b"a%%b", b"%c"]
    for pat in fast:
        for coll in (46, 309):
            w, t = P.S.compile_pattern(pat, BS, True)
            assert P.like_bytes_ok(w, t), pat
            run_item(LIKE, rows, const=pat, coll=coll, shifts=(2,))
    # one non-ASCII literal more: the rune walk
    for pat in ("%a%é%".encode(), "a%é".encode(), b"%a%\xe2\x82\xac%", b"%\xff%", b"%a" + FFFD, "%é%b%c%".encode(), b"a%_b"):
        for coll in (46, 309):
            w, t = P.S.compile_pattern(pat, BS, True)
            assert not P.like_bytes_ok(w, t), pat
            run_item(LIKE, rows, const=pat, coll=coll, shifts=(2,))


# ---- escapes ------------------------------------------------------------------------------------------------------------
def test_every_escape_byte():
    rows = [b"", b"a", b"%", b"_", b"\\", b"a%", b"a_", b"%a", b"_a", b"ab", b"\\a", "é".encode(), "é%".encode(), b"\xe9%",
            b"\xe9", b"a\xff", b"\xff", b"%%", b"__", b"a\\", b"\x00%", b"aa", b"a%b", b"\x7f_"] * 3
    for e in range(256):
        eb = bytes([e])
        pats = [b"a" + eb + b"%", eb + b"_%", b"%" + eb, eb + eb + b"%", "é".encode() + eb + b"%", b"a%" + eb + b"_"]
        for coll in COLLS:
            for pat in pats:
                run_item(LIKE, rows, const=pat, coll=coll, escape=e, shifts=(), sels=())
        run_item(LIKE, rows, const=pats[0], coll=46, escape=e, shifts=(e % 16,), sels=("sparse",))


# ---- PAD behaviour ------------------------------------------------------------------------------------------------------
def test_pad_collation_cuts_only_0x20():
    kept = [b"\t", b"\x00", b"\xa0", "　".encode(), b"\xc2\xa0"]
    rows = [b"a", b"a ", b"a   ", b"", b" ", b"   "] + [b"a" + k for k in kept] + [b"a" + k + b" " for k in kept] + \
           [b"a " + k for k in kept] + [b"b", b"a\x1f", b"a!"]
    rows = rows * 3
    for coll in (46, 83, 65, 47, 63, 309):
        for k in (b"a", b"a ", b"a    ", b"", b"  ", b"a\t", b"a\t  ", "a　".encode(), b"a\x00 "):
            for op in (LT, EQ, GT):
                run_item(CMP, rows, const=k, op=op, coll=coll, shifts=(1,), sels=("all",))
        run_item(CMP, rows, b_rows=rows[::-1], op=EQ, coll=coll, sels=())
    exp = np.array([P.compare(r, b"a", 46) == 0 for r in rows])
    assert exp[:3].all() and not exp[6:11].any()   # "a ", "a   " equal "a"; tab, NUL, NBSP, U+3000 are kept
    # LIKE does not cut
    for coll in (46, 309):
        m = run_item(LIKE, rows, const=b"a", coll=coll)
        assert m[0] and not m[1] and not m[2]
        run_item(LIKE, rows, const=b"a_", coll=coll)
        run_item(LIKE, rows, const=b"a ", coll=coll)


# ---- sel shapes ---------------------------------------------------------------------------------------------------------
def test_sel_shapes():
    rng = np.random.default_rng(4)
    rows, _ = aligned_tiles(rng, 700)
    n = len(rows)
    nl = rng.random(n) < 0.1
    a = column(rows, nl, lead=6)
    for it in (FilterItem(EQ, 0, is_string=True, str_kind=LIKE, const_bytes=b"%a%", collation=46),
               FilterItem(GT, 0, is_string=True, const_bytes=b"b", collation=63)):
        m = expected(it.str_kind, rows, const=it.const_bytes, op=it.op, coll=it.collation) & ~nl
        for sel in (np.zeros(0, np.int64), np.array([n - 1], np.int64), np.arange(n, dtype=np.int64),
                    np.sort(rng.choice(n, 37, replace=False)).astype(np.int64), np.arange(n - 1, -1, -1, dtype=np.int64)):
            for dev in ((False, True) if len(sel) else (False,)):
                rc, got, cnt = call_filter([a], [VC], [it], sel, dev, shift=13)
                assert rc == 0, abi.load_lib().tg_last_error()
                w = np.zeros(n, np.uint8)
                w[sel] = m[sel]
                # rows outside sel get 0: `selected` is cleared for every physical row before the items run
                assert np.array_equal(got, w), (len(sel), dev)
                assert cnt == int(w.sum())
        # an empty sel of device rows: a valid pointer with nsel 0 (a NULL sel pointer means "no sel")
        import torch
        from test_gpu_vec_string import Dev
        from tidb_b200.chunk import Chunk
        from tidb_b200.plan import filter_array, str_arg_array
        dv = Dev()
        chk = Chunk([a])
        cs = chk.to_struct()
        cs.cols[0] = dv.col(a, 13)
        one = torch.zeros(1, dtype=torch.int64, device="cuda")
        cs.sel, cs.nsel = one.data_ptr(), 0
        out = torch.full((n,), 7, dtype=torch.uint8, device="cuda")
        cnt = C.c_int64(-1)
        tps = (C.c_int32 * 1)(VC)
        lib = abi.load_lib()
        assert lib.tg_vec_filter_ex2(0, 1, C.byref(cs), tps, filter_array([it]), 1, None, str_arg_array([it]),
                                     C.c_void_p(out.data_ptr()), C.byref(cnt), None) == 0, lib.tg_last_error()
        torch.cuda.synchronize()
        assert cnt.value == 0 and int(out.sum()) == 0


# ---- a CNF that reuses the staging buffers -----------------------------------------------------------------------------
def test_cnf_reuses_staging_buffers():
    rng = np.random.default_rng(12)
    rows_a, _ = aligned_tiles(rng, 1900)
    n = len(rows_a)
    rows_b = [r if i % 3 else r[::-1] for i, r in enumerate(rows_a)]
    rows_c = tile_rows(rng, 900) * (n // 32)
    na, nb_, nc = rng.random(n) < 0.05, rng.random(n) < 0.05, rng.random(n) < 0.05
    iv = rng.integers(-10, 10, n).astype(np.int64)
    rv = np.floor(rng.random(n) * 100) / 10
    dv = rng.integers(-500, 500, n)
    cells = np.frombuffer(b"".join(A.cell(int(v), 15, 2) for v in dv), np.uint8).reshape(n, 40).copy()
    cols = [column(rows_a, na, 2), column(rows_b, nb_, 9), Column(iv), column(rows_c, nc, 0), Column(rv), Column(cells)]
    types = [VC, abi.TYPE_BLOB, L, abi.TYPE_STRING, DBL, DEC]
    s = lambda op, l, r=-1, **kw: FilterItem(op, l, r, is_string=True, **kw)
    cnfs = [
        [s(LE, 0, 0, collation=46), s(NE, 0, 1, collation=63), s(EQ, 3, str_kind=NOT_LIKE, const_bytes=b"%\xff\xff\xff%", collation=309),
         s(NE, 1, 3, collation=46), s(EQ, 0, str_kind=LIKE, const_bytes=b"%", collation=46), s(EQ, 3, 3, collation=309),
         s(EQ, 1, str_kind=NOT_LIKE, const_bytes=b"%b_y%", collation=46), s(LT, 3, 0, collation=63)],
        [s(EQ, 0, 0, collation=63), FilterItem(GT, 2, const_i64=-8), s(EQ, 1, str_kind=NOT_LIKE, const_bytes="%é%".encode(), collation=46),
         FilterItem(GE, 5, is_decimal=True, const_cell=A.cell(-400, 15, 2)), s(NE, 3, 1, collation=46),
         FilterItem(LE, 4, is_real=True, const_f64=9.5), s(EQ, 3, str_kind=LIKE, const_bytes=b"%_%", collation=309),
         s(GE, 0, 1, collation=309)],
    ]
    strs = {0: (rows_a, na), 1: (rows_b, nb_), 3: (rows_c, nc)}
    for items in cnfs:
        want = np.ones(n, bool)
        for it in items:
            if it.is_string:
                xa, xn = strs[it.lhs_col]
                if it.str_kind == CMP and it.rhs_col >= 0:
                    ya, yn = strs[it.rhs_col]
                    want &= expected(CMP, xa, ya, op=it.op, coll=it.collation) & ~xn & ~yn
                else:
                    want &= expected(it.str_kind, xa, const=it.const_bytes, op=it.op, coll=it.collation) & ~xn
            elif it.is_decimal:
                want &= apply_cmp(it.op, np.sign(dv + 400))
            elif it.is_real:
                want &= apply_cmp(it.op, np.sign(rv - 9.5))
            else:
                want &= apply_cmp(it.op, np.sign(iv + 8))
        assert 0 < want.sum() < n
        for sel in (None, np.sort(rng.choice(n, n // 2, replace=False)).astype(np.int64)):
            for dev in (False, True):
                rc, got, cnt = call_filter(cols, types, items, sel, dev, shift=7)
                assert rc == 0, abi.load_lib().tg_last_error()
                w = np.zeros(n, np.uint8)
                r = np.arange(n) if sel is None else sel
                w[r] = want[r]
                assert np.array_equal(got, w), (sel is None, dev, np.flatnonzero(got != w)[:8])
                assert cnt == int(w.sum())


# ---- size: a device column past 2^31 bytes -----------------------------------------------------------------------------
def test_device_column_past_2_31_bytes():
    import torch
    from test_gpu_vec_string import GUARD
    lib = abi.load_lib()
    body, nbig = 1000, 2_150_000
    tail_rows = tile_rows(np.random.default_rng(31), 1500) + [b"x" * 37 + "é".encode() + b"b", b"tail" + b"\xe2\x82", b"b"] + \
        tile_rows(np.random.default_rng(32), 300)
    assert nbig * body > (1 << 31)
    n = nbig + len(tail_rows)
    base_row = (b"ab" * 250 + "é".encode() * 100 + b"\xe2\x82\xac" * 100)[:body]
    assert len(base_row) == body
    total = nbig * body + sum(len(r) for r in tail_rows)
    data = torch.empty(total + 16, dtype=torch.uint8, device="cuda")
    data[:nbig * body].view(nbig, body).copy_(torch.frombuffer(bytearray(base_row), dtype=torch.uint8).cuda().expand(nbig, body))
    tb = b"".join(tail_rows)
    data[nbig * body:total] = torch.frombuffer(bytearray(tb), dtype=torch.uint8).cuda()
    lens = torch.tensor([len(r) for r in tail_rows], dtype=torch.int64)
    offs = torch.empty(n + 1, dtype=torch.int64, device="cuda")
    offs[:nbig + 1] = torch.arange(nbig + 1, dtype=torch.int64, device="cuda") * body
    offs[nbig + 1:] = (nbig * body + torch.cumsum(lens, 0)).cuda()
    assert int(offs[-1]) == total and int(offs[nbig]) > (1 << 31)
    col = abi.TgColumn()
    col.length, col.null_bitmap, col.offsets, col.data, col.elem_len = n, None, offs.data_ptr(), data.data_ptr(), -1
    res = torch.full((n,), 0x5A, dtype=torch.int64, device="cuda")
    bm = torch.full(((n + 7) // 8 + GUARD,), 0xA5, dtype=torch.uint8, device="cuda")
    tail_at = nbig
    for pat, coll in ((b"%b", 46), ("%é_".encode(), 309), (b"ab%\xe2\x82\xac", 46), (b"tail__", 46), (b"tail_", 63), (b"%", 63)):
        pb = (C.c_uint8 * len(pat)).from_buffer_copy(pat)
        assert lib.tg_vec_like(0, 1, coll, C.byref(col), pb, C.c_int64(len(pat)), BS, C.c_void_p(res.data_ptr()),
                               C.c_void_p(bm.data_ptr()), None) == 0, lib.tg_last_error()
        torch.cuda.synchronize()
        got = res.cpu().numpy()
        body_m = P.like(base_row, pat, BS, coll)
        assert (got[:tail_at] == int(body_m)).all(), pat
        exp_tail = [P.like(r, pat, BS, coll) for r in tail_rows]
        assert got[tail_at:].tolist() == [int(x) for x in exp_tail], pat
    k = tail_rows[32]
    kb = (C.c_uint8 * len(k)).from_buffer_copy(k)
    for op in (LT, EQ, GT):
        assert lib.tg_vec_compare_string(0, 1, op, 46, C.byref(col), None, kb, C.c_int64(len(k)), C.c_void_p(res.data_ptr()),
                                         C.c_void_p(bm.data_ptr()), None) == 0, lib.tg_last_error()
        torch.cuda.synchronize()
        got = res.cpu().numpy()
        assert (got[:tail_at] == int(apply_cmp(op, P.compare(base_row, k, 46)))).all()
        assert got[tail_at:].tolist() == [int(apply_cmp(op, P.compare(r, k, 46))) for r in tail_rows]
    # the sel path over the rows at the top of the range
    sel = torch.arange(n - 70, n, dtype=torch.int64, device="cuda")
    chk = abi.TgChunk()
    arr = (abi.TgColumn * 1)(col)
    chk.ncols, chk.cols, chk.sel, chk.nsel = 1, C.cast(arr, C.POINTER(abi.TgColumn)), sel.data_ptr(), 70
    out = torch.full((n,), 7, dtype=torch.uint8, device="cuda")
    cnt = C.c_int64(-1)
    from tidb_b200.plan import filter_array, str_arg_array
    items = [FilterItem(EQ, 0, is_string=True, str_kind=LIKE, const_bytes=b"%b", collation=46)]
    tps = (C.c_int32 * 1)(VC)
    assert lib.tg_vec_filter_ex2(0, 1, C.byref(chk), tps, filter_array(items), 1, None, str_arg_array(items),
                                 C.c_void_p(out.data_ptr()), C.byref(cnt), None) == 0, lib.tg_last_error()
    torch.cuda.synchronize()
    got = out[n - 70:].cpu().numpy()
    all_rows = [base_row] * (70 - len(tail_rows)) + tail_rows
    assert got.tolist() == [int(P.like(r, b"%b", BS, 46)) for r in all_rows]
    assert cnt.value == int(got.sum()) and int(out[:n - 70].sum()) == 0
    del data, offs, res, out
    torch.cuda.empty_cache()
