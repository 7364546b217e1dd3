"""The DECIMAL VecEval calls (csrc/vec.cu: tg_vec_compare_decimal, tg_vec_filter_ex) and the SelectionExec /
ProjectionExec shims over 40-byte MyDecimal cells, against the reference order of tests/topn_decimal.py (cmp_decimal,
pinned to TestCompareMyDecimal by tests/test_topn_decimal_reference.py).

Rows are drawn from a pool of cells: the TopN reference's hand cases (negative zeros, leading zero words, trailing zero
fraction words, 9-word cells, resultFrac and unused-word garbage, equal values in different forms), DECIMAL(15,2) cells in
FromBin's forms, and random cells of every scale up to 30 with their re-encodings.  The pool is ranked once with
cmp_decimal, so a row's expected comparison is the comparison of its cells' ranks.  Results are checked bit for bit:
0/1 values (0 under NULL), NULL bitmaps, `selected` bytes and counts."""
import ctypes as C
import functools
from fractions import Fraction

import numpy as np
import pytest

import mydecimal as D
import mydecimal_args as A
import test_gpu_vec_exact as VE
import test_topn_decimal_reference as TR
import topn_decimal as TD
import vec_reference as R
from tidb_b200 import abi
from tidb_b200.chunk import Chunk, Column
from tidb_b200.executor import HashAggExec, MockDataSource, ProjectionExec, SelectionExec, drain
from tidb_b200.plan import AggFunc, AggPlan, ColRef, Const, FieldType, FilterItem, ScalarFunc, dec_const_array, filter_array

pytestmark = pytest.mark.gpu
CMP_OPS = [abi.CMP_LT, abi.CMP_LE, abi.CMP_GT, abi.CMP_GE, abi.CMP_EQ, abi.CMP_NE]
SIZES = [1, 31, 33, 1061, 70_001, 4_200_001]
BIG = 4_200_001
GUARD = 8
L, DBL, DATE, DEC = abi.TYPE_LONGLONG, abi.TYPE_DOUBLE, abi.TYPE_DATE, abi.TYPE_NEWDECIMAL
D152 = FieldType(DEC, 0, 15, 2)
INT = FieldType(L, 0)


# ---- the cell pool ---------------------------------------------------------------------------------------------------
def _random_literal(rng):
    ip = "".join(rng.choice(list("0123456789"), int(rng.integers(0, 21))))
    fp = "".join(rng.choice(list("0123456789"), int(rng.integers(0, 31))))
    return ("-" if rng.random() < 0.4 else "") + (ip or "0") + ("." + fp if fp else "")


def _build_pool(seed=5):
    rng = np.random.default_rng(seed)
    cells = [c for cls in TR.ORDERED_CLASSES for c in cls]
    for _ in range(300):                                     # DECIMAL(15,2) as FromBin stores it, and its variants
        v = int(rng.integers(-10 ** 15 + 1, 10 ** 15))
        di = int(rng.choice([13, 27] + ([0] if abs(v) < 100 else [])))
        cells.append(A.cell(v, 15, 2, digits_int=di, result_frac=int(rng.integers(0, 31)), neg_zero=v == 0 and rng.random() < 0.5))
    for v in (0, 5, 7, 24 * 100, -5, 30000):                # values the constants below sit on
        cells += [A.cell(v, 15, 2), A.cell(v, 15, 2, digits_int=0 if abs(v) < 100 else 27, result_frac=9)]
    for _ in range(250):                                     # any scale up to 30, re-encoded with extra words
        s = _random_literal(rng)
        ip, _, fp = s.lstrip("-").partition(".")
        cells.append(TR.dec(s, result_frac=int(rng.integers(0, 128)), tail=(int(rng.integers(-2 ** 31, 2 ** 31)),)))
        di = len(ip.lstrip("0")) + 9
        if (di + 8) // 9 + (len(fp) + 9 + 8) // 9 <= 9:
            cells.append(TR.dec(s, digits_int=di, frac=len(fp) + 9))
    for _ in range(60):                                      # 9-word cells of every split
        wi = int(rng.integers(0, 10))
        words = [int(w) for w in rng.integers(0, 10 ** 9, 9)]
        cells.append(TR.raw(9 * wi - int(rng.integers(0, 9)) if wi else 0, 9 * (9 - wi), int(rng.random() < 0.5), words, rf=int(rng.integers(0, 31))))
    order = sorted(range(len(cells)), key=functools.cmp_to_key(lambda i, j: TD.cmp_decimal(cells[i], cells[j])))
    rank = np.zeros(len(cells), np.int64)
    for x in range(1, len(order)):
        rank[order[x]] = rank[order[x - 1]] + (TD.cmp_decimal(cells[order[x - 1]], cells[order[x]]) != 0)
    return np.frombuffer(b"".join(cells), np.uint8).reshape(len(cells), 40).copy(), rank


@pytest.fixture(scope="module")
def pool():
    return _build_pool()


def _const_ids(pool_rank, rng, k):
    return [int(x) for x in rng.choice(len(pool_rank), k, replace=False)]


def _malformed(rng, k):
    """k garbage cells that dec_cell_ok rejects"""
    g = rng.integers(0, 256, (k, 40), dtype=np.uint8)
    g[:, 0] = 0x90                                          # digitsInt -112
    return g


class Rows:
    """n rows of two DECIMAL operands drawn from the pool, ~10% NULL on each side, garbage (often malformed) under NULL"""

    def __init__(self, pool, n, seed):
        cells, rank = pool
        rng = np.random.default_rng(seed)
        self.ia, self.ib = rng.integers(0, len(rank), n), rng.integers(0, len(rank), n)
        self.a, self.b = cells[self.ia], cells[self.ib]
        self.an, self.bn = rng.random(n) < 0.1, rng.random(n) < 0.1
        self.a[self.an] = _malformed(rng, int(self.an.sum()))
        self.b[self.bn] = rng.integers(0, 256, (int(self.bn.sum()), 40), dtype=np.uint8)
        self.ra, self.rb = rank[self.ia], rank[self.ib]


def _col(v, nl):
    return Column(v, nl if nl is not None and nl.any() else None)


def _bitmap(nulls):
    return np.packbits(~np.asarray(nulls, bool), bitorder="little")


def _expect(op, ra, an, rb, bn):
    valid = ~an if bn is None else ~(an | bn)
    c = np.sign(ra - rb)
    return (R.holds_vec(op, c) & valid).astype(np.int64), _bitmap(~valid)


def call_compare(op, a, an, b, bn, cell, on_device=False):
    """-> (status, result values, result bitmap bytes); host outputs start as sentinels"""
    import torch
    lib = abi.load_lib()
    n = len(a)
    ca, cb = _col(a, an), (None if b is None else _col(b, bn))
    sa = ca.to_struct(); sb = None if cb is None else cb.to_struct()
    keep = []
    if on_device:
        for s, c in ((sa, ca), (sb, cb)):
            if s is None:
                continue
            d = torch.from_numpy(c.data).cuda(); keep.append(d); s.data = d.data_ptr()
            if c.null_bitmap is not None:
                m = torch.from_numpy(c.null_bitmap.copy()).cuda(); keep.append(m); s.null_bitmap = m.data_ptr()
        res_t = torch.full((n,), 0x5A5A5A5A, dtype=torch.int64, device="cuda")
        bm_t = torch.full(((n + 7) // 8 + GUARD,), 0xA5, dtype=torch.uint8, device="cuda")
        rp, bp = C.c_void_p(res_t.data_ptr()), C.c_void_p(bm_t.data_ptr())
    else:
        res = np.full(n, 0x5A5A5A5A, np.int64)
        bm = np.full((n + 7) // 8, 0xA5, np.uint8)
        rp, bp = res.ctypes.data_as(C.c_void_p), bm.ctypes.data_as(C.c_void_p)
    k = None if cell is None else (C.c_uint8 * 40).from_buffer_copy(bytes(cell))
    rc = lib.tg_vec_compare_decimal(0, int(on_device), op, C.byref(sa), None if sb is None else C.byref(sb), k, rp, bp, None)
    if on_device:
        torch.cuda.synchronize()
        res, bm = res_t.cpu().numpy(), bm_t.cpu().numpy()
        assert (bm[(n + 7) // 8:] == 0xA5).all(), "the result bitmap was written past its last byte"
    return rc, res, bm[:(n + 7) // 8]


# ---- tg_vec_compare_decimal ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", SIZES)
def test_compare_decimal_exact(pool, n):
    cells, rank = pool
    rows = Rows(pool, n, seed=n)
    rng = np.random.default_rng(n + 1)
    consts = _const_ids(rank, rng, 2 if n >= BIG else 6) + [0]
    for on_device in (False, True):
        for op in CMP_OPS:
            for rhs in [None] + consts:
                if rhs is None:
                    exp, ebm = _expect(op, rows.ra, rows.an, rows.rb, rows.bn)
                    rc, res, bm = call_compare(op, rows.a, rows.an, rows.b, rows.bn, None, on_device)
                else:
                    exp, ebm = _expect(op, rows.ra, rows.an, rank[rhs], None)
                    rc, res, bm = call_compare(op, rows.a, rows.an, None, None, cells[rhs], on_device)
                what = (op, rhs, on_device)
                assert rc == abi.TG_OK, (what, abi.load_lib().tg_last_error())
                bad = np.flatnonzero(res != exp)
                assert len(bad) == 0, (what, bad[:5])
                assert np.array_equal(bm, ebm), what


def test_compare_decimal_every_pool_pair(pool):
    # every ordered pair of pool cells, once against each other as columns and once as column against constant
    cells, rank = pool
    p = len(rank)
    ia, ib = np.repeat(np.arange(p), p), np.tile(np.arange(p), p)
    z = np.zeros(len(ia), bool)
    for op in (abi.CMP_LT, abi.CMP_EQ):
        exp, _ = _expect(op, rank[ia], z, rank[ib], z)
        rc, res, _ = call_compare(op, cells[ia], z, cells[ib], z, None)
        assert rc == abi.TG_OK and np.array_equal(res, exp), op
    for j in range(0, p, 7):
        exp, _ = _expect(abi.CMP_LE, rank, np.zeros(p, bool), rank[j], None)
        rc, res, _ = call_compare(abi.CMP_LE, cells, np.zeros(p, bool), None, None, cells[j])
        assert rc == abi.TG_OK and np.array_equal(res, exp), j


# ---- tg_vec_filter_ex ------------------------------------------------------------------------------------------------
def call_filter_ex(cols, types, items, sel=None, on_device=False, out=None):
    """cols[c] = (values or (n, 40) cells, NULL flags) -> (status, selected bytes, count); `out` (host) is reused when given"""
    import torch
    lib = abi.load_lib()
    chk = Chunk([_col(v, nl) for v, nl in cols], sel)
    cs = chk.to_struct()
    n = len(cols[0][0])
    keep = []
    if on_device:
        for i, c in enumerate(chk.columns):
            d = torch.from_numpy(np.ascontiguousarray(c.data).view(np.uint8).reshape(-1)).cuda(); keep.append(d); cs.cols[i].data = d.data_ptr()
            if c.null_bitmap is not None:
                m = torch.from_numpy(c.null_bitmap.copy()).cuda(); keep.append(m); cs.cols[i].null_bitmap = m.data_ptr()
        if sel is not None:
            s = torch.from_numpy(chk.sel.copy()).cuda(); keep.append(s); cs.sel = s.data_ptr()
        out_t = torch.full((max(n, 1),), 7, dtype=torch.uint8, device="cuda")
        out_p = C.c_void_p(out_t.data_ptr())
    else:
        out = np.full(max(n, 1), 7, np.uint8) if out is None else out
        out_p = out.ctypes.data_as(C.c_void_p)
    cnt = C.c_int64(-1)
    tps = (C.c_int32 * len(types))(*types)
    rc = lib.tg_vec_filter_ex(0, int(on_device), C.byref(cs), tps, filter_array(items), len(items), dec_const_array(items),
                              out_p, C.byref(cnt), None)
    if on_device:
        torch.cuda.synchronize()
        out = out_t.cpu().numpy()
    return rc, out[:n], cnt.value


def filter_reference(cols, ranks, items, sel=None):
    """R.filter_rows for the INT / REAL items, AND the DECIMAL items by rank (ranks[c]: the pool rank of each row's cell
    in DECIMAL column c; item.rank: the constant's rank)"""
    n = len(cols[0][0])
    plain = [it for it in items if not it.is_decimal]
    ok = R.filter_rows(cols, plain) if plain else np.ones(n, bool)
    for it in items:
        if not it.is_decimal:
            continue
        ln = cols[it.lhs_col][1]
        rn = cols[it.rhs_col][1] if it.rhs_col >= 0 else np.zeros(n, bool)
        rb = ranks[it.rhs_col] if it.rhs_col >= 0 else it.rank
        ok &= ~ln & ~rn & R.holds_vec(it.op, np.sign(ranks[it.lhs_col] - rb))
    if sel is not None:
        keep = np.zeros(n, bool)
        keep[sel] = True
        ok &= keep
    return ok


def _dec_item(op, lhs, pool, cid=None, rhs=-1):
    it = FilterItem(op, lhs, rhs_col=rhs, is_decimal=True, const_cell=None if cid is None else bytes(pool[0][cid]))
    it.rank = None if cid is None else pool[1][cid]
    return it


def _mixed_table(pool, n, seed):
    """0 int, 1 int, 2 double, 3 DATE (packed words, unsigned), 4-6 DECIMAL cells (6 without NULLs)"""
    cells, rank = pool
    rng = np.random.default_rng(seed)
    ids = [rng.integers(0, len(rank), n) for _ in range(3)]
    nulls = [rng.random(n) < 0.1, rng.random(n) < 0.1, np.zeros(n, bool)]
    cols = [(rng.integers(-1000, 1000, n).astype(np.int64), rng.random(n) < 0.1),
            (rng.integers(R.INT64_MIN, R.INT64_MAX, n, dtype=np.int64), np.zeros(n, bool)),
            (np.round(rng.normal(0, 100, n), 2), rng.random(n) < 0.1),
            (rng.integers(0, 1 << 50, n).astype(np.int64) << 4, rng.random(n) < 0.05)]
    ranks = {}
    for c in range(3):
        v = cells[ids[c]]
        v[nulls[c]] = _malformed(rng, int(nulls[c].sum()))
        cols.append((v, nulls[c]))
        ranks[4 + c] = rank[ids[c]]
    return cols, [L, L, DBL, DATE, DEC, DEC, DEC], ranks


def _item_sets(pool, seed):
    rng = np.random.default_rng(seed)
    k = _const_ids(pool[1], rng, 8)
    return [
        [_dec_item(abi.CMP_GE, 4, pool, k[0])],
        [_dec_item(abi.CMP_LT, 4, pool, rhs=5)],
        [_dec_item(abi.CMP_EQ, 6, pool, k[1]), _dec_item(abi.CMP_NE, 5, pool, k[1])],
        [_dec_item(abi.CMP_GE, 6, pool, k[2]), _dec_item(abi.CMP_LE, 6, pool, k[3])],          # BETWEEN
        [FilterItem(abi.CMP_GT, 0, const_i64=-300), _dec_item(abi.CMP_LE, 4, pool, rhs=6), FilterItem(abi.CMP_GE, 2, is_real=True, const_f64=-0.0),
         FilterItem(abi.CMP_GE, 3, const_i64=1 << 50, lhs_unsigned=True, rhs_unsigned=True), FilterItem(abi.CMP_LT, 3, const_i64=3 << 51, lhs_unsigned=True, rhs_unsigned=True)],
        [FilterItem(abi.CMP_NE, 0, rhs_col=1), _dec_item(abi.CMP_GT, 5, pool, k[4]), _dec_item(abi.CMP_NE, 4, pool, rhs=5),
         FilterItem(abi.CMP_LT, 2, is_real=True, const_f64=150.0), _dec_item(abi.CMP_LE, 6, pool, k[5]), FilterItem(abi.CMP_GT, 3, const_i64=1 << 40, lhs_unsigned=True, rhs_unsigned=True),
         _dec_item(abi.CMP_GE, 6, pool, rhs=4), FilterItem(abi.CMP_LE, 1, const_i64=R.INT64_MAX // 2)],
    ]


@pytest.mark.parametrize("n", [1, 33, 1061, 70_001, 1_000_003])
def test_filter_ex_mixed_cnf(pool, n):
    cols, types, ranks = _mixed_table(pool, n, seed=n)
    rng = np.random.default_rng(n + 2)
    sel = np.sort(rng.choice(n, max(1, n // 2), replace=False)).astype(np.int64)
    # DECIMAL rows outside sel hold malformed cells: only the rows the call evaluates are read
    out_sel = np.ones(n, bool); out_sel[sel] = False
    sel_cols = [(v.copy(), nl) for v, nl in cols]
    for c in (4, 5, 6):
        sel_cols[c][0][out_sel] = _malformed(rng, int(out_sel.sum()))
    for items in _item_sets(pool, n):
        for s, cs in ((None, cols), (sel, sel_cols)):
            exp = filter_reference(cs, ranks, items, s)
            for on_device in (False, True):
                rc, got, cnt = call_filter_ex(cs, types, items, s, on_device)
                assert rc == abi.TG_OK, (len(items), s is not None, on_device, abi.load_lib().tg_last_error())
                assert np.array_equal(got, exp.astype(np.uint8)) and cnt == int(exp.sum()), (len(items), s is not None, on_device)


@pytest.mark.parametrize("n", [1061, 70_001])
def test_filter_ex_equals_vec_filter_without_decimal_items(n):
    # the tg_vec_filter fixtures of test_gpu_vec_exact.py, unchanged: the same `selected` and count
    rng = np.random.default_rng(1)
    pools = VE._int_pool(rng), VE._real_pool(rng)
    cols = VE._filter_table(pools, n)
    sel = np.sort(np.random.default_rng(n).choice(n, n // 2, replace=False)).astype(np.int64)
    types = [L, L, L, DBL, DBL]
    for items in VE.FILTER_SETS:
        for s in (None, sel):
            for on_device in (False, True):
                rc0, want, c0 = VE.call_filter(cols, items, s, on_device)
                rc, got, cnt = call_filter_ex(cols, types, items, s, on_device)
                assert rc == rc0 == abi.TG_OK and np.array_equal(got, want) and cnt == c0, (items, s is not None, on_device)


# ---- malformed cells -------------------------------------------------------------------------------------------------
def test_malformed_cell_fails_and_writes_nothing(pool):
    cells, rank = pool
    n, pos = 1_000_000, 777_777
    rows = Rows(pool, n, seed=3)
    a, an, b, bn = rows.a.copy(), rows.an.copy(), rows.b.copy(), rows.bn.copy()
    an[pos] = bn[pos] = False
    a[pos], b[pos] = cells[rows.ia[pos]], cells[rows.ib[pos]]
    good_a = a[pos].copy()
    a[pos] = _malformed(np.random.default_rng(0), 1)[0]
    lib = abi.load_lib()
    k = (C.c_uint8 * 40).from_buffer_copy(bytes(cells[3]))
    # host buffers: sentinels stay untouched; then the same buffers take the next valid call
    ca, cb = _col(a, an), _col(b, bn)
    sa, sb = ca.to_struct(), cb.to_struct()
    res, bm = np.full(n, 0x5A5A5A5A, np.int64), np.full((n + 7) // 8, 0xA5, np.uint8)
    for pb, kk in ((None, k), (C.byref(sb), None)):
        rc = lib.tg_vec_compare_decimal(0, 0, abi.CMP_LT, C.byref(sa), pb, kk, res.ctypes.data_as(C.c_void_p), bm.ctypes.data_as(C.c_void_p), None)
        assert rc == abi.TG_ERR_INVALID
        assert (res == 0x5A5A5A5A).all() and (bm == 0xA5).all()
    # the bad cell on the right, with the left NULL at that row: still checked
    bn2 = bn.copy(); bn2[pos] = True
    assert call_compare(abi.CMP_GE, b, bn2, a, an, None)[0] == abi.TG_ERR_INVALID
    assert call_compare(abi.CMP_GE, a, an, None, None, cells[3], on_device=True)[0] == abi.TG_ERR_INVALID
    # filter: an INT item false on every row does not spare the DECIMAL cells from the check
    cols = [(np.zeros(n, np.int64), np.zeros(n, bool)), (a, an), (b, bn)]
    types = [L, DEC, DEC]
    never = FilterItem(abi.CMP_GT, 0, const_i64=5)
    for items in ([never, _dec_item(abi.CMP_LT, 1, pool, 3)], [_dec_item(abi.CMP_GE, 2, pool, rhs=1), never]):
        sel_out = np.full(n, 9, np.uint8)
        rc, got, cnt = call_filter_ex(cols, types, items, out=sel_out)
        assert rc == abi.TG_ERR_INVALID and (sel_out == 9).all() and cnt == -1
        assert call_filter_ex(cols, types, items, on_device=True)[0] == abi.TG_ERR_INVALID
        # under a sel vector that holds the row
        assert call_filter_ex(cols, types, items, sel=np.array([5, pos, n - 1], np.int64))[0] == abi.TG_ERR_INVALID
    # a bad cell under NULL or outside sel is never read
    an3 = an.copy(); an3[pos] = True
    exp, ebm = _expect(abi.CMP_LT, rows.ra, an3, rank[3], None)
    rc, r3, b3 = call_compare(abi.CMP_LT, a, an3, None, None, cells[3])
    assert rc == abi.TG_OK and np.array_equal(r3, exp) and np.array_equal(b3, ebm)
    sel = np.array([i for i in range(0, n, 1000) if i != pos], np.int64)
    items = [_dec_item(abi.CMP_LT, 1, pool, 3)]
    ranks = {1: rows.ra, 2: rows.rb}
    rc, got, cnt = call_filter_ex(cols, types, items, sel=sel)
    exp = filter_reference(cols, ranks, items, sel)
    assert rc == abi.TG_OK and np.array_equal(got, exp.astype(np.uint8)) and cnt == int(exp.sum())
    # the cell repaired: the next valid calls on the same host buffers succeed
    a[pos] = good_a
    ca = _col(a, an)                                        # keeps the packed bitmap alive for the call
    sa = ca.to_struct()
    rc = lib.tg_vec_compare_decimal(0, 0, abi.CMP_LT, C.byref(sa), None, k, res.ctypes.data_as(C.c_void_p), bm.ctypes.data_as(C.c_void_p), None)
    exp, ebm = _expect(abi.CMP_LT, rows.ra, an, rank[3], None)
    assert rc == abi.TG_OK and np.array_equal(res, exp) and np.array_equal(bm, ebm)
    sel_out = np.full(n, 9, np.uint8)
    items = [_dec_item(abi.CMP_GE, 2, pool, rhs=1)]
    rc, got, cnt = call_filter_ex(cols, types, items, out=sel_out)
    exp = filter_reference(cols, ranks, items)
    assert rc == abi.TG_OK and np.array_equal(got, exp.astype(np.uint8)) and cnt == int(exp.sum())


# ---- executors -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("required_rows", [1, 7, 1024])
def test_selection_and_projection_over_decimal_sel_vectors(pool, required_rows):
    cells, rank = pool
    rng = np.random.default_rng(40 + required_rows)
    n = 5000
    ia, ib = rng.integers(0, len(rank), n), rng.integers(0, len(rank), n)
    an, bn = rng.random(n) < 0.1, rng.random(n) < 0.1
    a, b = cells[ia], cells[ib]
    a[an] = _malformed(rng, int(an.sum()))
    cols = [(rng.integers(-1000, 1000, n).astype(np.int64), rng.random(n) < 0.1), (a, an), (b, bn)]
    schema = [INT, FieldType(DEC, 0, 65, 30), FieldType(DEC, 0, 65, 30)]
    chunks, logical = VE._sel_chunks(rng, cols)
    lcols = [(v[logical], nl[logical]) for v, nl in cols]
    ranks = {1: rank[ia][logical], 2: rank[ib][logical]}
    kid = int(rng.integers(0, len(rank)))
    filters = [FilterItem(abi.CMP_GT, 0, const_i64=-500), _dec_item(abi.CMP_GE, 1, pool, kid), _dec_item(abi.CMP_NE, 1, pool, rhs=2)]
    keep = filter_reference(lcols, ranks, filters)
    e = SelectionExec(MockDataSource(schema, chunks), filters, batch_rows=2048)
    for _ in range(2):                                       # Open again after Close re-executes
        out = drain(e, required_rows)
        assert all(0 < c.num_rows() <= required_rows for c in out)
        vals, nulls = VE._collect(out, 3)
        for c in range(3):
            assert np.array_equal(nulls[c], lcols[c][1][keep]), c
            assert np.array_equal(vals[c][~nulls[c]], lcols[c][0][keep][~lcols[c][1][keep]]), c
    exprs = [ColRef(1), ScalarFunc("cmp", abi.CMP_LE, (ColRef(1), Const(cell=bytes(cells[kid]))), is_decimal=True),
             ScalarFunc("cmp", abi.CMP_GT, (ColRef(2), ColRef(1)), is_decimal=True), ColRef(0)]
    e = ProjectionExec(MockDataSource(schema, chunks), exprs, batch_rows=2048)
    assert [t.tp for t in e.schema] == [DEC, L, L, L]
    (av, an_), (bv, bn_) = lcols[1], lcols[2]
    le, _ = _expect(abi.CMP_LE, ranks[1], an_, rank[kid], None)
    gt, _ = _expect(abi.CMP_GT, ranks[2], bn_, ranks[1], an_)
    for _ in range(2):
        out = drain(e, required_rows)
        assert all(0 < c.num_rows() <= required_rows for c in out)
        vals, nulls = VE._collect(out, 4)
        assert np.array_equal(nulls[0], an_) and np.array_equal(vals[0][~an_], av[~an_])
        assert np.array_equal(vals[1], le) and np.array_equal(nulls[1], an_)
        assert np.array_equal(vals[2], gt) and np.array_equal(nulls[2], an_ | bn_)
        assert np.array_equal(nulls[3], lcols[0][1]) and np.array_equal(vals[3][~nulls[3]], lcols[0][0][~lcols[0][1]])


# ---- Q6 and Q18 shapes -----------------------------------------------------------------------------------------------
def _d152(scaled, rng):
    """DECIMAL(15,2) cells in FromBin's form (digitsInt 13), some with digitsInt 0 / 27 and resultFrac garbage"""
    n = len(scaled)
    di = np.where(rng.random(n) < 0.2, 27, 13).astype(np.int64)
    di[(np.abs(scaled) < 100) & (rng.random(n) < 0.5)] = 0
    return A.cells_np(scaled.astype(np.int64), 15, 2, di, rng.integers(0, 31, n), scaled < 0)


def test_q6_shape_end_to_end():
    # SELECT sum(l_extendedprice * l_discount) FROM lineitem WHERE l_shipdate >= d0 AND l_shipdate < d1
    #   AND l_discount BETWEEN 0.05 AND 0.07 AND l_quantity < 24
    rng = np.random.default_rng(6)
    n = 300_000
    ship = rng.integers(8000, 10600, n).astype(np.int64)
    disc = rng.integers(0, 11, n).astype(np.int64)                  # 0.00 .. 0.10
    qty = rng.integers(100, 5001, n).astype(np.int64)               # 1.00 .. 50.00
    qty[::3] = rng.integers(1, 50, len(qty[::3])) * 100             # whole quantities, 24.00 among them
    price = rng.integers(90_000, 10_500_000, n).astype(np.int64)    # 900.00 .. 104999.99
    dn = rng.random(n) < 0.01
    cols = [Column(ship), Column(_d152(disc, rng), dn), Column(_d152(qty, rng)), Column(_d152(price, rng))]
    schema = [FieldType(L, abi.FLAG_NOT_NULL), D152, FieldType(DEC, abi.FLAG_NOT_NULL, 15, 2), FieldType(DEC, abi.FLAG_NOT_NULL, 15, 2)]
    d0, d1 = 8766, 9131
    filters = [FilterItem(abi.CMP_GE, 0, const_i64=d0), FilterItem(abi.CMP_LT, 0, const_i64=d1),
               FilterItem(abi.CMP_GE, 1, is_decimal=True, const_cell=TR.dec("0.05")),
               FilterItem(abi.CMP_LE, 1, is_decimal=True, const_cell=TR.dec("0.070", digits_int=9)),
               FilterItem(abi.CMP_LT, 2, is_decimal=True, const_cell=TR.dec("24"))]
    sel = SelectionExec(MockDataSource(schema, Chunk(cols).split(1024)), filters)
    plan = AggPlan(schema, [], [AggFunc(abi.AGG_SUM, 3, DEC, ret_type=DEC, ret_frac=4, arg_col2=1, arg_expr=abi.ARGEXPR_MUL)])
    out = drain(HashAggExec(plan, sel))
    assert len(out) == 1 and out[0].num_rows() == 1
    cell = bytes(out[0].columns[0].data[0])
    keep = (ship >= d0) & (ship < d1) & (disc >= 5) & (disc <= 7) & (qty < 2400) & ~dn
    assert keep.sum() > 1000
    total = sum(int(p) * int(d) for p, d in zip(price[keep], disc[keep]))
    assert D.value(cell) == Fraction(total, 10 ** 4)
    assert cell == A.sum_result(total, 4)


def test_q18_having_over_device_resident_sums():
    # SELECT o_orderkey, sum(l_quantity) FROM lineitem GROUP BY o_orderkey HAVING sum(l_quantity) > 300: the aggregate
    # stays on the device and tg_vec_filter_ex reads its SUM cells (DECIMAL(37,2), some wider than 18 digits)
    import torch
    from tidb_b200.device import DeviceAgg
    rng = np.random.default_rng(18)
    G = 150_000
    per = rng.integers(1, 15, G)
    keys = np.repeat(np.arange(G, dtype=np.int64) * 7 + 3, per)
    qty = rng.integers(100, 5001, len(keys)).astype(np.int64)
    whales = rng.choice(G, 40, replace=False)                      # groups whose sums pass 10^16 (19+ digits)
    wk = np.repeat(whales.astype(np.int64) * 7 + 3, 1500)
    wq = rng.integers(9 * 10 ** 14, 10 ** 15, len(wk)).astype(np.int64) * np.where(np.arange(len(wk)) // 1500 % 2 == 0, 1, -1)
    keys, qty = np.concatenate([keys, wk]), np.concatenate([qty, wq])
    perm = rng.permutation(len(keys))
    keys, qty = keys[perm], qty[perm]
    cells = _d152(qty, rng)
    plan = AggPlan([FieldType(L, abi.FLAG_NOT_NULL), FieldType(DEC, abi.FLAG_NOT_NULL, 15, 2)], [0],
                   [AggFunc(abi.AGG_FIRSTROW, 0), AggFunc(abi.AGG_SUM, 1, DEC, ret_type=DEC, ret_frac=2)])
    kt, ct = torch.from_numpy(keys).cuda(), torch.from_numpy(cells).cuda()
    torch.cuda.synchronize()
    agg = DeviceAgg(plan)
    lib = abi.load_lib()
    try:
        agg.push([kt, ct])
        rows, out_cols, out_nulls = agg.finish()
        chk = abi.TgChunk()
        arr = (abi.TgColumn * 2)()
        for i, (p, el) in enumerate(((out_cols[0], 8), (out_cols[1], 40))):
            arr[i].length, arr[i].data, arr[i].elem_len = rows, p, el
            arr[i].null_bitmap = out_nulls[i] or None
        chk.ncols, chk.cols = 2, C.cast(arr, C.POINTER(abi.TgColumn))
        sel_t = torch.full((rows,), 7, dtype=torch.uint8, device="cuda")
        items = [FilterItem(abi.CMP_GT, 1, is_decimal=True, const_cell=TR.dec("300"))]
        cnt = C.c_int64(-1)
        rc = lib.tg_vec_filter_ex(0, 1, C.byref(chk), (C.c_int32 * 2)(L, DEC), filter_array(items), 1, dec_const_array(items),
                                  C.c_void_p(sel_t.data_ptr()), C.byref(cnt), None)
        assert rc == abi.TG_OK, lib.tg_last_error()
        k = np.zeros(rows, np.int64)
        sums = np.zeros((rows, 40), np.uint8)
        for dst, src in ((k, out_cols[0]), (sums, out_cols[1])):
            abi.check(lib.tg_memcpy_d2h(0, C.c_void_p(dst.ctypes.data), C.c_void_p(src), C.c_size_t(dst.nbytes)))
        torch.cuda.synchronize()
        selected = sel_t.cpu().numpy().astype(bool)
    finally:
        agg.close()
    # reference: exact per-key sums with Python ints, through the codec of tests/mydecimal_args.py
    uk, inv = np.unique(keys, return_inverse=True)
    tot = [0] * len(uk)
    for g, q in zip(inv.tolist(), qty.tolist()):
        tot[g] += q
    want = {int(key): t for key, t in zip(uk, tot)}
    assert rows == len(uk) and sorted(k.tolist()) == sorted(want)
    wide = [r for r in range(rows) if abs(want[int(k[r])]) >= 10 ** 16]
    assert len(wide) == 40
    for r in wide + list(range(0, rows, 997)):
        assert bytes(sums[r]) == A.sum_result(want[int(k[r])], 2)
    exp = np.array([want[int(x)] > 300 * 100 for x in k])
    assert 1000 < exp.sum() < rows - 1000
    assert np.array_equal(selected, exp) and cnt.value == int(exp.sum())
    assert set(k[selected].tolist()) == {key for key, t in want.items() if t > 30000}
