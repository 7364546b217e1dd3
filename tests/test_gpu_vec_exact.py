"""The VecEval kernels (csrc/vec.cu: tg_vec_compare_*, tg_vec_arith_*, tg_vec_filter) and the SelectionExec /
ProjectionExec / TopNExec shims against the exact Python reference (tests/vec_reference.py).

Inputs are drawn from a pool of (lhs, rhs) pairs: every pair of edge values, pairs whose exact result lands on each
overflow edge or one past it, and random full-range pairs.  The pool is evaluated once by the reference, so rows up to
3,000,001 (the grid-stride loops run three sweeps, the last one partial) are checked value by value.  Results, NULL
bitmaps (bits past the last row included) and `selected` bytes must match exactly; REAL results bit for bit, except
that a NaN result only has to be a NaN (IEEE 754 leaves the sign and payload of a produced NaN open)."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest

import vec_reference as R
from tidb_b200 import abi
from tidb_b200 import executor as X
from tidb_b200.chunk import Chunk, Column
from tidb_b200.executor import MockDataSource, ProjectionExec, SelectionExec, TopNExec, drain
from tidb_b200.plan import ColRef, Const, FieldType, FilterItem, ScalarFunc, filter_array

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
import topn as OT   # noqa: E402

pytestmark = pytest.mark.gpu
SIGNS = [(False, False), (False, True), (True, False), (True, True)]
CMP_OPS = [abi.CMP_LT, abi.CMP_LE, abi.CMP_GT, abi.CMP_GE, abi.CMP_EQ, abi.CMP_NE]
ARITH_OPS = [abi.ARITH_PLUS, abi.ARITH_MINUS, abi.ARITH_MUL]
SIZES = [0, 1, 31, 32, 33, 127, 128, 129, 1061, 3_000_001]
BIG = 3_000_001
SWEEP = 132 * 8 * 256 * 4          # rows one grid sweep of the compare / arithmetic kernels covers on an H100
INT_CONSTS = [-1, R.INT64_MIN, R.INT64_MAX, 1 << 32, 3037000500]
REAL_CONSTS = [-0.0, math.inf, math.nan, 1e308]
GUARD = 8                          # bytes after a device result bitmap that no call may write


def _int_pool(rng):
    e = R.INT_EDGES
    a = [x for x in e for _ in e]
    b = [y for _ in e for y in e]
    anchors = e + [3, -3, 100, 1 << 40, -(1 << 40)]
    for x in anchors:
        for t in (R.INT64_MIN, R.INT64_MAX, 0, R.UINT64_MAX, -1, 1 << 63):
            for d in (-1, 0, 1):
                ys = [t + d - x, x - (t + d)]                                   # + and - land on t + d
                if x not in (0, 1 << 63):
                    ys += [(t + d) // x, (t + d) // x + 1]                     # * lands next to t + d
                for y in ys:
                    a.append(R.word(x)); b.append(R.word(y))
                    a.append(R.word(y)); b.append(R.word(x))
    m = 6000
    full = lambda: rng.integers(R.INT64_MIN, R.INT64_MAX, m, endpoint=True, dtype=np.int64)
    small = lambda: rng.integers(-1000, 1000, m).astype(np.int64)
    a = np.concatenate([np.array(a, np.int64), full(), small(), full() >> rng.integers(0, 63, m)])
    b = np.concatenate([np.array(b, np.int64), full(), small(), small()])
    return a, b


def _real_pool(rng):
    e = R.REAL_EDGES
    a = [x for x in e for _ in e] + [1.7976931348623157e308, 1e154, -1e300, 2.2250738585072014e-308, 1e-300]
    b = [y for _ in e for y in e] + [1e292, 1e154, 1e10, -0.5, -1e-300]
    m = 4000
    a = np.concatenate([np.array(a), rng.normal(0, 1e6, m), rng.integers(R.INT64_MIN, R.INT64_MAX, m, dtype=np.int64).view(np.float64)])
    b = np.concatenate([np.array(b), rng.normal(0, 1e-3, m), rng.integers(R.INT64_MIN, R.INT64_MAX, m, dtype=np.int64).view(np.float64)])
    return a, b


class Batch:
    """n rows drawn from a pair pool: every pool pair appears once when n allows, then random pairs"""

    def __init__(self, pool, n, seed):
        rng = np.random.default_rng(seed)
        self.pa, self.pb = pool
        p = len(self.pa)
        idx = rng.permutation(p)[:n]
        if n > p:
            idx = np.concatenate([idx, rng.integers(0, p, n - p)])
        self.idx = idx
        self.a, self.b = self.pa[idx], self.pb[idx]
        self.an, self.bn = rng.random(n) < 0.1, rng.random(n) < 0.1


def _col(v, nl):
    return Column(v, nl if nl is not None and nl.any() else None)


def _bitmap(nulls):
    return np.packbits(~np.asarray(nulls, bool), bitorder="little")


def call_binary(name, op, signs, a, an, b, bn, const, on_device=False):
    """-> (status, result values, result bitmap bytes)"""
    lib = abi.load_lib()
    n = len(a)
    real_out = name == "tg_vec_arith_real"
    ca, cb = _col(a, an), (None if b is None else _col(b, bn))
    sa = ca.to_struct(); sb = None if cb is None else cb.to_struct()
    keep = []
    if on_device:
        import torch
        for s, c in ((sa, ca), (sb, cb)):
            if s is None:
                continue
            d = torch.from_numpy(c.data.view(np.int64).copy()).cuda(); keep.append(d); s.data = d.data_ptr()
            if c.null_bitmap is not None:
                m = torch.from_numpy(c.null_bitmap.copy()).cuda(); keep.append(m); s.null_bitmap = m.data_ptr()
        res_t = torch.full((max(n, 1),), 0x5A5A5A5A, dtype=torch.int64, device="cuda")
        bm_t = torch.full(((n + 7) // 8 + GUARD,), 0xA5, dtype=torch.uint8, device="cuda")     # guard bytes past the bitmap
        rp, bp = C.c_void_p(res_t.data_ptr()), C.c_void_p(bm_t.data_ptr())
    else:
        res = np.full(max(n, 1), 0x5A5A5A5A, np.int64)
        bm = np.full(max((n + 7) // 8, 1), 0xA5, np.uint8)
        rp, bp = res.ctypes.data_as(C.c_void_p), bm.ctypes.data_as(C.c_void_p)
    pb = None if sb is None else C.byref(sb)
    fn = getattr(lib, name)
    if name in ("tg_vec_compare_int", "tg_vec_arith_int"):
        rc = fn(0, int(on_device), op, int(signs[0]), int(signs[1]), C.byref(sa), pb, C.c_int64(R.word(int(const))), rp, bp, None)
    else:
        rc = fn(0, int(on_device), op, C.byref(sa), pb, C.c_double(float(const)), rp, bp, None)
    if on_device:
        torch.cuda.synchronize()
        res, bm = res_t.cpu().numpy(), bm_t.cpu().numpy()
        assert (bm[(n + 7) // 8:] == 0xA5).all(), "the result bitmap was written past its last byte"
    res = res[:n]
    return rc, (res.view(np.float64) if real_out else res), bm[:(n + 7) // 8]


def _assert_real_equal(got, exp, what):
    en, gn = np.isnan(exp), np.isnan(got)
    assert np.array_equal(en, gn), (what, np.flatnonzero(en != gn)[:5])
    bad = np.flatnonzero(got[~en].view(np.int64) != exp[~en].view(np.int64))
    assert len(bad) == 0, (what, got[~en][bad[:5]], exp[~en][bad[:5]])


@pytest.fixture(scope="module")
def pools():
    rng = np.random.default_rng(1)
    return _int_pool(rng), _real_pool(rng)


@pytest.mark.parametrize("n", SIZES)
def test_vec_compare_exact(pools, n):
    for pool, is_real in ((pools[0], False), (pools[1], True)):
        bt = Batch(pool, n, seed=n + is_real)
        for op in CMP_OPS:
            for signs in ([(False, False)] if is_real else SIGNS):
                consts = (REAL_CONSTS if is_real else INT_CONSTS) if n < BIG else [math.nan if is_real else R.INT64_MIN]
                for rhs in [None] + consts:
                    b, bn = (bt.b, bt.bn) if rhs is None else (None, None)
                    if is_real:
                        exp, enul = R.compare_real_col(op, bt.a.view(np.float64), bt.an, b, bn, 0.0 if rhs is None else rhs)
                        rc, res, bm = call_binary("tg_vec_compare_real", op, signs, bt.a, bt.an, b, bn, 0.0 if rhs is None else rhs)
                    else:
                        exp, enul = R.compare_int_col(op, bt.a, bt.an, b, bn, 0 if rhs is None else rhs, *signs)
                        rc, res, bm = call_binary("tg_vec_compare_int", op, signs, bt.a, bt.an, b, bn, 0 if rhs is None else rhs)
                    what = (op, signs, rhs, is_real)
                    assert rc == abi.TG_OK, what
                    bad = np.flatnonzero(res != exp)
                    assert len(bad) == 0, (what, bad[:5], bt.a[bad[:5]], None if b is None else b[bad[:5]])
                    assert np.array_equal(bm, _bitmap(enul)), what


_POOL_RESULTS = {}


def _int_pool_results(pool, op, signs, const):
    """(result, overflow) of every pool pair, or of every pool lhs with the constant; evaluated once per process"""
    key = (op, signs, const)
    if key not in _POOL_RESULTS:
        p_b = pool[1] if const is None else None
        z = np.zeros(len(pool[0]), bool)
        _, res, _ = R.arith_int_vec(op, pool[0], z, p_b, z, const or 0, *signs)
        _POOL_RESULTS[key] = res, R.arith_int_overflow_rows(op, pool[0], p_b, const or 0, *signs)
    return _POOL_RESULTS[key]


@pytest.mark.parametrize("n", SIZES)
def test_vec_arith_int_exact(pools, n):
    pool = pools[0]
    bt = Batch(pool, n, seed=100 + n)
    consts = INT_CONSTS if n < BIG else [R.INT64_MAX, -1]
    for op in ARITH_OPS:
        for signs in SIGNS:
            for rhs in [None] + consts:
                b = bt.b if rhs is None else None
                k = 0 if rhs is None else rhs
                what = (op, signs, rhs)
                p_res, p_ovf = _int_pool_results(pool, op, signs, rhs)     # rows gather the pool's results
                ovf = p_ovf[bt.idx]
                an = bt.an | ovf                                   # every overflowing row under NULL
                bn = None if b is None else bt.bn
                enul = an if b is None else (an | bn)
                rc, res, bm = call_binary("tg_vec_arith_int", op, signs, bt.a, an, b, bn, k)
                assert rc == abi.TG_OK, (what, abi.load_lib().tg_last_error())
                exp = p_res[bt.idx]
                bad = np.flatnonzero(res != exp)
                assert len(bad) == 0, (what, [(int(bt.a[i]), None if b is None else int(b[i]), int(res[i]), int(exp[i])) for i in bad[:5]])
                assert np.array_equal(bm, _bitmap(enul)), what
                # one overflowing row left non-NULL fails the call: in the tail word, and in the second grid sweep
                hits = np.flatnonzero(p_ovf)
                if n == 0 or len(hits) == 0:
                    continue
                j = int(hits[len(hits) // 2])
                for pos in ([n - 1, SWEEP + 37] if n > SWEEP else [n - 1]):
                    a2, an2 = bt.a.copy(), an.copy()
                    a2[pos], an2[pos] = pool[0][j], False
                    b2, bn2 = (None, None) if b is None else (b.copy(), bn.copy())
                    if b2 is not None:
                        b2[pos], bn2[pos] = pool[1][j], False
                    rc, res2, bm2 = call_binary("tg_vec_arith_int", op, signs, a2, an2, b2, bn2, k)
                    assert rc == abi.TG_ERR_OVERFLOW, (what, pos)
                    assert (res2 == 0x5A5A5A5A).all() and (bm2 == 0xA5).all(), (what, pos)   # host buffers untouched


@pytest.mark.parametrize("n", SIZES)
def test_vec_arith_real_exact(pools, n):
    pool = pools[1]
    bt = Batch(pool, n, seed=200 + n)
    a = bt.a.view(np.float64)
    for op in ARITH_OPS:
        for rhs in [None] + REAL_CONSTS:
            b = bt.b.view(np.float64) if rhs is None else None
            k = 0.0 if rhs is None else rhs
            p_b = pool[1] if rhs is None else None
            _, p_res, _, p_ovf = R.arith_real_vec(op, pool[0], np.zeros(len(pool[0]), bool), p_b, np.zeros(len(pool[0]), bool), k)
            ovf = p_ovf[bt.idx]
            an = bt.an | ovf
            bn = None if b is None else bt.bn
            rc, res, bm = call_binary("tg_vec_arith_real", op, None, a, an, b, bn, k)
            what = (op, rhs)
            assert rc == abi.TG_OK, what
            _assert_real_equal(res, p_res[bt.idx], what)
            assert np.array_equal(bm, _bitmap(an if b is None else an | bn)), what
            if n and ovf.any():
                pos = n - 1
                j = int(np.flatnonzero(p_ovf)[0])
                a2, an2 = a.copy(), an.copy()
                a2[pos], an2[pos] = pool[0][j], False
                b2, bn2 = (None, None) if b is None else (b.copy(), bn.copy())
                if b2 is not None:
                    b2[pos], bn2[pos] = pool[1][j], False
                rc, res2, bm2 = call_binary("tg_vec_arith_real", op, None, a2, an2, b2, bn2, k)
                assert rc == abi.TG_ERR_OVERFLOW, what
                assert (res2.view(np.int64) == 0x5A5A5A5A).all() and (bm2 == 0xA5).all(), what   # host buffers untouched


def test_vec_real_signed_zero_nan_and_inf_times_zero():
    a = np.array([-0.0, -0.0, 0.0, 0.0, 5.0, np.inf, -np.inf, np.nan, 5e-324, -5e-324])
    b = np.array([-0.0, 0.0, -0.0, -3.0, -5.0, 0.0, 0.0, 2.0, 0.5, 0.5])
    for op in ARITH_OPS:
        _, e, _, ovf = R.arith_real_vec(op, a, np.zeros(10, bool), b, np.zeros(10, bool))
        rc, res, _ = call_binary("tg_vec_arith_real", op, None, a, ovf, b, None, 0.0)
        assert rc == abi.TG_OK
        _assert_real_equal(res, e, op)
    # -0 results and inf * 0 = NaN without an error
    rc, res, _ = call_binary("tg_vec_arith_real", abi.ARITH_MUL, None, a[:7], np.zeros(7, bool), b[:7], None, 0.0)
    assert rc == abi.TG_OK
    assert [math.copysign(1, x) for x in res[:5]] == [1, -1, -1, -1, -1] and np.isnan(res[5:7]).all()


@pytest.mark.parametrize("n", [33, 70_001])
def test_vec_on_device_every_entry_point(pools, n):
    bi, br = Batch(pools[0], n, 7), Batch(pools[1], n, 8)
    exp, enul = R.compare_int_col(abi.CMP_LE, bi.a, bi.an, bi.b, bi.bn, 0, True, False)
    rc, res, bm = call_binary("tg_vec_compare_int", abi.CMP_LE, (True, False), bi.a, bi.an, bi.b, bi.bn, 0, on_device=True)
    assert rc == 0 and np.array_equal(res, exp) and np.array_equal(bm, _bitmap(enul))
    exp, enul = R.compare_real_col(abi.CMP_GE, br.a.view(np.float64), br.an, None, None, -0.0)
    rc, res, bm = call_binary("tg_vec_compare_real", abi.CMP_GE, None, br.a, br.an, None, None, -0.0, on_device=True)
    assert rc == 0 and np.array_equal(res, exp) and np.array_equal(bm, _bitmap(enul))
    for signs in SIGNS:
        ovf = R.arith_int_overflow_rows(abi.ARITH_MUL, bi.a, bi.b, 0, *signs)
        _, exp, enul = R.arith_int_vec(abi.ARITH_MUL, bi.a, bi.an | ovf, bi.b, bi.bn, 0, *signs)
        rc, res, bm = call_binary("tg_vec_arith_int", abi.ARITH_MUL, signs, bi.a, bi.an | ovf, bi.b, bi.bn, 0, on_device=True)
        assert rc == 0 and np.array_equal(res, exp) and np.array_equal(bm, _bitmap(enul)), signs
    _, _, _, ovf = R.arith_real_vec(abi.ARITH_MINUS, br.a.view(np.float64), br.an, br.b.view(np.float64), br.bn)
    _, exp, enul, _ = R.arith_real_vec(abi.ARITH_MINUS, br.a.view(np.float64), br.an | ovf, br.b.view(np.float64), br.bn)
    rc, res, bm = call_binary("tg_vec_arith_real", abi.ARITH_MINUS, None, br.a, br.an | ovf, br.b, br.bn, 0.0, on_device=True)
    assert rc == 0 and np.array_equal(bm, _bitmap(enul))
    _assert_real_equal(res, exp, "on device")
    run_filter_check(pools, n, on_device=True)


# ---- tg_vec_filter ------------------------------------------------------------------------------------------
def _filter_table(pools, n):
    bi, bi2, br = Batch(pools[0], n, 30), Batch(pools[0], n, 31), Batch(pools[1], n, 32)
    cols = [(bi.a, bi.an), (bi.b, bi.bn), (bi2.a, np.zeros(n, bool)), (br.a, br.an), (br.b, br.bn)]
    return cols


FILTER_SETS = [
    [FilterItem(abi.CMP_GT, 0, const_i64=-2, lhs_unsigned=True, rhs_unsigned=True)],
    [FilterItem(abi.CMP_LT, 0, rhs_col=1, lhs_unsigned=True)],
    [FilterItem(abi.CMP_GE, 1, rhs_col=2, rhs_unsigned=True)],
    [FilterItem(abi.CMP_EQ, 2, const_i64=R.INT64_MIN, lhs_unsigned=True, rhs_unsigned=True)],
    [FilterItem(abi.CMP_LE, 0, const_i64=R.INT64_MAX, rhs_unsigned=True), FilterItem(abi.CMP_NE, 1, rhs_col=0, lhs_unsigned=True, rhs_unsigned=True)],
    [FilterItem(abi.CMP_EQ, 3, is_real=True, const_f64=-0.0)],
    [FilterItem(abi.CMP_LT, 3, rhs_col=4, is_real=True)],
    [FilterItem(abi.CMP_LE, 4, is_real=True, const_f64=math.nan)],
    [FilterItem(abi.CMP_GT, 0, const_i64=-1000), FilterItem(abi.CMP_LT, 1, const_i64=-1, rhs_unsigned=True),
     FilterItem(abi.CMP_NE, 0, rhs_col=2, lhs_unsigned=True), FilterItem(abi.CMP_GE, 2, const_i64=1 << 32, lhs_unsigned=True),
     FilterItem(abi.CMP_GT, 3, is_real=True, const_f64=-math.inf), FilterItem(abi.CMP_NE, 4, is_real=True, const_f64=0.0),
     FilterItem(abi.CMP_LE, 1, rhs_col=0, rhs_unsigned=True), FilterItem(abi.CMP_GE, 3, rhs_col=4, is_real=True)],
]


def call_filter(cols, items, sel=None, on_device=False):
    lib = abi.load_lib()
    chk = Chunk([_col(v, nl) for v, nl in cols], sel)
    cs = chk.to_struct()
    n = len(cols[0][0])
    keep = []
    if on_device:
        import torch
        for i, c in enumerate(chk.columns):
            d = torch.from_numpy(c.data.view(np.int64).copy()).cuda(); keep.append(d); cs.cols[i].data = d.data_ptr()
            if c.null_bitmap is not None:
                m = torch.from_numpy(c.null_bitmap.copy()).cuda(); keep.append(m); cs.cols[i].null_bitmap = m.data_ptr()
        if sel is not None:
            s = torch.from_numpy(chk.sel.copy()).cuda(); keep.append(s); cs.sel = s.data_ptr()
        out_t = torch.full((max(n, 1),), 7, dtype=torch.uint8, device="cuda")
        out_p = C.c_void_p(out_t.data_ptr())
    else:
        out = np.full(max(n, 1), 7, np.uint8)
        out_p = out.ctypes.data_as(C.c_void_p)
    cnt = C.c_int64(-1)
    rc = lib.tg_vec_filter(0, int(on_device), C.byref(cs), filter_array(items), len(items), out_p, C.byref(cnt), None)
    if on_device:
        torch.cuda.synchronize()
        out = out_t.cpu().numpy()
    return rc, out[:n], cnt.value


def run_filter_check(pools, n, on_device=False):
    cols = _filter_table(pools, n)
    sel = np.sort(np.random.default_rng(n).choice(n, n // 2, replace=False)).astype(np.int64)
    for items in FILTER_SETS:
        for s in (None, sel):
            exp = R.filter_rows(cols, items, s)
            rc, got, cnt = call_filter(cols, items, s, on_device)
            assert rc == abi.TG_OK
            assert np.array_equal(got, exp.astype(np.uint8)) and cnt == int(exp.sum()), (items, s is not None)


@pytest.mark.parametrize("n", [1061, BIG])
def test_vec_filter_exact(pools, n):
    run_filter_check(pools, n)


# ---- executors ------------------------------------------------------------------------------------------------
INT, UINT, DBL = FieldType(abi.TYPE_LONGLONG, 0), FieldType(abi.TYPE_LONGLONG, abi.FLAG_UNSIGNED), FieldType(abi.TYPE_DOUBLE, 0)


def _sel_chunks(rng, cols, rows_per_chunk=1024):
    """physical columns cut into chunks, each carrying a sel vector of about 2/3 of its rows; -> (chunks, logical rows)"""
    n = len(cols[0][0])
    chunks, logical = [], []
    for lo in range(0, n, rows_per_chunk):
        hi = min(n, lo + rows_per_chunk)
        keep = np.sort(rng.choice(hi - lo, max(1, (hi - lo) * 2 // 3), replace=False)).astype(np.int64)
        chunks.append(Chunk([_col(v[lo:hi].copy(), nl[lo:hi]) for v, nl in cols], keep))
        logical.append(lo + keep)
    return chunks, np.concatenate(logical)


def _collect(chunks, ncols):
    vals = [np.concatenate([c.columns[i].data for c in chunks]) if chunks else np.zeros(0, np.int64) for i in range(ncols)]
    nulls = [np.concatenate([c.columns[i].nulls() for c in chunks]) if chunks else np.zeros(0, bool) for i in range(ncols)]
    return vals, nulls


def _exec_table(rng, n):
    a = rng.integers(-1000, 1000, n).astype(np.int64)
    u = np.where(rng.random(n) < 0.5, rng.integers(1000, 5000, n), rng.integers(R.INT64_MIN, R.INT64_MIN + 1000, n)).astype(np.int64)
    x = np.round(rng.normal(0, 100, n), 2); x[::17] = -0.0; x[::23] = np.nan
    return [(a, rng.random(n) < 0.1), (u, rng.random(n) < 0.1), (x, rng.random(n) < 0.1)]


@pytest.mark.parametrize("required_rows", [1, 7, 1024])
def test_selection_and_projection_over_sel_vectors(required_rows):
    rng = np.random.default_rng(required_rows)
    cols = _exec_table(rng, 5000)
    schema = [INT, UINT, DBL]
    chunks, logical = _sel_chunks(rng, cols)
    lcols = [(v[logical], nl[logical]) for v, nl in cols]
    filters = [FilterItem(abi.CMP_GT, 1, const_i64=500, lhs_unsigned=True), FilterItem(abi.CMP_NE, 0, rhs_col=1, rhs_unsigned=True),
               FilterItem(abi.CMP_GE, 2, is_real=True, const_f64=-0.0)]
    keep = R.filter_rows(lcols, filters)
    e = SelectionExec(MockDataSource(schema, chunks), filters, batch_rows=2048)
    for _ in range(2):                                       # Open again after Close re-executes
        out = drain(e, required_rows)
        assert all(0 < c.num_rows() <= required_rows for c in out)
        vals, nulls = _collect(out, 3)
        for c in range(3):
            assert np.array_equal(nulls[c], lcols[c][1][keep])
            assert np.array_equal(vals[c].view(np.int64)[~nulls[c]], lcols[c][0].view(np.int64)[keep][~lcols[c][1][keep]])
    exprs = [ColRef(2), ScalarFunc("arith", abi.ARITH_PLUS, (ColRef(1), ColRef(0)), a_unsigned=True),
             ScalarFunc("arith", abi.ARITH_MINUS, (ColRef(1), Const(-7)), a_unsigned=True),
             ScalarFunc("cmp", abi.CMP_LT, (ColRef(0), ColRef(1)), b_unsigned=True),
             ScalarFunc("arith", abi.ARITH_MUL, (ColRef(2), Const(-1.0, True)), is_real=True)]
    e = ProjectionExec(MockDataSource(schema, chunks), exprs, batch_rows=2048)
    assert [t.flag & abi.FLAG_UNSIGNED for t in e.schema] == [0, abi.FLAG_UNSIGNED, abi.FLAG_UNSIGNED, 0, 0]
    (av, an), (uv, un), (xv, xn) = lcols
    _, s_, sn = R.arith_int_vec(abi.ARITH_PLUS, uv, un, av, an, 0, True, False)
    _, d_, dn = R.arith_int_vec(abi.ARITH_MINUS, uv, un, None, None, -7, True, False)
    lt, ltn = R.compare_int_col(abi.CMP_LT, av, an, uv, un, 0, False, True)
    _, m_, mn, _ = R.arith_real_vec(abi.ARITH_MUL, xv, xn, None, None, -1.0)
    exp = [(xv, xn), (s_, sn), (d_, dn), (lt, ltn), (m_, mn)]
    for _ in range(2):
        out = drain(e, required_rows)
        assert all(0 < c.num_rows() <= required_rows for c in out)
        vals, nulls = _collect(out, len(exprs))
        for c, (ev, en) in enumerate(exp):
            assert np.array_equal(nulls[c], en), c
            g, w = vals[c][~en], np.asarray(ev)[~en]
            if g.dtype == np.float64:
                _assert_real_equal(g, w, c)
            else:
                assert np.array_equal(g, w), c


def test_unsigned_projection_feeds_topn():
    # ProjectionExec(u + a) over an UNSIGNED u is UNSIGNED: a TopN above it orders sums past 2^63 as large values
    rng = np.random.default_rng(12)
    n = 20_000
    u = np.where(rng.random(n) < 0.5, rng.integers(2000, 1 << 40, n), rng.integers(R.INT64_MIN, R.INT64_MIN + (1 << 40), n)).astype(np.int64)
    a = rng.integers(-1000, 1000, n).astype(np.int64)
    ids = rng.permutation(n).astype(np.int64)
    un = rng.random(n) < 0.05
    src = Chunk([Column(u, un), Column(a), Column(ids)]).split(1024)
    _, s_, sn = R.arith_int_vec(abi.ARITH_PLUS, u, un, a, np.zeros(n, bool), 0, True, False)
    for desc in (False, True):
        proj = ProjectionExec(MockDataSource([UINT, INT, INT], src), [ScalarFunc("arith", abi.ARITH_PLUS, (ColRef(0), ColRef(1)), a_unsigned=True), ColRef(2)])
        out = drain(TopNExec(proj, [(0, desc)], 3, 50), 1024)
        vals, nulls = _collect(out, 2)
        exp = OT.topn_order([(s_, sn), (ids, np.zeros(n, bool))], ["uint", "int"], [(0, desc)], 3, 50)
        assert len(vals[0]) == len(exp) == 50
        row = np.argsort(ids)[vals[1]]                      # the input row of each output row
        assert np.array_equal(nulls[0], sn[row]) and np.array_equal(vals[0][~nulls[0]], s_[row][~nulls[0]])
        gk = OT.item_keys([(s_, sn)], ["uint"], [(0, desc)], row)
        ek = OT.item_keys([(s_, sn)], ["uint"], [(0, desc)], exp)
        assert np.array_equal(gk, ek), desc


def test_topn_exec_huge_limit_allocates_by_input(monkeypatch):
    # LIMIT 10^12 over 300 rows returns the 300 rows in order, and the output buffer is sized by the input
    sizes = []
    real = X._out_chunk

    def recording(schema, capacity):
        sizes.append(capacity)
        assert capacity <= 1 << 20, f"TopNExec asked for a {capacity}-row output buffer"
        return real(schema, capacity)

    monkeypatch.setattr(X, "_out_chunk", recording)
    rng = np.random.default_rng(4)
    n = 300
    v = rng.integers(-50, 50, n).astype(np.int64)
    vn = rng.random(n) < 0.1
    ids = rng.permutation(n).astype(np.int64)
    for offset, exp_rows in ((0, n), (10, n - 10), (n, 0), (10**12, 0)):
        out = drain(TopNExec(MockDataSource([INT, INT], Chunk([Column(v, vn), Column(ids)]).split(64)), [(0, True)], offset, 10**12), 100)
        vals, nulls = _collect(out, 2)
        assert len(vals[1]) == exp_rows and len(np.unique(vals[1])) == exp_rows
        exp = OT.topn_order([(v, vn), (ids, np.zeros(n, bool))], ["int", "int"], [(0, True)], offset, 10**12)
        row = np.argsort(ids)[vals[1]]
        assert np.array_equal(OT.item_keys([(v, vn)], ["int"], [(0, True)], row), OT.item_keys([(v, vn)], ["int"], [(0, True)], exp))
    assert sizes and max(sizes) <= n
