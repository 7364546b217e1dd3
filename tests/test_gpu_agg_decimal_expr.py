"""SUM / AVG of a * b and a * (c - b) over DECIMAL(p <= 18) columns on every update path of the CUDA hash aggregation,
compared exactly.

Each case forces one path through the TG_AGG_* switches, proves from tg_agg_stats.paths / local_rows that it ran, and
compares every group's 40-byte MyDecimal cell byte for byte with tests/mydecimal_expr.py.  The data holds groups of
+-(10^p - 1) products whose sums pass 2^64 and 2^128 in both directions, groups that cancel to 0, all-NULL groups, products
of exactly -1 and 2^64 - 1, NULLs in either operand, and cells in the stored form's variants with garbage under NULL
(tests/test_gpu_agg_decimal_args.py builds them)."""
import ctypes as C
import functools

import numpy as np
import pytest

import mydecimal as D
import mydecimal_args as A
import mydecimal_expr as X
import test_gpu_agg_decimal_args as T
from tidb_b200 import abi
from tidb_b200.chunk import Chunk, Column, unpack_nulls
from tidb_b200.executor import HashAggExec, MockDataSource
from tidb_b200.plan import AggFunc, AggPlan, FieldType

pytestmark = pytest.mark.gpu

P = abi
DEC = abi.TYPE_NEWDECIMAL
INT = FieldType(abi.TYPE_LONGLONG, 0)
INT_NN = FieldType(abi.TYPE_LONGLONG, abi.FLAG_NOT_NULL)
SWITCHES = ("TG_AGG_LOCAL", "TG_AGG_LOCAL_SLOTS", "TG_AGG_V1")
K_MAX, K_MIN, K_CANCEL, K_ALLNULL, K_M1, K_U64 = (7_000_000_000_000 + j for j in range(6))
# (p_a, s_a, p_b, s_b): the scale pairs (0,0), (2,2), (9,9), (18,0), (12,18) (s = 30) and DECIMAL(15,2) x DECIMAL(15,2)
SCALES = [(18, 0, 18, 0), (18, 2, 18, 2), (18, 9, 18, 9), (18, 18, 18, 0), (18, 12, 18, 18), (15, 2, 15, 2)]
# the paths that share their update code with one already run at every scale (V2 global, the AVG cases) take three pairs:
# scale 0, scale 30 and the TPC-H columns
SOME = [SCALES[0], SCALES[4], SCALES[5]]


@pytest.fixture(autouse=True)
def _default_switches(monkeypatch):
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)


# ---- data --------------------------------------------------------------------------------------------------------
# columns: 0 g BIGINT key (nullable) | 1 a DECIMAL(pa, sa) (nullable) | 2 b DECIMAL(pb, sb) (nullable)
#          3 a' DECIMAL(pa, sa) NOT NULL | 4 b' DECIMAL(pb, sb) NOT NULL | 5 k BIGINT NOT NULL (second GROUP BY column)
def types_of(sc):
    pa, sa, pb, sb = sc
    return [INT, FieldType(DEC, 0, pa, sa), FieldType(DEC, 0, pb, sb), FieldType(DEC, abi.FLAG_NOT_NULL, pa, sa),
            FieldType(DEC, abi.FLAG_NOT_NULL, pb, sb), INT_NN]


def make_rows(rng, n, ngroups, sc):
    pa, sa, pb, sb = sc
    la, lb = 10 ** pa - 1, 10 ** pb - 1
    g = (rng.integers(0, ngroups, n) * 2654435761 % (1 << 40) - (1 << 39)).astype(np.int64)
    sp = rng.random(n) < 0.06
    g[sp] = rng.choice(np.array([K_MAX, K_MIN, K_CANCEL, K_ALLNULL, K_M1, K_U64], dtype=np.int64), int(sp.sum()))
    gn = rng.random(n) < 0.01
    g[gn] = 0
    a, b, a2, b2 = (T.dec_values(rng, n, p, s) for p, s in ((pa, sa), (pb, sb), (pa, sa), (pb, sb)))
    for k, va, vb in ((K_MAX, la, lb), (K_MIN, -la, lb), (K_M1, 1, -1), (K_U64, (1 << 32) - 1, (1 << 32) + 1)):
        m = (g == k) & ~gn
        a[m], a2[m], b[m] = va, va, vb
        b2[m] = vb if k != K_MIN else -vb                  # a' * b' of K_MIN is positive, a * b negative
    idx = np.flatnonzero((g == K_CANCEL) & ~gn)            # (x, y) / (-x, y) pairs: every product sum is exactly 0
    for col in (a, a2):
        col[idx[1::2]] = -col[idx[0:len(idx) // 2 * 2:2]]
        if len(idx) % 2:
            col[idx[-1]] = 0
    for col in (b, b2):
        col[idx[1::2]] = col[idx[0:len(idx) // 2 * 2:2]]
    an = (rng.random(n) < 0.05) | ((g == K_ALLNULL) & ~gn)
    bn = (rng.random(n) < 0.05) & (g != K_MAX) & (g != K_MIN) & (g != K_CANCEL)
    k2 = rng.integers(-3, 4, n).astype(np.int64)
    chunk = Chunk([Column(g, gn), Column(T.encode(rng, a, pa, sa, an), an), Column(T.encode(rng, b, pb, sb, bn), bn),
                   Column(T.encode(rng, a2, pa, sa)), Column(T.encode(rng, b2, pb, sb)), Column(k2)])
    z = np.zeros(n, dtype=bool)
    return chunk, {0: (g, gn), 1: (a, an), 2: (b, bn), 3: (a2, z), 4: (b2, z), 5: (k2, z)}


@functools.lru_cache(maxsize=None)
def dataset(sc, n=120_000, ngroups=5000, seed=0):
    return make_rows(np.random.default_rng(seed + sum(sc)), n, ngroups, sc)


def consts(sc):
    """c = 1 (1 - l_discount) and the largest |c| the bound allows, negative: c * 10^s_b = -10^18"""
    return 1, -(10 ** (18 - sc[3]))


def xf(name, a, b, f, expr=X.MUL, c=0):
    return AggFunc(name, a, DEC, ret_type=DEC, ret_frac=f, arg_col2=b, arg_expr=expr, arg_const=float(c))


def plans(sc, group_by=(0,), expected_groups=0, local=True):
    """lists of at most 4 device states (the CTA-local level takes no more), and with local=False one plan mixing the
    products with COUNT(*) and a DECIMAL column SUM"""
    s = sc[1] + sc[3]
    c1, c2 = consts(sc)
    f1, f2 = min(s + 4, 30), 30
    S, V = P.AGG_SUM, P.AGG_AVG
    fr = [AggFunc(P.AGG_FIRSTROW, g) for g in group_by]
    lists = [[xf(S, 1, 2, s)], [xf(S, 3, 4, s, X.MUL_CSUB, c1)], [xf(V, 3, 2, f1)], [xf(V, 1, 4, f2, X.MUL_CSUB, c2)],
             [xf(S, 3, 4, s, X.MUL_CSUB, c2)], [xf(V, 3, 4, f1, X.MUL_CSUB, c1)]]
    if not local:   # the same column twice (a' * a' or b' * b', whichever scale stays <= 30), and b' * a
        same = xf(V, 3, 3, min(2 * sc[1] + 1, 30)) if 2 * sc[1] <= 30 else xf(V, 4, 4, min(2 * sc[3] + 1, 30))
        lists.append([xf(S, 1, 2, s), xf(V, 1, 2, f1, X.MUL_CSUB, c1), xf(S, 3, 4, s, X.MUL_CSUB, c2), AggFunc(P.AGG_COUNT, -1),
                      AggFunc(P.AGG_SUM, 1, DEC, ret_type=DEC, ret_frac=sc[1]), same, xf(S, 4, 1, s)])
    return [AggPlan(types_of(sc), list(group_by), fr + fs, expected_groups=expected_groups) for fs in lists]


# ---- exact reference ---------------------------------------------------------------------------------------------
def expected(plan, vals):
    """group key tuple -> {function index: expected cell / count / None} for every function but FIRSTROW"""
    inv, tuples = T._group_ids(plan, vals)
    ng = len(tuples)
    out = {t: {} for t in tuples}
    for k, f in enumerate(plan.funcs):
        if f.name == P.AGG_FIRSTROW:
            continue
        if f.name == P.AGG_COUNT:
            cnt = np.bincount(inv, minlength=ng)
            for j, t in enumerate(tuples):
                out[t][k] = int(cnt[j])
            continue
        ta, (va, na) = plan.col_types[f.arg_col], vals[f.arg_col]
        if f.arg_expr == X.MUL or f.arg_expr == X.MUL_CSUB:
            tb, (vb, nb) = plan.col_types[f.arg_col2], vals[f.arg_col2]
            v, keep, s = X.products(va, vb, f.arg_expr, int(f.arg_const), tb.decimal), ~(na | nb), ta.decimal + tb.decimal
        else:
            v, keep, s = va.astype(object), ~na, ta.decimal
        sums, cnt = X.group_sums(v, keep, inv, ng)
        for j, cell in enumerate(X.expected_cells(sums, cnt, f.name == P.AGG_AVG, s, f.ret_frac)):
            out[tuples[j]][k] = cell
    return out


def check(plan, vals, got_rows):
    exp = expected(plan, vals)
    ng = len(plan.group_by)
    got = {}
    for r in got_rows:
        key = tuple(r[:ng])
        assert key not in got, f"group {key} emitted twice"
        got[key] = r
    assert set(got) == set(exp), sorted(set(map(repr, exp)) ^ set(map(repr, got)))[:10]
    for key, want in exp.items():
        for k, cell in want.items():
            g = got[key][k]
            if isinstance(cell, bytes) and isinstance(g, bytes):
                assert g == cell, f"group {key!r} aggregate {k}: got {D.to_string(g)} {D.decode(g)}, want {D.to_string(cell)} {D.decode(cell)}"
            else:
                assert g == cell, (key, k, g, cell)
    return len(exp)


def check_all(plan_list, chunks, vals, want, dont=0, local=None):
    st = None
    for plan in plan_list:
        rows, st = T.run_host(plan, chunks)
        check(plan, vals, rows)
        assert st.paths & want == want, (hex(st.paths), hex(want))
        assert st.paths & dont == 0, (hex(st.paths), hex(dont))
        if local is not None:
            assert (st.local_rows > 0) == local, st.local_rows
    return st


# ---- paths -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sc", SOME)
def test_no_group_by(sc):
    chunk, vals = dataset(sc)
    check_all(plans(sc, group_by=(), local=False), chunk.split(1 << 15), vals, want=P.AGG_PATH_NOGROUP, dont=~P.AGG_PATH_NOGROUP)


@pytest.mark.parametrize("sc", SCALES)
def test_v2_global(sc, monkeypatch):
    monkeypatch.setenv("TG_AGG_LOCAL", "0")
    chunk, vals = dataset(sc)
    check_all(plans(sc, local=False), chunk.split(1 << 15), vals, want=P.AGG_PATH_V2_GLOBAL, dont=P.AGG_PATH_V2_LOCAL | P.AGG_PATH_MERGE, local=False)


@pytest.mark.parametrize("sc", SOME)
def test_v2_cta_local(sc):
    chunk, vals = make_rows(np.random.default_rng(40 + sum(sc)), 150_000, 60, sc)
    check_all(plans(sc), chunk.split(1 << 15), vals, want=P.AGG_PATH_V2_LOCAL, local=True)


@pytest.mark.parametrize("sc", [SCALES[1], SCALES[4], SCALES[5]])
def test_v2_local_spills_and_merges(sc, monkeypatch):
    monkeypatch.setenv("TG_AGG_LOCAL", "2")
    chunk, vals = dataset(sc)
    st = check_all(plans(sc, expected_groups=64), chunk.split(1 << 16), vals, want=P.AGG_PATH_V2_LOCAL | P.AGG_PATH_MERGE, local=True)
    assert st.table_slots > 1024


@pytest.mark.parametrize("sc", SOME)
def test_multi_key(sc):
    chunk, vals = make_rows(np.random.default_rng(50 + sum(sc)), 150_000, 50, sc)
    check_all(plans(sc, group_by=(0, 5), expected_groups=16, local=False), chunk.split(1 << 15), vals, want=P.AGG_PATH_MULTI_KEY,
              dont=~P.AGG_PATH_MULTI_KEY)


@pytest.mark.parametrize("ngroups,hint,want", [(60, 0, P.AGG_PATH_V1_LOCAL | P.AGG_PATH_MERGE), (60_000, 60_000, P.AGG_PATH_V1_GLOBAL)])
@pytest.mark.parametrize("sc", [SCALES[4], SCALES[5]])
def test_v1_paths(ngroups, hint, want, sc, monkeypatch):
    monkeypatch.setenv("TG_AGG_V1", "1")
    monkeypatch.setenv("TG_AGG_LOCAL_SLOTS", "512")
    chunk, vals = make_rows(np.random.default_rng(60 + ngroups + sum(sc)), 150_000, ngroups, sc)
    check_all(plans(sc, expected_groups=hint), chunk.split(1 << 15), vals, want=want, dont=P.AGG_PATH_V2_LOCAL | P.AGG_PATH_V2_GLOBAL, local=False)


# ---- AVG rounding and signs at every scale ------------------------------------------------------------------------
AVG_CASES = [(1, 2), (-1, 2), (3, 2), (-3, 2), (1, 8), (-1, 8), (1, 32), (-1, 32), (5, 16), (-5, 16), (2, 3), (-2, 3), (-1, 3),
             (7, 7), (0, 5), (1, 64), (-1, 64), (99999, 100000), (-99999, 100000)]


@pytest.mark.parametrize("sc", SCALES)
@pytest.mark.parametrize("local", ["0", "2"])
def test_avg_ties_and_signs_every_frac(sc, local, monkeypatch):
    # one group per (sum, count): a row whose product is `sum` units of 10^-s and count - 1 zero rows, for AVG at every
    # ret_frac from s to 30, as a * b (b = 10^-s_b) and as a * (1 - b) (b = 1 - 10^-s_b)
    monkeypatch.setenv("TG_AGG_LOCAL", local)
    pa, sa, pb, sb = sc
    s = sa + sb
    lim = 10 ** min(pa, 18) - 1
    cases = AVG_CASES + [(lim, 2), (-lim, 2), (lim, 1), (-lim, 3)]
    g, x = [], []
    for j, (sm, n) in enumerate(cases):
        g += [j] * n
        x += [sm] + [0] * (n - 1)
    rng = np.random.default_rng(90 + s + int(local))
    perm = rng.permutation(len(g))
    g = np.array(g, dtype=np.int64)[perm]
    x = np.array(x, dtype=np.int64)[perm]
    one = np.ones(len(g), dtype=np.int64)
    bm = np.full(len(g), 10 ** sb - 1, dtype=np.int64)     # 1 - b = 10^-s_b
    z = np.zeros(len(g), dtype=bool)
    chunk = Chunk([Column(g), Column(T.encode(rng, x, pa, sa)), Column(T.encode(rng, one, pb, sb)), Column(T.encode(rng, bm, pb, sb))])
    cols = [INT_NN, FieldType(DEC, abi.FLAG_NOT_NULL, pa, sa), FieldType(DEC, abi.FLAG_NOT_NULL, pb, sb), FieldType(DEC, abi.FLAG_NOT_NULL, pb, sb)]
    vals = {0: (g, z), 1: (x, z), 2: (one, z), 3: (bm, z)}
    fracs = list(range(s, 31))
    for lo in range(0, len(fracs), 8):                     # 3 state words each: 8 per plan
        funcs = [xf(P.AGG_AVG, 1, 2, f) if (f + lo) % 2 else xf(P.AGG_AVG, 1, 3, f, X.MUL_CSUB, 1) for f in fracs[lo:lo + 8]]
        plan = AggPlan(cols, [0], [AggFunc(P.AGG_FIRSTROW, 0)] + funcs)
        rows, _ = T.run_host(plan, chunk.split(1 << 15))
        assert check(plan, vals, rows) == len(cases)
        for r in rows:
            for cell in r[1:]:
                assert not (D.decode(cell).negative and D.value(cell) == 0), D.to_string(cell)


# ---- input routes ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("misalign", [False, True])
def test_device_pushes(misalign):
    sc = SCALES[5]
    rng = np.random.default_rng(70 + misalign)
    parts = [make_rows(rng, n, g, sc) for n, g in ((50_001, 30), (100_000, 3000), (99_999, 30_000))]
    vals = T._concat([v for _, v in parts])
    for plan in plans(sc, expected_groups=16, local=False)[::3]:
        rows, st = T.run_dev(plan, [c for c, _ in parts], misalign)
        check(plan, vals, rows)
        assert st.table_slots > 1024
    plan = plans(sc, group_by=(), local=False)[-1]
    rows, _ = T.run_dev(plan, [c for c, _ in parts], misalign)
    check(plan, vals, rows)


def test_host_pushes_with_sel():
    # the rows a sel vector leaves out hold cells in no valid form: they must never reach the decoder
    sc = SCALES[2]
    rng = np.random.default_rng(80)
    chunk, vals = make_rows(rng, 120_000, 500, sc)
    n = chunk.num_rows()
    cols = []
    for col in chunk.columns:
        if col.data.ndim == 2:
            data = rng.integers(0, 256, (2 * n, 40), dtype=np.uint8)
            data[:, 1] = 77                                # digitsFrac != s
        else:
            data = rng.integers(-5, 5, 2 * n).astype(col.data.dtype)
        data[0::2] = col.data
        nl = np.zeros(2 * n, dtype=bool)
        nl[0::2] = col.nulls()
        cols.append(Column(data, nl))
    big = Chunk(cols)
    chunks = []
    for lo in range(0, 2 * n, 1 << 14):
        part = Chunk([c.slice(lo, min(2 * n, lo + (1 << 14))) for c in big.columns])
        chunks.append(Chunk(part.columns, np.arange(0, part.num_rows(), 2)))
    check_all(plans(sc), chunks, vals, want=P.AGG_PATH_V2_LOCAL)
    check_all(plans(sc, local=False)[-1:], chunks, vals, want=P.AGG_PATH_V2_GLOBAL)


def test_paging_and_result_dev():
    sc = SCALES[5]
    chunk, vals = dataset(sc)
    chunks = chunk.split(1 << 15)
    plan = AggPlan(types_of(sc), [0], [AggFunc(P.AGG_FIRSTROW, 0), xf(P.AGG_SUM, 1, 2, 4), AggFunc(P.AGG_COUNT, -1),
                                       xf(P.AGG_AVG, 3, 4, 9, X.MUL_CSUB, 1)], expected_groups=5000)
    rows, _ = T.run_host(plan, chunks, page=37)          # 37-row pages: cells and bitmaps start inside a byte
    assert check(plan, vals, rows) > 5000
    lib = abi.load_lib()
    e = HashAggExec(plan, MockDataSource(plan.col_types, chunks))
    e.open()
    try:
        e.next(8)
        nrows = C.c_int64(0)
        cols = (C.c_void_p * 4)(); nulls = (C.c_void_p * 4)()
        abi.check(lib.tg_agg_result_dev(e._h, C.byref(nrows), cols, nulls))
        m = nrows.value
        keys = np.zeros(m, dtype=np.int64)
        abi.check(lib.tg_memcpy_d2h(0, C.c_void_p(keys.ctypes.data), C.c_void_p(cols[0]), C.c_size_t(m * 8)))
        knb = np.zeros((m + 7) // 8, dtype=np.uint8)
        abi.check(lib.tg_memcpy_d2h(0, C.c_void_p(knb.ctypes.data), C.c_void_p(nulls[0]), C.c_size_t(len(knb))))
        kn = unpack_nulls(knb, m)
        exp = expected(plan, vals)
        for k in (1, 3):
            host = np.zeros((m, 40), dtype=np.uint8)
            abi.check(lib.tg_memcpy_d2h(0, C.c_void_p(host.ctypes.data), C.c_void_p(cols[k]), C.c_size_t(m * 40)))
            nb = np.zeros((m + 7) // 8, dtype=np.uint8)
            abi.check(lib.tg_memcpy_d2h(0, C.c_void_p(nb.ctypes.data), C.c_void_p(nulls[k]), C.c_size_t(len(nb))))
            sn = unpack_nulls(nb, m)
            for r in range(m):
                key = (None if kn[r] else int(keys[r]),)
                assert (None if sn[r] else bytes(host[r])) == exp[key][k], (key, k)
    finally:
        e.close()


def test_bad_cell_in_the_second_operand_fails_the_push():
    import torch
    sc = SCALES[5]
    rng = np.random.default_rng(100)
    good_chunk, good_vals = make_rows(rng, 20_000, 300, sc)
    bad_chunk, _ = make_rows(rng, 20_000, 300, sc)
    cells = bad_chunk.columns[4].data.copy()
    cells[11, 1] = 3                                       # digitsFrac 3 in a DECIMAL(15, 2) column
    bad_chunk = Chunk(bad_chunk.columns[:4] + [Column(cells)] + bad_chunk.columns[5:])
    plan = plans(sc, local=False)[-1]
    lib = abi.load_lib()
    e = HashAggExec(plan, MockDataSource(plan.col_types, []))
    e.open()
    try:
        chk, keep = T.dev_columns(good_chunk)
        abi.check(lib.tg_agg_push_dev(e._h, C.byref(chk)))
        chk, keep2 = T.dev_columns(bad_chunk)
        assert lib.tg_agg_push_dev(e._h, C.byref(chk)) == abi.TG_ERR_INVALID
        assert b"column 4" in lib.tg_last_error(), lib.tg_last_error()
        abi.check(lib.tg_agg_finish(e._h))
        e._prepared = True
        rows = []
        while True:
            c = e.next(1 << 20)
            if c.num_rows() == 0:
                break
            rows.extend(T.rows_of(c))
        check(plan, good_vals, rows)                       # the table holds the good rows only
    finally:
        e.close()
    torch.cuda.synchronize()


# ---- TPC-H shapes and scale ----------------------------------------------------------------------------------------
def _price_disc(rng, n):
    price = rng.integers(90_000, 10_500_000, n, dtype=np.int64)   # l_extendedprice 900.00 .. 105000.00
    disc = rng.integers(0, 11, n, dtype=np.int64)                 # l_discount 0.00 .. 0.10
    return price, disc


def test_q3_shape_three_group_columns():
    # GROUP BY l_orderkey, o_orderdate, o_shippriority; FIRSTROW x 3; SUM(l_extendedprice * (1 - l_discount)), DECIMAL(15,2)
    rng = np.random.default_rng(120)
    n = 1_500_000
    ok = rng.integers(0, 600_000, n, dtype=np.int64)
    od = (ok * 7919) % 2400 + 8000
    sp = np.zeros(n, dtype=np.int64)
    price, disc = _price_disc(rng, n)
    dt = FieldType(DEC, abi.FLAG_NOT_NULL, 15, 2)
    z = np.zeros(n, dtype=bool)
    cells = lambda v: A.cells_np(v, 15, 2, np.full(n, 13), np.zeros(n, dtype=np.int64), v < 0)
    chunk = Chunk([Column(ok), Column(od), Column(sp), Column(cells(price)), Column(cells(disc))])
    plan = AggPlan([INT_NN, INT_NN, INT_NN, dt, dt], [0, 1, 2], [AggFunc(P.AGG_FIRSTROW, g) for g in (0, 1, 2)] +
                   [xf(P.AGG_SUM, 3, 4, 4, X.MUL_CSUB, 1)])
    vals = {0: (ok, z), 1: (od, z), 2: (sp, z), 3: (price, z), 4: (disc, z)}
    rows, st = T.run_host(plan, chunk.split(1 << 20))
    assert st.paths & P.AGG_PATH_MULTI_KEY
    inv, tuples = T._group_ids(plan, vals)
    sums, cnt = X.group_sums(price * (100 - disc), np.ones(n, dtype=bool), inv, len(tuples))   # < 2^63: int64 is exact
    want = {t: X.sum_result(sums[j], 4) for j, t in enumerate(tuples)}
    assert len(rows) == len(want)
    for r in rows:
        assert r[3] == want[tuple(r[:3])], r[:3]


def test_full_scale_100m_rows_1m_groups():
    # SUM(price * (1 - disc)) over DECIMAL(15,2) and COUNT on 100 M device-resident rows in 1 M groups; the cells are built on
    # the device in FromBin's form; the group sums stay below 2^63, so an int64 index_add is exact
    import torch
    from tidb_b200.device import DeviceAgg
    n, G = 100_000_000, 1_000_000
    gen = torch.Generator(device="cuda").manual_seed(22)
    keys = torch.randint(0, G, (n,), device="cuda", dtype=torch.int64, generator=gen)

    def cells(v):
        w = torch.zeros((n, 10), dtype=torch.int32, device="cuda")
        w[:, 0] = 13 | (2 << 8)
        w[:, 1] = (v // 100 // 10 ** 9).to(torch.int32)
        w[:, 2] = (v // 100 % 10 ** 9).to(torch.int32)
        w[:, 3] = ((v % 100) * 10 ** 7).to(torch.int32)
        return w.view(torch.uint8).view(n, 40)

    price = torch.randint(90_000, 10_500_000, (n,), device="cuda", dtype=torch.int64, generator=gen)
    disc = torch.randint(0, 11, (n,), device="cuda", dtype=torch.int64, generator=gen)
    pc, dc = cells(price), cells(disc)
    want = torch.zeros(G, dtype=torch.int64, device="cuda").index_add_(0, keys, price * (100 - disc))
    del price, disc
    torch.cuda.synchronize()   # the aggregation reads its input on a stream of its own: it must be written first
    dt = FieldType(DEC, abi.FLAG_NOT_NULL, 15, 2)
    plan = AggPlan([INT_NN, dt, dt], [0], [AggFunc(P.AGG_FIRSTROW, 0), xf(P.AGG_SUM, 1, 2, 4, X.MUL_CSUB, 1), AggFunc(P.AGG_COUNT, -1)],
                   expected_groups=G)
    agg = DeviceAgg(plan)
    try:
        agg.push([keys, pc, dc])
        rows, cols, _ = agg.finish()
        assert rows == G
        k = np.zeros(rows, dtype=np.int64)
        out = np.zeros((rows, 40), dtype=np.uint8)
        cnt = np.zeros(rows, dtype=np.int64)
        lib = abi.load_lib()
        for dst, src in ((k, cols[0]), (out, cols[1]), (cnt, cols[2])):
            abi.check(lib.tg_memcpy_d2h(0, C.c_void_p(dst.ctypes.data), C.c_void_p(src), C.c_size_t(dst.nbytes)))
    finally:
        agg.close()
    del pc, dc
    want = want.cpu().numpy()[k]
    assert np.array_equal(cnt, torch.bincount(keys, minlength=G).cpu().numpy()[k])
    c = out.view(np.int32).astype(np.int64)
    hdr = c[:, 0]
    assert ((hdr & 0xFF) == 9).all() and (((hdr >> 8) & 0xFFFF) == (4 | (4 << 8))).all() and ((hdr >> 24) == 0).all()
    assert (c[:, 2] % 10 ** 5 == 0).all()                   # one fraction word: 4 digits, left-aligned
    assert np.array_equal(c[:, 1] * 10 ** 4 + c[:, 2] // 10 ** 5, want)
    for r in np.random.default_rng(0).integers(0, G, 200):   # spot checks through the codec
        assert bytes(out[r]) == X.sum_result(int(want[r]), 4)
