"""The hash join's general count -> scan -> write path and its row-store (mode G) tables, against the exact reference of
tests/join_reference.py: every join type at scale, probe calls split into 16 M-row sub-batches, constructed collisions of the
multi-column candidate key, FLOAT (4-byte) keys and payloads, linear-probe runs that wrap past the last slot or start on an
odd slot, the INT64_MIN key's side slot under the build-side scan, and mixed-signedness keys at full range.  Every output
row is compared (integers bit-exact, FLOAT / DOUBLE / DECIMAL cells by their bits, NULL != 0), and tg_join_stats shows which
kernel families and which table mode ran."""
import numpy as np
import pytest

import join_keys as K
from join_reference import assert_same_rows, join_reference
from test_join_reference import F32_POOL, F64_EXTRA, needs_build_scan
from test_join_slice_sizing import table_slots
from test_oracle_join import JOIN_TYPES
from tidb_b200 import abi
from tidb_b200.chunk import Chunk, Column, pack_not_null_bitmap, unpack_nulls
from tidb_b200.executor import HashJoinExec, MockDataSource, np_dtype_of
from tidb_b200.plan import FieldType, FilterItem, JoinPlan, OtherCond

pytestmark = pytest.mark.gpu

INT = FieldType(abi.TYPE_LONGLONG, 0)
INT_NN = FieldType(abi.TYPE_LONGLONG, abi.FLAG_NOT_NULL)
UINT = FieldType(abi.TYPE_LONGLONG, abi.FLAG_UNSIGNED)
FLT = FieldType(abi.TYPE_FLOAT, 0)
FLT_NN = FieldType(abi.TYPE_FLOAT, abi.FLAG_NOT_NULL)
DBL = FieldType(abi.TYPE_DOUBLE, 0)
DEC = FieldType(abi.TYPE_NEWDECIMAL, 0, 15, 2)
GENERAL, UQ = abi.JOIN_PATH_PROBE_GENERAL, abi.JOIN_PATH_PROBE_UQ
PROBE_ENV = ("TG_PROBE_PARTITION", "TG_PROBE_PARTS", "TG_PROBE_PART_MIN_MB", "TG_PROBE_PART_MIN_ROWS", "TG_PROBE_UQ", "TG_PROBE_INPLACE")
H100_L2 = 50 << 20
SENTINEL = K.SENTINEL


@pytest.fixture(autouse=True)
def _default_probe(monkeypatch):
    for k in PROBE_ENV:
        monkeypatch.delenv(k, raising=False)


def type_cases():
    """every join type x both build sides NewJoinProbe allows"""
    return [(jt, brt) for jt in JOIN_TYPES for brt in (True, False)
            if brt or jt not in (abi.JOIN_LEFT_OUTER_SEMI, abi.JOIN_ANTI_LEFT_OUTER_SEMI)]


# ---- chunks in, columns out ------------------------------------------------------------------------------------------
def make_chunks(cols, nulls, rows, rng=None, keep=None):
    """cut columns into chunks of `rows` physical rows; keep = fraction of each chunk's rows a sel vector keeps (None = no
    sel).  -> (chunks, the physical row of every logical row)"""
    n = len(cols[0])
    out, logical = [], []
    for lo in range(0, n, rows):
        hi = min(n, lo + rows)
        ch = Chunk([Column(c[lo:hi], None if nl is None else nl[lo:hi]) for c, nl in zip(cols, nulls)])
        if keep is not None:
            ch.sel = np.nonzero(rng.random(hi - lo) < keep)[0].astype(np.int64)
            logical.append(ch.sel + lo)
        else:
            logical.append(np.arange(lo, hi, dtype=np.int64))
        out.append(ch)
    return out, (np.concatenate(logical) if logical else np.zeros(0, np.int64))


def flat(cols, nulls, idx=None):
    """(values, nulls) columns of the logical rows idx (None = all)"""
    out = []
    for c, nl in zip(cols, nulls):
        nl = np.zeros(len(c), dtype=bool) if nl is None else nl
        out.append((c, nl) if idx is None else (c[idx], nl[idx]))
    return out


def run_host(plan, left, right, required_rows=1_000_003):
    """HashJoinExec over chunk lists; -> ((values, nulls) per output column, tg_join_stats)"""
    e = HashJoinExec(plan, MockDataSource(plan.left_types, left), MockDataSource(plan.right_types, right))
    e.open()
    parts = [[] for _ in plan.out_schema()]
    try:
        while True:
            c = e.next(required_rows)
            n = c.num_rows()
            if n == 0:
                break
            assert n <= required_rows
            for i, col in enumerate(c.columns):
                parts[i].append((col.data, col.nulls()))
        st = e.stats()
    finally:
        e.close()
    out = []
    for t, p in zip(plan.out_schema(), parts):
        dt = np.dtype(np_dtype_of(t))
        if not p:
            out.append((np.zeros((0,) + dt.shape, dtype=dt.base), np.zeros(0, dtype=bool)))
        else:
            out.append((np.concatenate([v for v, _ in p]), np.concatenate([nl for _, nl in p])))
    return out, st


def check(want, got, st, paths=GENERAL, mode=None, what=""):
    assert_same_rows(want, got, what)
    assert st.paths & paths == paths, (what, hex(st.paths))
    if mode is not None:
        assert st.table_mode == mode, (what, st.table_mode)


def sides(brt, probe, build):
    """(left, right) of a plan whose probe / build sides are given"""
    return (probe, build) if brt else (build, probe)


# ---- 1. every join type at scale on a G table -------------------------------------------------------------------------
@pytest.fixture(scope="module")
def scale_data():
    """~2.5 M build rows over 600 K distinct keys (duplicate counts 1-64, one key with 100 K rows, INT64_MIN 7 times), 5 M
    probe rows; 5 % NULL keys, nullable payloads, a filter column on each side"""
    rng = np.random.default_rng(2024)
    keys = np.unique(rng.integers(-(1 << 62), 1 << 62, 620_000))[:600_001]
    keys = rng.permutation(keys)
    hot = keys[0]
    cnt = np.where(rng.random(len(keys)) < 0.05, rng.integers(1, 65, len(keys)), rng.integers(1, 5, len(keys)))
    cnt[0] = 100_000
    keys[1], cnt[1] = SENTINEL, 7
    bk = rng.permutation(np.repeat(keys, cnt))
    nb = len(bk)
    b_cols = [bk, rng.integers(-1 << 40, 1 << 40, nb), rng.integers(0, 100, nb)]
    b_nulls = [rng.random(nb) < 0.05, rng.random(nb) < 0.1, None]
    npr = 5_000_000
    pk = rng.integers(-(1 << 62), 1 << 62, npr)                    # misses (a hit among them is harmless: the reference sees it)
    hit = rng.random(npr) < 0.25
    pk[hit] = keys[rng.integers(2, len(keys), int(hit.sum()))]
    pk[rng.choice(npr, 3, replace=False)] = hot
    pk[rng.choice(npr, 50, replace=False)] = SENTINEL
    p_cols = [np.arange(npr, dtype=np.int64), pk, rng.integers(-1 << 40, 1 << 40, npr), rng.integers(0, 100, npr)]
    p_nulls = [None, rng.random(npr) < 0.05, rng.random(npr) < 0.1, None]
    return (b_cols, b_nulls), (p_cols, p_nulls)


@pytest.mark.parametrize("jt,brt", type_cases())
def test_every_join_type_at_scale_on_a_row_store_table(jt, brt, scale_data):
    (b_cols, b_nulls), (p_cols, p_nulls) = scale_data
    rng = np.random.default_rng(jt * 2 + int(brt))
    if brt:   # probe: 1024-row chunks with sel vectors (host staging); build: 64 K-row chunks
        probe, pidx = make_chunks(p_cols, p_nulls, 1024, rng, keep=0.7)
        build, bidx = make_chunks(b_cols, b_nulls, 1 << 16)
    else:     # probe: 256 K-row chunks (copied straight to the device); build: 1024-row chunks with sel vectors
        probe, pidx = make_chunks(p_cols, p_nulls, 1 << 18)
        build, bidx = make_chunks(b_cols, b_nulls, 1024, rng, keep=0.8)
    ptypes, btypes = [INT_NN, INT, INT, INT_NN], [INT, INT, INT_NN]
    semi = jt >= abi.JOIN_SEMI
    ltypes, rtypes = sides(brt, ptypes, btypes)
    lk, rk = sides(brt, [1], [0])
    plan = JoinPlan(jt, ltypes, rtypes, lk, rk, build_is_right=brt, lused=list(range(len(ltypes))), rused=[] if semi else list(range(len(rtypes))),
                    probe_filter=[FilterItem(abi.CMP_GE, 3, const_i64=10)], build_filter=[FilterItem(abi.CMP_LT, 2, const_i64=90)])
    L, R = sides(brt, flat(p_cols, p_nulls, pidx), flat(b_cols, b_nulls, bidx))
    want = join_reference(plan, L, R, flat=True)
    got, st = run_host(plan, *sides(brt, probe, build))
    check(want, got, st, GENERAL, 2, f"jt={jt} brt={brt}")
    if needs_build_scan(jt, brt):
        # the build-side scan wrote rows whose probe-side cells are all NULL (semi / anti: every output row is a build row)
        rowid = 0 if brt else len(ltypes)
        scanned = int(want[rowid][1].sum()) if jt in (abi.JOIN_LEFT_OUTER, abi.JOIN_RIGHT_OUTER) else len(want[0][0])
        assert scanned > 1000


# ---- 2. sub-batches of one general-path call -----------------------------------------------------------------------------
NSUB = (1 << 24) + 4105
PLANT = [(1 << 24) - 1, 1 << 24, (1 << 24) + 1]


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def run_dev(plan, b_cols, b_nulls, p_cols, p_nulls):
    """build and probe through tg_join_build_push_dev / tg_join_probe_dev (one general-path call over every probe row)"""
    import torch
    from tidb_b200.device import DeviceJoin, fetch_device
    bt = [_dev(c) for c in b_cols]
    bn = [None if x is None else _dev(pack_not_null_bitmap(x)) for x in b_nulls]
    pt = [_dev(c) for c in p_cols]
    pn = [None if x is None else _dev(pack_not_null_bitmap(x)) for x in p_nulls]
    torch.cuda.synchronize()
    j = DeviceJoin(plan)
    try:
        j.build(bt, bn)
        rows, cols, nulls = j.probe(pt, pn)
        st = j.stats()
        out = []
        for t, p, q in zip(plan.out_schema(), cols, nulls):
            dt = np.dtype(np_dtype_of(t))
            raw = fetch_device(p, rows * dt.itemsize)
            v = raw.reshape(rows, 40) if dt.shape else raw.view(dt)
            nl = unpack_nulls(fetch_device(q, (rows + 7) // 8), rows) if q else np.zeros(rows, dtype=bool)
            out.append((v, nl))
    finally:
        j.close()
    return out, st


def sub_batch_want(kind):
    """(case, reference result)"""
    case = sub_batch_case(kind)
    plan, b_cols, b_nulls, p_cols, p_nulls = case
    return case, join_reference(plan, flat(p_cols, p_nulls), flat(b_cols, b_nulls), flat=True)


@pytest.fixture(scope="module")
def outer_sub_batch_case():
    """the left outer case, shared by the device-input and the host-push test"""
    return sub_batch_want("outer")


def sub_batch_case(kind):
    rng = np.random.default_rng(77)
    n = NSUB
    rowid = np.arange(n, dtype=np.int64)
    if kind == "multikey":
        bt = rng.integers(0, 1 << 20, (200_000, 3))
        pick = rng.random(n) < 0.5
        pt = rng.integers(0, 1 << 20, (n, 3))
        pt[pick] = bt[rng.integers(0, len(bt), int(pick.sum()))]
        b_cols = [bt[:, 0], bt[:, 1], bt[:, 2], rng.integers(0, 1000, len(bt))]
        b_nulls = [None, rng.random(len(bt)) < 0.02, None, None]
        pn1 = rng.random(n) < 0.05
        pn1[PLANT] = True
        pn1[:2] = False
        p_cols = [rowid, pt[:, 0], pt[:, 1], pt[:, 2], rng.integers(0, 1000, n)]
        p_nulls = [None, pn1, None, None, None]
        plan = JoinPlan(abi.JOIN_INNER, [INT_NN, INT, INT, INT, INT], [INT, INT, INT, INT], [1, 2, 3], [0, 1, 2], lused=[0, 1, 4], rused=[3, 1],
                        other_cond=[OtherCond(abi.CMP_LE, 0, 4, 1, 3)])
        return plan, b_cols, b_nulls, p_cols, p_nulls
    dup = kind == "decimal"
    bk = rng.permutation(1 << 22)[:100_000].astype(np.int64) * 7 + 1
    if dup:
        bk = np.repeat(bk, rng.integers(1, 4, len(bk)))
    nb = len(bk)
    pk = rng.integers(0, 7 << 22, n).astype(np.int64)
    hit = rng.random(n) < (0.1 if dup else 0.5)
    pk[hit] = bk[rng.integers(0, nb, int(hit.sum()))]
    pkn = rng.random(n) < 0.05
    pkn[PLANT] = True
    pkn[:2] = False
    if kind == "outer":
        ppn = rng.random(n) < 0.1
        ppn[PLANT] = True
        ppn[:2] = False
        b_cols, b_nulls = [bk, rng.integers(-1 << 40, 1 << 40, nb)], [None, rng.random(nb) < 0.2]
        p_cols, p_nulls = [rowid, pk, rng.integers(-1 << 40, 1 << 40, n)], [None, pkn, ppn]
        plan = JoinPlan(abi.JOIN_LEFT_OUTER, [INT_NN, INT, INT], [INT, INT], [1], [0], lused=[0, 1, 2], rused=[1])
    elif kind == "anti":
        b_cols, b_nulls = [bk], [None]
        p_cols, p_nulls = [rowid, pk, rng.integers(0, 100, n)], [None, pkn, None]
        plan = JoinPlan(abi.JOIN_ANTI_SEMI, [INT_NN, INT, INT_NN], [INT_NN], [1], [0], lused=[0, 1], rused=[],
                        probe_filter=[FilterItem(abi.CMP_LT, 2, const_i64=80)])
    else:     # duplicated build keys, a DECIMAL probe payload: its row ids are offset by the sub-batch start as well
        cells = rng.integers(0, 256, (n, 40), dtype=np.uint8)
        dn = rng.random(n) < 0.05
        dn[PLANT] = True
        dn[:2] = False
        b_cols, b_nulls = [bk, np.arange(nb, dtype=np.int64)], [None, None]
        p_cols, p_nulls = [rowid, pk, cells], [None, pkn, dn]
        plan = JoinPlan(abi.JOIN_INNER, [INT_NN, INT, DEC], [INT_NN, INT_NN], [1], [0], lused=[0, 2], rused=[1])
    return plan, b_cols, b_nulls, p_cols, p_nulls


@pytest.mark.parametrize("kind", ["outer", "anti", "multikey", "decimal"])
def test_general_probe_sub_batches(kind, request):
    # 2^24 + 4105 probe rows in one call: the second sub-batch starts at row 2^24 with a tail that is not a multiple of 8, its
    # data, NULL-bitmap, composite-key and row-id views offset; NULLs are planted at rows 2^24 - 1, 2^24 and 2^24 + 1
    (plan, b_cols, b_nulls, p_cols, p_nulls), want = request.getfixturevalue("outer_sub_batch_case") if kind == "outer" else sub_batch_want(kind)
    got, st = run_dev(plan, b_cols, b_nulls, p_cols, p_nulls)
    check(want, got, st, GENERAL, 2 if kind in ("multikey", "decimal", "outer") else None, kind)
    assert st.probe_rows == NSUB
    rows = got[0][0]
    if kind == "outer":
        for r in PLANT:      # a NULL probe key is padded once, its NULL payload stays NULL
            at = np.nonzero(rows == r)[0]
            assert len(at) == 1 and got[1][1][at[0]] and got[2][1][at[0]] and got[3][1][at[0]]
    elif kind == "anti":
        assert set(PLANT) <= set(rows.tolist())            # no key: an anti join result
    else:
        assert not set(PLANT) & set(rows.tolist())          # no key: never an inner join result


def test_general_probe_sub_batches_host_push(outer_sub_batch_case):
    # the same left outer join as one host push of the whole chunk (copied straight to the device, one probe call)
    (plan, b_cols, b_nulls, p_cols, p_nulls), want = outer_sub_batch_case
    probe = [Chunk([Column(c, nl) for c, nl in zip(p_cols, p_nulls)])]
    build, _ = make_chunks(b_cols, b_nulls, 1 << 16)
    got, st = run_host(plan, probe, build, required_rows=(1 << 22) + 3)
    check(want, got, st, GENERAL, 2, "host push")
    for r in PLANT:
        at = np.nonzero(got[0][0] == r)[0]
        assert len(at) == 1 and got[1][1][at[0]] and got[2][1][at[0]] and got[3][1][at[0]]


# ---- 3. constructed collisions of the multi-column candidate key ---------------------------------------------------------
COLLISION_TYPES = [(abi.JOIN_INNER, True), (abi.JOIN_LEFT_OUTER, True), (abi.JOIN_RIGHT_OUTER, False), (abi.JOIN_SEMI, True),
                   (abi.JOIN_ANTI_SEMI, True)]


@pytest.mark.parametrize("ncols", [2, 3, 4])
@pytest.mark.parametrize("jt,brt", COLLISION_TYPES)
def test_composite_key_collisions(ncols, jt, brt):
    # ~30 % of the probe tuples differ from a build tuple but share its candidate key: the residual key equalities must reject
    # every such pair, so an outer probe row whose candidates all fail is padded once and an anti row is emitted.  The last key
    # column is UNSIGNED on the build side: a colliding probe tuple whose solved last column is negative has no key at all
    rng = np.random.default_rng(300 + ncols * 10 + jt)
    nbt = 5000
    bt = np.column_stack([rng.integers(-1000, 1000, (nbt, ncols - 1)), rng.integers(0, 1 << 40, nbt)]).astype(np.int64)
    bt = np.unique(bt, axis=0)
    brows = np.repeat(np.arange(len(bt)), rng.integers(1, 4, len(bt)))
    npr = 20_000
    src = rng.integers(0, len(bt), npr)
    pt = bt[src].copy()
    kind = rng.random(npr)
    coll = kind < 0.3
    for i in np.nonzero(coll)[0]:
        pt[i] = K.colliding_keys(tuple(int(x) for x in pt[i]), ncols, delta=int(rng.integers(1, 1 << 20)))
    miss = kind > 0.85
    pt[miss, 0] += 1 << 30
    pnull = [rng.random(npr) < 0.03 for _ in range(ncols)]
    b_cols = [bt[brows, c] for c in range(ncols)] + [np.arange(len(brows), dtype=np.int64)]
    b_nulls = [None] * ncols + [None]
    p_cols = [np.arange(npr, dtype=np.int64)] + [pt[:, c] for c in range(ncols)]
    p_nulls = [None] + pnull
    btypes = [INT] * (ncols - 1) + [UINT, INT_NN]
    ptypes = [INT_NN] + [INT] * ncols
    semi = jt >= abi.JOIN_SEMI
    ltypes, rtypes = sides(brt, ptypes, btypes)
    lk, rk = sides(brt, list(range(1, ncols + 1)), list(range(ncols)))
    plan = JoinPlan(jt, ltypes, rtypes, lk, rk, build_is_right=brt, lused=list(range(len(ltypes))), rused=[] if semi else list(range(len(rtypes))))
    pc, bc = make_chunks(p_cols, p_nulls, 1024)[0], make_chunks(b_cols, b_nulls, 1024)[0]
    want = join_reference(plan, *sides(brt, flat(p_cols, p_nulls), flat(b_cols, b_nulls)), flat=True)
    got, st = run_host(plan, *sides(brt, pc, bc), required_rows=4099)
    check(want, got, st, GENERAL, 2, f"ncols={ncols} jt={jt}")
    # the collisions are real: colliding probe rows with every key non-NULL and a non-negative last column reach the
    # candidate stage, and a fair share of them exist
    live = coll & ~np.any(np.column_stack(pnull), axis=1) & (pt[:, -1] >= 0)
    assert live.sum() > 0.1 * npr
    cand = {K.candidate_key(tuple(int(x) for x in r)) for r in bt}
    assert all(K.candidate_key(tuple(int(x) for x in pt[i])) in cand for i in np.nonzero(live)[0][:200])


# ---- 4. FLOAT (4-byte) columns --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rtype", ["float", "double"])
@pytest.mark.parametrize("jt,brt", [(abi.JOIN_INNER, True), (abi.JOIN_INNER, False), (abi.JOIN_LEFT_OUTER, True),
                                    (abi.JOIN_ANTI_SEMI, True), (abi.JOIN_RIGHT_OUTER, True)])
def test_float_keys(rtype, jt, brt):
    # a FLOAT key compares as float64(f32): -0.0f = 0.0, 0.1f != 0.1 (= float64(0.1f)), 0.5f = 0.5, +-FLT_MAX, subnormals, +-inf
    rng = np.random.default_rng(41 + jt + 2 * int(brt))
    nl, nr = 3000, 4000
    lk = F32_POOL[rng.integers(0, len(F32_POOL), nl)]
    if rtype == "float":
        rk, rt = F32_POOL[rng.integers(0, len(F32_POOL), nr)], FLT
    else:
        pool = np.concatenate([F32_POOL.astype(np.float64), F64_EXTRA])
        rk, rt = pool[rng.integers(0, len(pool), nr)], DBL
    l_cols = [np.arange(nl, dtype=np.int64), lk, rng.random(nl).astype(np.float32)]
    l_nulls = [None, rng.random(nl) < 0.05, rng.random(nl) < 0.1]
    r_cols = [rk, np.arange(nr, dtype=np.int64) * 3]
    r_nulls = [rng.random(nr) < 0.05, None]
    semi = jt >= abi.JOIN_SEMI
    plan = JoinPlan(jt, [INT_NN, FLT, FLT], [rt, INT_NN], [1], [0], build_is_right=brt, lused=[0, 1, 2], rused=[] if semi else [0, 1])
    lc, rc = make_chunks(l_cols, l_nulls, 1024, rng, keep=0.8)[0], make_chunks(r_cols, r_nulls, 700)[0]
    want = join_reference(plan, lc, rc)
    got, st = run_host(plan, lc, rc, required_rows=1 << 16)
    check(want, got, st, GENERAL, 2, "float keys")
    # the special values really meet: -0.0f finds +0.0 and 0.5f finds 0.5
    if jt == abi.JOIN_INNER:
        lv, rv = got[1][0], got[3][0]
        assert np.any(np.signbit(lv) & (lv == 0) & ~np.signbit(rv)) and np.any(lv == 0.5)


@pytest.mark.parametrize("jt,brt", type_cases())
def test_float_payloads_every_join_type(jt, brt):
    # 4-byte payload columns on both sides, NULLs and sel vectors: the 4-byte sel gather, row-store words, probe writes and
    # build-side scan cells
    rng = np.random.default_rng(500 + jt * 2 + int(brt))
    nl, nr = 20_000, 12_000
    l_cols = [np.arange(nl, dtype=np.int64), rng.integers(-300, 300, nl).astype(np.int64), (rng.standard_normal(nl) * 1e3).astype(np.float32)]
    l_nulls = [None, rng.random(nl) < 0.05, rng.random(nl) < 0.15]
    r_cols = [rng.integers(-300, 300, nr).astype(np.int64), (rng.standard_normal(nr) * 1e-3).astype(np.float32), rng.integers(0, 1 << 40, nr).astype(np.int64)]
    r_nulls = [rng.random(nr) < 0.05, rng.random(nr) < 0.15, None]
    r_cols[1][::97] = np.float32(-0.0)
    semi = jt >= abi.JOIN_SEMI
    plan = JoinPlan(jt, [INT_NN, INT, FLT], [INT, FLT, INT_NN], [1], [0], build_is_right=brt, lused=[2, 0, 1], rused=[] if semi else [1, 2, 1])
    lc = make_chunks(l_cols, l_nulls, 1024, rng, keep=0.75)[0]
    rc = make_chunks(r_cols, r_nulls, 1024, rng, keep=0.75)[0]
    want = join_reference(plan, lc, rc)
    got, st = run_host(plan, lc, rc, required_rows=5003)
    check(want, got, st, GENERAL, 2, f"jt={jt} brt={brt}")
    assert got[0][0].dtype == np.float32


def test_float_key_unique_single_pass_and_float_payload_row_store():
    rng = np.random.default_rng(9)
    nb, npr = 50_000, 400_000
    bk = np.unique(rng.integers(-(1 << 22), 1 << 22, nb * 2).astype(np.float32) / np.float32(64))[:nb]
    bk = rng.permutation(bk)
    bk[0] = np.float32(0.0)
    nb = len(bk)
    pk = np.where(rng.random(npr) < 0.6, bk[rng.integers(0, nb, npr)], np.float32(1e30)).astype(np.float32)
    pk[:10] = np.float32(-0.0)
    pkn = rng.random(npr) < 0.05
    probe = [Chunk([Column(pk, pkn), Column(np.arange(npr, dtype=np.int64))])]
    # (a) a FLOAT key that is not output, an 8-byte NOT NULL payload: the unique-key single-pass kernel (load_key KEY_F32)
    build = [Chunk([Column(bk), Column(np.arange(nb, dtype=np.int64) * 5)])]
    plan = JoinPlan(abi.JOIN_INNER, [FLT, INT_NN], [FLT_NN, INT_NN], [0], [0], lused=[1], rused=[1])
    got, st = run_host(plan, probe, build, required_rows=1 << 20)
    check(join_reference(plan, probe, build), got, st, UQ, 1, "uq")
    assert not st.paths & GENERAL and len(got[0][0]) > 200_000
    assert np.any(got[0][0] < 10)                       # the -0.0f probe keys found the +0.0f build key
    # (b) a FLOAT payload forces the row store (mode G) although every key is unique
    build = [Chunk([Column(bk), Column((np.arange(nb) * 0.25).astype(np.float32)), Column(np.arange(nb, dtype=np.int64))])]
    plan = JoinPlan(abi.JOIN_INNER, [FLT, INT_NN], [FLT_NN, FLT_NN, INT_NN], [0], [0], lused=[1, 0], rused=[1, 0])
    got, st = run_host(plan, probe, build, required_rows=1 << 20)
    check(join_reference(plan, probe, build), got, st, GENERAL, 2, "float payload")


@pytest.mark.parametrize("required_rows", [1, 3, 13])
def test_small_next_windows_over_float_columns(required_rows):
    rng = np.random.default_rng(required_rows)
    nl, nr = 150, 120
    l_cols = [rng.integers(-20, 20, nl).astype(np.int64), rng.random(nl).astype(np.float32)]
    l_nulls = [rng.random(nl) < 0.1, rng.random(nl) < 0.2]
    r_cols = [rng.integers(-20, 20, nr).astype(np.int64), rng.random(nr).astype(np.float32)]
    r_nulls = [rng.random(nr) < 0.1, rng.random(nr) < 0.2]
    for jt, brt in ((abi.JOIN_LEFT_OUTER, True), (abi.JOIN_LEFT_OUTER, False)):
        plan = JoinPlan(jt, [INT, FLT], [INT, FLT], [0], [0], build_is_right=brt)
        lc, rc = make_chunks(l_cols, l_nulls, 64, rng, keep=0.7)[0], make_chunks(r_cols, r_nulls, 50)[0]
        got, st = run_host(plan, lc, rc, required_rows=required_rows)
        check(join_reference(plan, lc, rc), got, st, GENERAL, 2, "small next")


# ---- 5. row-store runs: wrapped, odd-started, misses inside them, the sentinel's side slot ---------------------------------
def run_keys(nslots):
    """build keys: 64 distinct keys homed on the last two homes (their run wraps to slot 0), 5 keys homed on the home below a
    middle home H and 40 homed at H (the 5 fill H - 4 .. H, so the run of the 40 starts on the odd slot H + 1 unless a filler
    key got there first), and INT64_MIN.  Probe: those keys, and misses homed inside both clusters and in the wrapped part."""
    last = nslots - K.HOME_WIDTH
    wrap = [K.key_with_home(last - K.HOME_WIDTH * (i % 2), nslots, salt=1000 + i) for i in range(64)]
    H = (nslots // 2) & ~(K.HOME_WIDTH - 1)
    below = [K.key_with_home(H - K.HOME_WIDTH, nslots, salt=2000 + i) for i in range(5)]
    odd = [K.key_with_home(H, nslots, salt=3000 + i) for i in range(40)]
    cluster = np.array(wrap + below + odd + [SENTINEL], dtype=np.int64)
    misses = np.array([K.key_with_home(h, nslots, salt=9000 + i) for i, h in
                       enumerate([last, last - 4, H, H - 4, 0, 4, 8] * 6)], dtype=np.int64)
    return cluster, misses


@pytest.mark.parametrize("jt,brt", type_cases())
def test_row_store_runs_wrap_and_start_odd(jt, brt):
    rng = np.random.default_rng(800 + jt * 2 + int(brt))
    nb = 18_000
    nslots = table_slots(nb, H100_L2, load_factor=0.9)
    cluster, misses = run_keys(nslots)
    cdup = np.repeat(cluster, rng.integers(1, 6, len(cluster)))
    filler = rng.integers(-(1 << 62), 1 << 62, nb - len(cdup)) // 4 * 4   # filler keys repeat too
    filler = filler[rng.integers(0, len(filler), len(filler))]
    bk = rng.permutation(np.concatenate([cdup, filler]))
    b_cols, b_nulls = [bk, np.arange(nb, dtype=np.int64)], [rng.random(nb) < 0.02, rng.random(nb) < 0.1]
    npr = 30_000
    pk = np.concatenate([np.repeat(cluster, 20), np.repeat(misses, 10), filler[rng.integers(0, len(filler), npr)]])[:npr]
    pk[-5000:] = rng.integers(0, 1 << 40, 5000) * 4 + 1
    pk = rng.permutation(pk)
    p_cols, p_nulls = [np.arange(npr, dtype=np.int64), pk], [None, rng.random(npr) < 0.02]
    semi = jt >= abi.JOIN_SEMI
    ltypes, rtypes = sides(brt, [INT_NN, INT], [INT, INT])
    lk, rk = sides(brt, [1], [0])
    plan = JoinPlan(jt, ltypes, rtypes, lk, rk, build_is_right=brt, lused=[0, 1], rused=[] if semi else [0, 1], load_factor=0.9)
    pc, bc = make_chunks(p_cols, p_nulls, 4096)[0], make_chunks(b_cols, b_nulls, 4096)[0]
    want = join_reference(plan, *sides(brt, flat(p_cols, p_nulls), flat(b_cols, b_nulls)), flat=True)
    got, st = run_host(plan, *sides(brt, pc, bc), required_rows=7777)
    assert st.table_slots == nslots
    check(want, got, st, GENERAL, 2, f"jt={jt} brt={brt}")


@pytest.mark.parametrize("path,env,bit", [
    ("direct", dict(TG_PROBE_PARTITION="0"), abi.JOIN_PATH_PROBE_DIRECT),
    ("lean segment", dict(TG_PROBE_INPLACE="0"), abi.JOIN_PATH_PROBE_SEG),
    ("in place", dict(TG_PROBE_INPLACE="1"), abi.JOIN_PATH_PROBE_SEG),
])
def test_unique_clusters_on_interior_slice_boundaries(path, env, bit, monkeypatch):
    # a U1 table sliced 8 ways, with a cluster of 24 keys on the last home below each interior slice boundary (its run
    # reaches into the next slice) and misses homed there too
    for k, v in dict(env, TG_PROBE_PARTS="8", TG_PROBE_PART_MIN_MB="0", TG_PROBE_PART_MIN_ROWS="0").items():
        monkeypatch.setenv(k, v)
    rng = np.random.default_rng(31)
    nb, npr, P = 300_000, 2_000_000, 8
    nslots = table_slots(nb, H100_L2, load_factor=0.9)
    homes = [K.home_slot((K.first_hi32_of_slice(p, P) - 1) << 32, nslots) for p in range(1, P)]
    cl = [K.key_with_home(h, nslots, salt=100 * p + i) for p, h in enumerate(homes) for i in range(24)]
    ms = [K.key_with_home(h, nslots, salt=50_000 + 100 * p + i) for p, h in enumerate(homes) for i in range(3)]
    filler = np.unique(rng.integers(-(1 << 62), 1 << 62, nb) * 2)
    filler = filler[~np.isin(filler, cl)][:nb - len(cl)]
    bk = rng.permutation(np.concatenate([np.array(cl, dtype=np.int64), filler]))
    assert len(bk) == nb
    pk = np.where(rng.random(npr) < 0.9, bk[rng.integers(0, nb, npr)], rng.integers(0, 1 << 40, npr) * 2 + 1)
    pk[:len(cl) * 4] = np.repeat(np.array(cl, dtype=np.int64), 4)
    pk[len(cl) * 4:len(cl) * 4 + len(ms)] = ms
    pk = rng.permutation(pk)
    probe = [Chunk([Column(pk), Column(np.arange(npr, dtype=np.int64))])]
    build = [Chunk([Column(bk), Column(np.arange(nb, dtype=np.int64) * 3 + 1)])]
    plan = JoinPlan(abi.JOIN_INNER, [INT_NN, INT_NN], [INT_NN, INT_NN], [0], [0], load_factor=0.9)
    got, st = run_host(plan, probe, build, required_rows=1 << 22)
    assert st.table_slots == nslots and st.table_mode == 1
    assert st.paths & bit and not st.paths & GENERAL, (path, hex(st.paths))
    assert_same_rows(join_reference(plan, probe, build), got, path)


# ---- 6. mixed signedness at full range ------------------------------------------------------------------------------------
@pytest.mark.parametrize("unsigned_left", [True, False])
@pytest.mark.parametrize("jt,brt", type_cases())
def test_mixed_signedness_full_range(unsigned_left, jt, brt):
    # unsigned keys in [2^63, 2^64) against signed keys with the same bits never match; equal non-negative values do.
    # Outer, anti and left outer semi joins turn the rejected rows into padded rows, anti rows and flag 0
    rng = np.random.default_rng(600 + jt * 4 + 2 * int(brt) + int(unsigned_left))
    nl, nr = 6000, 5000
    shared = np.concatenate([rng.integers(-(1 << 63), -1, 300), rng.integers(0, 1 << 62, 300), [-1, -(1 << 63), (1 << 63) - 1, 0]]).astype(np.int64)
    lk = shared[rng.integers(0, len(shared), nl)]
    rk = shared[rng.integers(0, len(shared), nr)]
    l_cols, l_nulls = [np.arange(nl, dtype=np.int64), lk], [None, rng.random(nl) < 0.03]
    r_cols, r_nulls = [rk, np.arange(nr, dtype=np.int64)], [rng.random(nr) < 0.03, None]
    U, S = (UINT, INT) if unsigned_left else (INT, UINT)
    semi = jt >= abi.JOIN_SEMI
    plan = JoinPlan(jt, [INT_NN, U], [S, INT_NN], [1], [0], build_is_right=brt, rused=[] if semi else None)
    lc, rc = make_chunks(l_cols, l_nulls, 1024)[0], make_chunks(r_cols, r_nulls, 1024)[0]
    want = join_reference(plan, lc, rc)
    got, st = run_host(plan, lc, rc, required_rows=3001)
    check(want, got, st, GENERAL, 2, f"jt={jt} brt={brt}")
    if jt == abi.JOIN_INNER:
        assert len(got[0][0]) > 0 and np.all(got[1][0] >= 0)      # only non-negative bit patterns ever match
