"""DECIMAL payload columns through the CUDA hash join: 40-byte MyDecimal cells are moved, never interpreted, on every join
type, build side, probe path and input route.  A non-NULL output cell must be byte-identical to its input cell (whatever
its bytes: random, negative zero, odd resultFrac), a cell under NULL is zero bytes, and the NULL bitmaps are exact.
Results are compared as sorted row multisets against the CPU oracle (oracle/join.cpp) or an index-gather reference, and
tg_join_stats.paths proves which probe path carried the cells."""
import ctypes as C

import numpy as np
import pytest

import mydecimal_args as A
import oracle_lib as O
from nested_loop import assert_rows_equal
from test_oracle_join import INT, INT_NN, JOIN_TYPES, make_case
from tidb_b200 import abi
from tidb_b200.chunk import DECIMAL_DTYPE, Chunk, Column, MutChunk, chunk_array
from tidb_b200.executor import HashJoinExec, MockDataSource
from tidb_b200.plan import FieldType, FilterItem, JoinPlan, OtherCond

pytestmark = pytest.mark.gpu

DEC = FieldType(abi.TYPE_NEWDECIMAL, 0, 15, 2)
DEC_NN = FieldType(abi.TYPE_NEWDECIMAL, abi.FLAG_NOT_NULL, 15, 2)
SPECIAL = [A.cell(0, 15, 2, neg_zero=True), A.cell(12345, 15, 2, result_frac=29), A.cell(-7, 15, 2, digits_int=0, result_frac=3),
           bytes(range(40)), b"\xff" * 40]
PROBE_ENV = ("TG_PROBE_PARTITION", "TG_PROBE_PARTS", "TG_PROBE_PART_MIN_MB", "TG_PROBE_PART_MIN_ROWS", "TG_PROBE_UQ", "TG_PROBE_INPLACE")


@pytest.fixture(autouse=True)
def _default_probe(monkeypatch):
    for k in PROBE_ENV:
        monkeypatch.delenv(k, raising=False)


def cells(rng, n):
    """random 40-byte cells, most of them bytes no canonical form produces, with the SPECIAL cells spread in"""
    c = rng.integers(0, 256, (n, 40), dtype=np.uint8)
    for i, s in enumerate(SPECIAL):
        c[i::37 + i] = np.frombuffer(s, dtype=np.uint8)
    return c


def add_decimal(rng, chunks, null_frac, nn_too=True):
    """append a nullable DECIMAL column (garbage bytes under NULL) and a NOT NULL one to every chunk"""
    for ch in chunks:
        n = ch.columns[0].length
        nl = rng.random(n) < null_frac if null_frac else None
        ch.columns.append(Column(cells(rng, n), nl))
        if nn_too:
            ch.columns.append(Column(cells(rng, n)))
    return chunks


def rows_of(cols):
    """[(values, nulls)] -> row tuples: None for NULL, bytes for a cell, Python scalars otherwise"""
    if not cols:
        return []
    n = len(cols[0][0])
    out = []
    for v, nl in cols:
        if v.ndim == 2:
            out.append([None if nl[i] else v[i].tobytes() for i in range(n)])
        else:
            out.append([None if nl[i] else v[i].item() for i in range(n)])
    return list(zip(*out))


def zero_under_null(cols):
    for v, nl in cols:
        if v.ndim == 2 and nl.any():
            assert not v[nl].any(), "a cell under NULL must be zero bytes"


def oracle_rows(plan, left, right):
    build, probe = (right, left) if plan.build_is_right else (left, right)
    j = O.OracleJoin(plan, 4)
    try:
        ba, pa = chunk_array(build), chunk_array(probe)
        assert O.lib().orc_join_run(j._h, ba, C.c_int64(len(build)), pa, C.c_int64(len(probe))) == 0
        n = O.lib().orc_join_result_rows(j._h)
        dts = [DECIMAL_DTYPE if t.tp == abi.TYPE_NEWDECIMAL else O._np_dtype(t) for t in plan.out_schema()]
        out = MutChunk([np.dtype(d).itemsize for d in dts], n, dts)
        assert O.lib().orc_join_result_fetch(j._h, C.byref(out.struct)) == 0
        return rows_of(out.columns(n)) if n else []
    finally:
        j.close()


def gpu_rows(plan, left, right, required_rows=1024, wait=False):
    """drain the join through tg_join_next (or tg_join_next_wait) -> (rows, stats)"""
    e = HashJoinExec(plan, MockDataSource(plan.left_types, left), MockDataSource(plan.right_types, right))
    e.open()
    try:
        rows = []
        if wait:
            e._build()
            for ch in (left if plan.build_is_right else right):
                cs = ch.to_struct()
                abi.check(e._lib.tg_join_probe_push(e._h, C.byref(cs)))
            abi.check(e._lib.tg_join_probe_finish(e._h))
            out = MutChunk([40 if t.tp == abi.TYPE_NEWDECIMAL else 8 for t in plan.out_schema()], required_rows,
                           [DECIMAL_DTYPE if t.tp == abi.TYPE_NEWDECIMAL else np.int64 for t in plan.out_schema()])
            n = C.c_int64(0)
            while True:
                abi.check(e._lib.tg_join_next_wait(e._h, C.byref(out.struct), C.c_int64(required_rows), C.byref(n)))
                if n.value == 0:
                    break
                cols = out.columns(n.value)
                zero_under_null(cols)
                rows.extend(rows_of(cols))
        else:
            while True:
                c = e.next(required_rows)
                if c.num_rows() == 0:
                    break
                cols = [(col.data, col.nulls()) for col in c.columns]
                zero_under_null(cols)
                rows.extend(rows_of(cols))
        return rows, e.stats()
    finally:
        e.close()


# ---- every join type x build side x {no NULLs, NULLs + duplicate keys, sel vectors} -----------------------------------
# left: 0 INT | 1 INT key | 2 INT | 3 DECIMAL | 4 DECIMAL NOT NULL      right: 0 INT key | 1 INT | 2 INT | 3 DECIMAL | 4 DECIMAL NN
@pytest.mark.parametrize("jt", JOIN_TYPES)
@pytest.mark.parametrize("build_is_right", [True, False])
@pytest.mark.parametrize("nulls,dup,with_sel", [(0.0, False, False), (0.15, True, False), (0.1, True, True)])
def test_decimal_payload_all_join_types(jt, build_is_right, nulls, dup, with_sel):
    if jt in (abi.JOIN_LEFT_OUTER_SEMI, abi.JOIN_ANTI_LEFT_OUTER_SEMI) and not build_is_right:
        pytest.skip("left outer semi joins need the right side as build side")
    rng = np.random.default_rng(9100 + jt * 7 + int(build_is_right) + int(nulls * 100))
    ltypes, rtypes, l, r = make_case(rng, 3000, 4000, nulls, dup, with_sel)
    add_decimal(rng, l, nulls); add_decimal(rng, r, nulls)
    ltypes, rtypes = ltypes + [DEC, DEC_NN], rtypes + [DEC, DEC_NN]
    semi = jt >= abi.JOIN_SEMI
    plan = JoinPlan(jt, ltypes, rtypes, [1], [0], build_is_right=build_is_right, lused=[3, 0, 4, 1], rused=[] if semi else [4, 2, 3])
    want = oracle_rows(plan, l, r)
    got, st = gpu_rows(plan, l, r)
    assert_rows_equal(want, got)
    if want:
        assert st.paths & abi.JOIN_PATH_CELL_GATHER


def test_noncanonical_cells_pass_through_unchanged():
    # inner join on unique keys: every probe row matches once, so each SPECIAL cell must come back byte for byte
    rng = np.random.default_rng(9200)
    n = 5000
    key = rng.permutation(n).astype(np.int64)
    pc, bc = cells(rng, n), cells(rng, n)
    left = [Chunk([Column(key), Column(np.arange(n, dtype=np.int64)), Column(pc)])]
    right = [Chunk([Column(np.arange(n, dtype=np.int64)), Column(bc)])]
    plan = JoinPlan(abi.JOIN_INNER, [INT_NN, INT_NN, DEC_NN], [INT_NN, DEC_NN], [0], [0], lused=[1, 2], rused=[0, 1])
    got, st = gpu_rows(plan, left, right)
    assert len(got) == n
    for prow, pcell, bkey, bcell in got:
        assert pcell == pc[prow].tobytes() and bcell == bc[bkey].tobytes() and bkey == key[prow]
    outs = {g[1] for g in got} | {g[3] for g in got}
    assert all(s in outs for s in SPECIAL)


# ---- each probe path carries DECIMAL, proven by tg_join_stats.paths ----------------------------------------------------
def unique_case(rng, nb, npr, match=0.7, probe_dec=2, build_dec=1, probe_nulls=False):
    bkey = rng.permutation(nb).astype(np.int64) * 3 + 1
    pkey = np.where(rng.random(npr) < match, bkey[rng.integers(0, nb, npr)], -5 - rng.integers(0, 1000, npr)).astype(np.int64)
    pcols = [Column(pkey), Column(np.arange(npr, dtype=np.int64))]
    for _ in range(probe_dec):
        pcols.append(Column(cells(rng, npr), (rng.random(npr) < 0.1) if probe_nulls else None))
    bcols = [Column(bkey), Column(np.arange(nb, dtype=np.int64) * 5)] + [Column(cells(rng, nb)) for _ in range(build_dec)]
    return pcols, bcols


@pytest.mark.parametrize("shape", ["u1_only_decimal_payload", "u1_no_payload", "uq_row_store", "general_probe_nulls"])
def test_decimal_on_unfused_and_direct_probe_paths(shape):
    rng = np.random.default_rng(9300)
    npr, nb = 200_000, 50_000           # >= 128 K rows: the probe chunk is copied straight to the device
    pcols, bcols = unique_case(rng, nb, npr, probe_nulls=shape == "general_probe_nulls")
    lt, rt = [INT_NN, INT_NN, DEC_NN, DEC_NN], [INT_NN, INT_NN, DEC_NN]
    if shape == "u1_only_decimal_payload":     # the DECIMAL column is the only build payload: a U1 table, the fused warp probe
        plan, want_path = JoinPlan(abi.JOIN_INNER, lt, rt, [0], [0], lused=[0, 2, 3], rused=[2]), abi.JOIN_PATH_PROBE_DIRECT
    elif shape == "u1_no_payload":
        plan, want_path = JoinPlan(abi.JOIN_INNER, lt, rt, [0], [0], lused=[3, 1, 0, 2], rused=[]), abi.JOIN_PATH_PROBE_DIRECT
    elif shape == "uq_row_store":              # two build payload columns and a probe filter: k_probe_inner_uq
        plan = JoinPlan(abi.JOIN_INNER, lt, rt, [0], [0], lused=[2, 1, 3], rused=[2, 1], probe_filter=[FilterItem(abi.CMP_GT, 1, const_i64=1000)])
        want_path = abi.JOIN_PATH_PROBE_UQ
    else:                                      # nullable DECIMAL probe columns, left outer: count -> scan -> write
        lt = [INT_NN, INT_NN, DEC, DEC]
        plan, want_path = JoinPlan(abi.JOIN_LEFT_OUTER, lt, rt, [0], [0], lused=[2, 1, 3], rused=[2]), abi.JOIN_PATH_PROBE_GENERAL
    left, right = [Chunk(pcols)], Chunk(bcols).split(1024)
    got, st = gpu_rows(plan, left, right, required_rows=1 << 18)
    assert st.paths & want_path and st.paths & abi.JOIN_PATH_CELL_GATHER, hex(st.paths)
    if want_path == abi.JOIN_PATH_PROBE_DIRECT:
        assert st.table_mode == 1
    assert_rows_equal(oracle_rows(plan, left, right), got)


def test_decimal_on_build_side_scan_multi_key_and_other_condition():
    rng = np.random.default_rng(9400)
    ltypes, rtypes, l, r = make_case(rng, 3000, 4000, 0.1, True, False)
    add_decimal(rng, l, 0.1); add_decimal(rng, r, 0.1)
    ltypes, rtypes = ltypes + [DEC, DEC_NN], rtypes + [DEC, DEC_NN]
    # outer side = build side: unmatched build rows come from the build-side scan, NULL-padded probe cells
    scan = JoinPlan(abi.JOIN_LEFT_OUTER, ltypes, rtypes, [1], [0], build_is_right=False, lused=[3, 1, 4], rused=[3, 4])
    got, st = gpu_rows(scan, l, r)
    assert_rows_equal(oracle_rows(scan, l, r), got)
    assert st.paths & abi.JOIN_PATH_CELL_GATHER
    other = JoinPlan(abi.JOIN_INNER, ltypes, rtypes, [1], [0], lused=[0, 3, 4], rused=[4, 3, 1],
                     other_cond=[OtherCond(abi.CMP_LE, 0, 0, 1, 1), OtherCond(abi.CMP_NE, 1, 2, -1, -1, const_i64=7)])
    got, st = gpu_rows(other, l, r)
    want = oracle_rows(other, l, r)
    assert want and st.table_mode == 2
    assert_rows_equal(want, got)
    multi = JoinPlan(abi.JOIN_LEFT_OUTER, ltypes, rtypes, [1, 2], [0, 2], build_is_right=True, lused=[3, 4, 1], rused=[0, 3])
    assert_rows_equal(oracle_rows(multi, l, r), gpu_rows(multi, l, r)[0])


def test_small_next_windows_next_wait_and_rewind():
    rng = np.random.default_rng(9500)
    ltypes, rtypes, l, r = make_case(rng, 2000, 3000, 0.1, True, True)
    add_decimal(rng, l, 0.1); add_decimal(rng, r, 0.1)
    plan = JoinPlan(abi.JOIN_LEFT_OUTER, ltypes + [DEC, DEC_NN], rtypes + [DEC, DEC_NN], [1], [0], lused=[3, 1, 4], rused=[4, 3])
    want = oracle_rows(plan, l, r)
    for req in (1, 7, 333):        # read cursors inside a byte of the NULL bitmap
        assert_rows_equal(want, gpu_rows(plan, l, r, required_rows=req)[0])
    assert_rows_equal(want, gpu_rows(plan, l, r, required_rows=5, wait=True)[0])
    # probe_rewind: a second probe pass against the same table gives the same rows
    inner = JoinPlan(abi.JOIN_INNER, plan.left_types, plan.right_types, [1], [0], lused=[3, 1, 4], rused=[4, 3])
    want = oracle_rows(inner, l, r)
    e = HashJoinExec(inner, MockDataSource(inner.left_types, l), MockDataSource(inner.right_types, r))
    e.open()
    try:
        for _ in range(2):
            rows = []
            while True:
                c = e.next(512)
                if c.num_rows() == 0:
                    break
                rows.extend(rows_of([(col.data, col.nulls()) for col in c.columns]))
            assert_rows_equal(want, rows)
            abi.check(e._lib.tg_join_probe_rewind(e._h))
            e.probe_child.open()
            e._probe_done = False
    finally:
        e.close()


def test_next_with_8_byte_output_for_decimal_is_invalid():
    rng = np.random.default_rng(9600)
    pcols, bcols = unique_case(rng, 1000, 3000)
    plan = JoinPlan(abi.JOIN_INNER, [INT_NN, INT_NN, DEC_NN, DEC_NN], [INT_NN, INT_NN, DEC_NN], [0], [0], lused=[0, 2], rused=[2])
    lib = abi.load_lib()
    d, keep = plan.to_struct()
    h = C.c_void_p()
    abi.check(lib.tg_join_open(C.byref(d), C.byref(h)))
    try:
        for ch in (Chunk(bcols),):
            cs = ch.to_struct(); abi.check(lib.tg_join_build_push(h, C.byref(cs)))
        abi.check(lib.tg_join_build_finish(h))
        cs = Chunk(pcols).to_struct(); abi.check(lib.tg_join_probe_push(h, C.byref(cs)))
        abi.check(lib.tg_join_probe_finish(h))
        n = C.c_int64(0)
        bad = MutChunk([8, 8, 8], 4096)
        assert lib.tg_join_next(h, C.byref(bad.struct), C.c_int64(4096), C.byref(n)) == abi.TG_ERR_INVALID
        good = MutChunk([8, 40, 40], 4096, [np.int64, DECIMAL_DTYPE, DECIMAL_DTYPE])
        abi.check(lib.tg_join_next(h, C.byref(good.struct), C.c_int64(4096), C.byref(n)))
        assert n.value > 0
    finally:
        lib.tg_join_close(h)


# ---- device-resident routes ----------------------------------------------------------------------------------------
def _dev_cells(ptr, n):
    import torch
    from tidb_b200.q3 import _view
    return _view(ptr, n * 5, torch.device("cuda")).view(torch.uint8).view(n, 40) if n else torch.zeros((0, 40), dtype=torch.uint8, device="cuda")


@pytest.mark.parametrize("mode", ["direct", "lean_segments", "inplace_segments", "probe_dev_seg"])
def test_device_resident_fused_paths(mode, monkeypatch):
    # build_push_dev / probe_dev; the L2 partition pass forced on a small input (lean and in-place segment probes), and a
    # segmented probe chunk (tg_join_probe_dev_seg accepts DECIMAL probe columns the fused kernels carry as row ids)
    import torch
    from tidb_b200.device import DeviceJoin
    from tidb_b200.q3 import _view
    if mode != "direct":
        for k, v in dict(TG_PROBE_PARTITION="1", TG_PROBE_PARTS="8", TG_PROBE_PART_MIN_MB="0", TG_PROBE_PART_MIN_ROWS="0").items():
            monkeypatch.setenv(k, v)
        monkeypatch.setenv("TG_PROBE_INPLACE", "1" if mode == "inplace_segments" else "0")
    g = torch.Generator(device="cuda").manual_seed(9700)
    nb, npr = 300_000, 2_000_000
    perm = torch.randperm(nb, device="cuda", generator=g)
    bkey = perm.to(torch.int64) * 7 + 3
    bdec = torch.randint(0, 256, (nb, 40), device="cuda", dtype=torch.uint8, generator=g)
    match = 1.0 if mode == "inplace_segments" else 0.8
    pkey = torch.where(torch.rand(npr, device="cuda", generator=g) < match, bkey[torch.randint(0, nb, (npr,), device="cuda", generator=g)],
                       torch.full((npr,), -1, device="cuda", dtype=torch.int64))
    prow = torch.arange(npr, device="cuda", dtype=torch.int64)
    pd1 = torch.randint(0, 256, (npr, 40), device="cuda", dtype=torch.uint8, generator=g)
    pd2 = torch.randint(0, 256, (npr, 40), device="cuda", dtype=torch.uint8, generator=g)
    plan = JoinPlan(abi.JOIN_INNER, [INT_NN, INT_NN, DEC_NN, DEC_NN], [INT_NN, DEC_NN], [0], [0], lused=[0, 1, 2, 3], rused=[1])
    torch.cuda.synchronize()
    j = DeviceJoin(plan)
    try:
        j.build([bkey, bdec])
        if mode == "probe_dev_seg":
            cap, nseg = 1 << 20, 2
            c0, c1 = npr // 2 - 1000, npr // 2 - 7
            cnt = torch.tensor([c0, c1], device="cuda", dtype=torch.int64)
            seg = lambda t: torch.cat([t[:npr // 2], torch.zeros((cap - npr // 2,) + tuple(t.shape[1:]), dtype=t.dtype, device="cuda"),
                                       t[npr // 2:], torch.zeros((cap - npr // 2,) + tuple(t.shape[1:]), dtype=t.dtype, device="cuda")])
            live = torch.cat([prow[:c0], prow[npr // 2:npr // 2 + c1]])
            sk, sr, s1, s2 = seg(pkey), seg(prow), seg(pd1), seg(pd2)
            torch.cuda.synchronize()
            n, cols, nulls = j.probe_segments([sk, sr, s1, s2], cnt, cap)
        else:
            live = prow
            n, cols, nulls = j.probe([pkey, prow, pd1, pd2])
        st = j.stats()
        ok, orow = _view(cols[0], n, "cuda").clone(), _view(cols[1], n, "cuda").clone()
        o1, o2, ob = _dev_cells(cols[2], n).clone(), _dev_cells(cols[3], n).clone(), _dev_cells(cols[4], n).clone()
        assert not any(nulls)
    finally:
        j.close()
    matched = live[pkey[live] >= 0]
    assert n == matched.numel()
    assert torch.equal(torch.sort(orow).values, torch.sort(matched).values)
    assert torch.equal(ok, pkey[orow]) and torch.equal(o1, pd1[orow]) and torch.equal(o2, pd2[orow])
    inv = torch.empty_like(perm); inv[perm] = torch.arange(nb, device="cuda")
    assert torch.equal(ob, bdec[inv[(ok - 3) // 7]])
    assert st.table_mode == 1 and st.paths & abi.JOIN_PATH_CELL_GATHER
    assert st.paths & (abi.JOIN_PATH_PROBE_DIRECT if mode in ("direct", "probe_dev_seg") else abi.JOIN_PATH_PROBE_SEG), hex(st.paths)


def test_full_scale_100m_probe_rows_10m_unique_build_keys():
    # the J2 shape at scale, device-resident: two DECIMAL probe columns and one DECIMAL build column, checked against a
    # torch index gather
    import torch
    from tidb_b200.device import DeviceJoin
    from tidb_b200.q3 import _view
    g = torch.Generator(device="cuda").manual_seed(9800)
    nb, npr = 10_000_000, 100_000_000
    perm = torch.randperm(nb, device="cuda", generator=g)
    bkey = perm.to(torch.int64) * 4 + 1
    bdec = torch.randint(0, 256, (nb, 40), device="cuda", dtype=torch.uint8, generator=g)
    pkey = bkey[torch.randint(0, nb, (npr,), device="cuda", generator=g)]
    prow = torch.arange(npr, device="cuda", dtype=torch.int64)
    pd1 = torch.randint(0, 256, (npr, 40), device="cuda", dtype=torch.uint8, generator=g)
    pd2 = torch.randint(0, 256, (npr, 40), device="cuda", dtype=torch.uint8, generator=g)
    plan = JoinPlan(abi.JOIN_INNER, [INT_NN, INT_NN, DEC_NN, DEC_NN], [INT_NN, DEC_NN], [0], [0], lused=[0, 1, 2, 3], rused=[1])
    torch.cuda.synchronize()
    j = DeviceJoin(plan)
    try:
        j.build([bkey, bdec])
        n, cols, _ = j.probe([pkey, prow, pd1, pd2])
        st = j.stats()
        assert n == npr
        orow = _view(cols[1], n, "cuda")
        assert torch.equal(torch.sort(orow).values, prow)
        assert torch.equal(_view(cols[0], n, "cuda"), pkey[orow])
        assert torch.equal(_dev_cells(cols[2], n), pd1[orow])
        assert torch.equal(_dev_cells(cols[3], n), pd2[orow])
        inv = torch.empty_like(perm); inv[perm] = torch.arange(nb, device="cuda")
        assert torch.equal(_dev_cells(cols[4], n), bdec[inv[(pkey[orow] - 1) // 4]])
        assert st.paths & abi.JOIN_PATH_CELL_GATHER and st.paths & (abi.JOIN_PATH_PROBE_SEG | abi.JOIN_PATH_PROBE_DIRECT)
    finally:
        j.close()


def test_q3_shape_pipeline_with_decimal_prices():
    # J1 = orders JOIN customer, J2 = lineitem JOIN J1, both device-resident, carrying DECIMAL(15,2) l_extendedprice /
    # l_discount (probe side of J2) and o_totalprice (through J1, then the build side of J2); then DeviceAgg
    # SUM(l_extendedprice * (1 - l_discount)) GROUP BY l_orderkey, o_orderdate, o_shippriority, compared exactly
    import torch
    import mydecimal_expr as X
    from tidb_b200.device import DeviceAgg, DeviceJoin
    from tidb_b200.plan import AggFunc, AggPlan
    from tidb_b200.q3 import DATE, SEGMENT, _view
    dev = torch.device("cuda")
    g = torch.Generator(device="cuda").manual_seed(9900)
    nc, no, nl = 30_000, 300_000, 1_200_000
    ri = lambda lo, hi, n: torch.randint(lo, hi, (n,), device=dev, generator=g, dtype=torch.int64)

    def dcells(v):   # FromBin's form of DECIMAL(15,2): digitsInt 13, one fraction word
        w = torch.zeros((v.numel(), 10), dtype=torch.int32, device=dev)
        w[:, 0] = 13 | (2 << 8)
        w[:, 1] = (v // 100 // 10 ** 9).to(torch.int32)
        w[:, 2] = (v // 100 % 10 ** 9).to(torch.int32)
        w[:, 3] = ((v % 100) * 10 ** 7).to(torch.int32)
        return w.view(torch.uint8).view(v.numel(), 40)

    c_key, c_seg = torch.randperm(nc, device=dev, generator=g), ri(0, 5, nc)
    o_key, o_cust, o_date, o_prio = torch.randperm(no, device=dev, generator=g) * 4 + 1, ri(0, nc, no), ri(0, 2406, no), ri(0, 5, no)
    o_total = ri(0, 50_000_000, no)
    l_key, l_price, l_disc, l_ship = ri(0, no, nl) * 4 + 1, ri(90_000, 10_500_000, nl), ri(0, 11, nl), ri(0, 2406, nl)
    o_tc, l_pc, l_dc = dcells(o_total), dcells(l_price), dcells(l_disc)
    torch.cuda.synchronize()
    D = DEC_NN
    j1 = DeviceJoin(JoinPlan(abi.JOIN_INNER, [INT_NN, INT_NN, INT_NN, INT_NN, D], [INT_NN, INT_NN], [1], [0], lused=[0, 2, 3, 4], rused=[],
                             build_filter=[FilterItem(abi.CMP_EQ, 1, const_i64=SEGMENT)], probe_filter=[FilterItem(abi.CMP_LT, 2, const_i64=DATE)]))
    j2 = DeviceJoin(JoinPlan(abi.JOIN_INNER, [INT_NN, D, D, INT_NN], [INT_NN, INT_NN, INT_NN, D], [0], [0], lused=[0, 1, 2], rused=[1, 2, 3],
                             probe_filter=[FilterItem(abi.CMP_GT, 3, const_i64=DATE)]))
    try:
        j1.build([c_key, c_seg])
        n1, c1, _ = j1.probe([o_key, o_cust, o_date, o_prio, o_tc])
        j2.build([_view(c1[0], n1, dev), _view(c1[1], n1, dev), _view(c1[2], n1, dev), _dev_cells(c1[3], n1)])
        n2, c2, _ = j2.probe([l_key, l_pc, l_dc, l_ship])
        st1, st2 = j1.stats(), j2.stats()
        lk, price, disc = _view(c2[0], n2, dev), _dev_cells(c2[1], n2), _dev_cells(c2[2], n2)
        od, op, ot = _view(c2[3], n2, dev), _view(c2[4], n2, dev), _dev_cells(c2[5], n2)
        # reference joins by index: the orders row of an order key, the customer row of a customer key
        oinv = torch.empty_like(o_key); oinv[(o_key - 1) // 4] = torch.arange(no, device=dev)
        cinv = torch.empty_like(c_key); cinv[c_key] = torch.arange(nc, device=dev)
        orow, lrow = oinv[(lk - 1) // 4], oinv[(l_key - 1) // 4]
        keep = (l_ship > DATE) & (o_date[lrow] < DATE) & (c_seg[cinv[o_cust[lrow]]] == SEGMENT)
        assert n2 == int(keep.sum())
        assert torch.equal(od, o_date[orow]) and torch.equal(op, o_prio[orow]) and torch.equal(ot, o_tc[orow])
        assert st1.paths & abi.JOIN_PATH_CELL_GATHER and st2.paths & abi.JOIN_PATH_CELL_GATHER
        agg = DeviceAgg(AggPlan([INT_NN, D, D, INT_NN, INT_NN], [0, 3, 4],
                                [AggFunc(abi.AGG_FIRSTROW, 0), AggFunc(abi.AGG_FIRSTROW, 3), AggFunc(abi.AGG_FIRSTROW, 4),
                                 AggFunc(abi.AGG_SUM, 1, abi.TYPE_NEWDECIMAL, ret_type=abi.TYPE_NEWDECIMAL, ret_frac=4, arg_col2=2,
                                         arg_expr=abi.ARGEXPR_MUL_CSUB, arg_const=1.0)], expected_groups=max(n1, 1)))
        try:
            torch.cuda.synchronize()
            agg.push([lk, price, disc, od, op])
            ng, ca, _ = agg.finish()
            gk, gd, gp = (_view(ca[i], ng, dev).cpu().numpy() for i in range(3))
            gs = _dev_cells(ca[3], ng).cpu().numpy()
        finally:
            agg.close()
    finally:
        j2.close(); j1.close()
    kk = keep.cpu().numpy()
    lk_h, p_h, d_h = l_key.cpu().numpy()[kk], l_price.cpu().numpy()[kk], l_disc.cpu().numpy()[kk]
    tuples, inv = np.unique(lk_h, return_inverse=True)
    sums, _ = X.group_sums(p_h * (100 - d_h), np.ones(len(lk_h), dtype=bool), inv, len(tuples))
    want = {int(k): X.sum_result(s, 4) for k, s in zip(tuples.tolist(), sums)}
    assert ng == len(want) > 0
    od_h, op_h = o_date.cpu().numpy(), o_prio.cpu().numpy()
    oinv_h = oinv.cpu().numpy()
    for r in range(ng):
        k = int(gk[r])
        assert gs[r].tobytes() == want[k], k
        assert gd[r] == od_h[oinv_h[(k - 1) // 4]] and gp[r] == op_h[oinv_h[(k - 1) // 4]]
