"""The hash aggregation's find-or-insert loops on keys crafted through the hash (tests/agg_keys.py), against the exact
references (tests/agg_reference.py, tests/agg_distinct_reference.py).

Keys whose hashes share their top 32 bits share a home at every table size, so a cluster of them is one run that no
growth shortens.  Each cluster is mixed into about 100 K uniform background rows whose homes keep out of the cluster's
window, with the NULL group and the INT64_MIN (empty-sentinel) key.  Each case forces one update path through the TG_AGG_*
switches and proves it from tg_agg_stats.paths, compares every group (COUNT, MIN, MAX and FIRSTROW bit-exact, SUM and AVG
within the order-free bound), asserts the exact group count, and bounds table_slots / set_slots by the growth rule's
bound for as many entries (agg_keys.slots_bound): a crafted cluster costs no more table than uniform groups."""
import numpy as np
import pytest

import agg_distinct_reference as DR
import agg_keys as K
import agg_reference as R
from test_gpu_agg_distinct import cnt, davg, dsum, run_host as run_host_distinct
from test_gpu_agg_paths import run_dev, run_host
from tidb_b200 import abi
from tidb_b200.chunk import Chunk, Column
from tidb_b200.plan import AggFunc, AggPlan, FieldType

pytestmark = pytest.mark.gpu

P = abi
I64_MIN = -(1 << 63)
INT = FieldType(abi.TYPE_LONGLONG, 0)
INT_NN = FieldType(abi.TYPE_LONGLONG, abi.FLAG_NOT_NULL)
UINT = FieldType(abi.TYPE_LONGLONG, abi.FLAG_UNSIGNED)
DBL = FieldType(abi.TYPE_DOUBLE, 0)
DBL_NN = FieldType(abi.TYPE_DOUBLE, abi.FLAG_NOT_NULL)
SWITCHES = ("TG_AGG_LOCAL", "TG_AGG_LOCAL_SLOTS", "TG_AGG_V1")
TOP = 0x12345678
N_BG = 100_000

# path -> (switches, background groups, expected_groups, path bits wanted, path bits that must stay clear)
PATHS = {
    "v2_global": ({"TG_AGG_LOCAL": "0"}, 10_000, 0, P.AGG_PATH_V2_GLOBAL, P.AGG_PATH_V2_LOCAL | P.AGG_PATH_MERGE),
    "v2_local": ({"TG_AGG_LOCAL": "2"}, 60, 0, P.AGG_PATH_V2_LOCAL, P.AGG_PATH_V1_LOCAL | P.AGG_PATH_V1_GLOBAL),
    "v1_local": ({"TG_AGG_V1": "1"}, 60, 0, P.AGG_PATH_V1_LOCAL | P.AGG_PATH_MERGE, P.AGG_PATH_V2_LOCAL | P.AGG_PATH_V2_GLOBAL),
    "v1_global": ({"TG_AGG_V1": "1"}, 10_000, 20_000, P.AGG_PATH_V1_GLOBAL, P.AGG_PATH_V1_LOCAL | P.AGG_PATH_V2_GLOBAL),
}


@pytest.fixture(autouse=True)
def _default_switches(monkeypatch):
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)


def set_path(monkeypatch, path):
    for k, v in PATHS[path][0].items():
        monkeypatch.setenv(k, v)


# ---- single GROUP BY column ----------------------------------------------------------------------------------------
def plans1(key_type, hint):
    """two function lists of <= 4 state words each (the CTA-local levels take no more); columns: 0 key | 1 x DOUBLE
    (nullable) | 2 i BIGINT NOT NULL"""
    types = [key_type, DBL, INT_NN]
    fr = [AggFunc(P.AGG_FIRSTROW, 0), AggFunc(P.AGG_COUNT, -1)]
    return [AggPlan(types, [0], fr + [AggFunc(P.AGG_SUM, 1, P.TYPE_DOUBLE), AggFunc(P.AGG_AVG, 1, P.TYPE_DOUBLE)], expected_groups=hint),
            AggPlan(types, [0], fr + [AggFunc(P.AGG_MIN, 2), AggFunc(P.AGG_MAX, 2), AggFunc(P.AGG_COUNT, 1, P.TYPE_DOUBLE)], expected_groups=hint)]


def background(rng, n, ngroups, tops, min_slots, double=False):
    """n rows over ngroups uniform keys whose homes keep out of the clusters' windows, plus NULL and (BIGINT) INT64_MIN rows"""
    pool = rng.integers(-(1 << 62), 1 << 62, ngroups * 2)
    if double:
        pool = (pool >> 11).astype(np.float64) * 0.25
        bits = np.where(pool == 0, 0, pool.view(np.int64))
    else:
        bits = pool
    pool = pool[K.outside_window(bits, tops, min_slots)][:ngroups]
    keys = pool[rng.integers(0, len(pool), n)]
    nulls = rng.random(n) < 0.01
    if not double:
        keys[rng.random(n) < 0.002] = I64_MIN
    return keys, nulls


def single_chunks(rng, clusters, ngroups, min_slots, double=False, rows_per_key=2, n_bg=N_BG):
    """the clusters' keys (rows_per_key rows each) mixed into the background, shuffled; -> (key, null) arrays, x, i"""
    tops = [(t, len(ks)) for t, ks in clusters]
    bk, bn = background(rng, n_bg, ngroups, tops, min_slots, double)
    ck = np.repeat(np.array([k for _, ks in clusters for k in ks], dtype=np.float64 if double else np.int64), rows_per_key)
    keys = np.concatenate([bk, ck])
    nulls = np.concatenate([bn, np.zeros(len(ck), dtype=bool)])
    if double:   # -0.0 and +0.0 form one group
        z = rng.random(len(keys)) < 0.002
        keys[z] = np.where(rng.random(int(z.sum())) < 0.5, -0.0, 0.0)
    n = len(keys)
    perm = rng.permutation(n)
    x = (rng.random(n) - 0.5) * 1e6
    xn = rng.random(n) < 0.05
    i = rng.integers(I64_MIN, (1 << 63) - 1, n, endpoint=True, dtype=np.int64)
    return keys[perm], nulls[perm], x[perm], xn[perm], i[perm], len(ck)


def to_chunk(keys, nulls, x, xn, i):
    return Chunk([Column(keys, nulls), Column(x, xn), Column(i)])


def check_single(plan_list, chunks, want, dont, first, cluster_rows, runner=None, local=None):
    for plan in plan_list:
        rows, st = (runner or run_host)(plan, chunks)
        groups = R.check(plan, chunks, rows)
        assert st.groups == groups, (st.groups, groups)
        assert st.paths & want == want, (hex(st.paths), hex(want))
        assert st.paths & dont == 0, (hex(st.paths), hex(dont))
        if local is not None:
            assert (st.local_rows > 0) == local, st.local_rows
        bound = K.slots_bound(first, groups + cluster_rows)
        assert st.table_slots <= bound, (st.table_slots, bound)
    return st


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("c", [49, 50, 51, 200, 5000])
def test_single_column_cluster(c, path, monkeypatch):
    set_path(monkeypatch, path)
    _, ngroups, hint, want, dont = PATHS[path]
    rng = np.random.default_rng(c + len(path))
    clusters = [(TOP, K.top_keys(c, TOP))]
    n_total = N_BG + 2 * c
    first = K.first_slots(n_total, hint)
    keys, nulls, x, xn, i, crows = single_chunks(rng, clusters, ngroups, first)
    chunks = to_chunk(keys, nulls, x, xn, i).split(1 << 15)
    if c >= 50 and path in ("v2_local", "v1_local"):
        want |= P.AGG_PATH_MERGE   # the cluster's local groups find no global slot within the limit: merged after
    check_single(plans1(INT, hint), chunks, want, dont, first, crows, local=(path == "v2_local") or None)


@pytest.mark.parametrize("path", list(PATHS))
def test_wrap_cluster_and_home_zero_cluster(path, monkeypatch):
    # a cluster on the last slot at every size wraps to slot 0, where a second cluster has its home: one run of 260 keys
    set_path(monkeypatch, path)
    _, ngroups, hint, want, dont = PATHS[path]
    rng = np.random.default_rng(100)
    clusters = [(0xFFFFFFFF, K.top_keys(130, 0xFFFFFFFF)), (0, K.top_keys(130, 0))]
    first = K.first_slots(N_BG + 520, hint)
    keys, nulls, x, xn, i, crows = single_chunks(rng, clusters, ngroups, first)
    check_single(plans1(INT, hint), to_chunk(keys, nulls, x, xn, i).split(1 << 15), want, dont, first, crows)


@pytest.mark.parametrize("path", ["v2_global", "v2_local", "v1_global"])
def test_unsigned_keys(path, monkeypatch):
    # BIGINT UNSIGNED: the same 8 bytes, keys above 2^63 among them
    set_path(monkeypatch, path)
    _, ngroups, hint, want, dont = PATHS[path]
    rng = np.random.default_rng(200)
    ks = K.top_keys(300, TOP)
    assert any(k < 0 for k in ks)      # read as unsigned: above 2^63
    first = K.first_slots(N_BG + 600, hint)
    keys, nulls, x, xn, i, crows = single_chunks(rng, [(TOP, ks)], ngroups, first)
    check_single(plans1(UINT, hint), to_chunk(keys, nulls, x, xn, i).split(1 << 15), want, dont, first, crows)


@pytest.mark.parametrize("path", ["v2_global", "v2_local", "v1_local", "v1_global"])
def test_double_keys(path, monkeypatch):
    set_path(monkeypatch, path)
    _, ngroups, hint, want, dont = PATHS[path]
    rng = np.random.default_rng(300)
    first = K.first_slots(N_BG + 600, hint)
    keys, nulls, x, xn, i, crows = single_chunks(rng, [(TOP, K.top_doubles(300, TOP))], ngroups, first, double=True)
    if path == "v1_local":
        want |= P.AGG_PATH_MERGE
    check_single(plans1(DBL, hint), to_chunk(keys, nulls, x, xn, i).split(1 << 15), want, dont, first, crows)


@pytest.mark.parametrize("c", [50, 5000])
@pytest.mark.parametrize("hint_kind", ["none", "fits_cluster"])
def test_expected_groups_hint(c, hint_kind, monkeypatch):
    # hint 0 sizes the first table from the rows; a hint of the cluster's size makes the first table just fit it
    monkeypatch.setenv("TG_AGG_LOCAL", "0")
    rng = np.random.default_rng(400 + c)
    hint = c if hint_kind == "fits_cluster" else 0
    n_total = N_BG + 2 * c
    first = K.first_slots(n_total, hint)
    keys, nulls, x, xn, i, crows = single_chunks(rng, [(TOP, K.top_keys(c, TOP))], 100, first)
    check_single(plans1(INT, hint), to_chunk(keys, nulls, x, xn, i).split(1 << 15), P.AGG_PATH_V2_GLOBAL, 0, first, crows)


@pytest.mark.parametrize("path", ["v2_global", "v2_local", "v1_global"])
def test_device_pushes_split_cluster(path, monkeypatch):
    # four tg_agg_push_dev batches, each carrying a quarter of one 400-key cluster: every batch meets the run the
    # earlier ones left
    set_path(monkeypatch, path)
    _, ngroups, hint, want, dont = PATHS[path]
    rng = np.random.default_rng(500)
    ks = K.top_keys(400, TOP)
    n_bg = N_BG // 4
    first = K.first_slots(n_bg + 200, hint)
    batches, crows = [], 0
    for q in range(4):
        keys, nulls, x, xn, i, cr = single_chunks(rng, [(TOP, ks[q * 100:(q + 1) * 100])], ngroups, first, n_bg=n_bg)
        batches.append(to_chunk(keys, nulls, x, xn, i))
        crows += cr
    check_single(plans1(INT, hint), batches, want, dont, first, crows, runner=run_dev)


@pytest.mark.parametrize("slots", ["512", "2048"])
def test_cta_local_cluster_wraps_at_ls(slots, monkeypatch):
    # 600 keys that share the CTA-local table's last slot at every local size: their local run wraps at ls and fills the
    # table to its limit, so part of the cluster goes to the global table beside the background
    monkeypatch.setenv("TG_AGG_LOCAL", "2")
    monkeypatch.setenv("TG_AGG_LOCAL_SLOTS", slots)
    rng = np.random.default_rng(600)
    ks = K.local_top_keys(600)
    first = K.first_slots(N_BG + 1200)
    bk, bn = background(rng, N_BG, 60, [], first)
    # the cluster's rows stay together in the middle of the input, so that one CTA's tiles hold most of them
    keys = np.concatenate([bk[:N_BG // 2], np.array(ks + ks, dtype=np.int64), bk[N_BG // 2:]])
    nulls = np.concatenate([bn[:N_BG // 2], np.zeros(1200, dtype=bool), bn[N_BG // 2:]])
    n = len(keys)
    x = (rng.random(n) - 0.5) * 1e6
    i = rng.integers(I64_MIN, (1 << 63) - 1, n, endpoint=True, dtype=np.int64)
    chunks = to_chunk(keys, nulls, x, rng.random(n) < 0.05, i).split(1 << 15)
    check_single(plans1(INT, 0), chunks, P.AGG_PATH_V2_LOCAL, 0, first, 1200, local=True)


# ---- several GROUP BY columns ----------------------------------------------------------------------------------------
KINDS = {2: ["f", "i"], 3: ["i", "f", "i"], 4: ["i", "f", "i", "i"]}


def mk_types(ncols, nullable):
    t = {"i": INT if nullable else INT_NN, "f": DBL if nullable else DBL_NN}
    return [t[k] for k in KINDS[ncols]] + [DBL, INT_NN]


def mk_plans(ncols, nullable):
    types = mk_types(ncols, nullable)
    fr = [AggFunc(P.AGG_FIRSTROW, c) for c in range(ncols)]
    return [AggPlan(types, list(range(ncols)), fr + [AggFunc(P.AGG_COUNT, -1), AggFunc(P.AGG_SUM, ncols, P.TYPE_DOUBLE),
                                                     AggFunc(P.AGG_AVG, ncols, P.TYPE_DOUBLE), AggFunc(P.AGG_MIN, ncols + 1),
                                                     AggFunc(P.AGG_MAX, ncols + 1)])]


def mk_background(rng, n, ncols, nullable, tops, min_slots):
    """n rows over small-range key columns (NULLs and both zeros among them when nullable), whose rows hash outside the
    clusters' windows"""
    kinds = KINDS[ncols]
    cols, nls = [], []
    for k in kinds:
        v = rng.integers(-20, 21, 3 * n)
        cols.append(v.astype(np.float64) * 0.5 if k == "f" else v.astype(np.int64))
        nls.append(rng.random(3 * n) < (0.05 if nullable else 0))
    words = []
    nb = np.zeros(3 * n, dtype=np.int64)
    for j, (k, v, nl) in enumerate(zip(kinds, cols, nls)):
        w = np.where(v == 0, 0, v.view(np.int64)) if k == "f" else v
        words.append(np.where(nl, 0, w))
        nb |= nl.astype(np.int64) << j
    if nullable:
        words.append(nb)
    ok = np.nonzero(K.outside_window_h(K.hash_words_np(words), tops, min_slots))[0][:n]
    return [(c[ok], nl[ok]) for c, nl in zip(cols, nls)]


def mk_chunks(rng, ncols, nullable, crafted, tops, min_slots):
    """background rows plus each crafted row twice, shuffled, with the argument columns; -> chunks, crafted rows"""
    bg = mk_background(rng, N_BG, ncols, nullable, tops, min_slots)
    kinds = KINDS[ncols]
    cols = []
    for j, k in enumerate(kinds):
        cv = np.array([0 if r[j] is None else r[j] for r in crafted for _ in range(2)], dtype=np.float64 if k == "f" else np.int64)
        cn = np.array([r[j] is None for r in crafted for _ in range(2)], dtype=bool)
        cols.append((np.concatenate([bg[j][0], cv]), np.concatenate([bg[j][1], cn])))
    n = len(cols[0][0])
    perm = rng.permutation(n)
    x = (rng.random(n) - 0.5) * 1e6
    i = rng.integers(I64_MIN, (1 << 63) - 1, n, endpoint=True, dtype=np.int64)
    chunk = Chunk([Column(v[perm], nl[perm] if nullable else None) for v, nl in cols] + [Column(x, rng.random(n) < 0.05), Column(i)])
    return chunk.split(1 << 15), 2 * len(crafted)


@pytest.mark.parametrize("nullable", [False, True])
@pytest.mark.parametrize("ncols", [2, 3, 4])
def test_multi_key_cluster_and_equal_hash_rows(ncols, nullable):
    kinds = KINDS[ncols]
    seed = {2: [0.5, 0], 3: [7, None if nullable else 0.5, 3], 4: [7, 0.5, None if nullable else 3, 11]}[ncols]
    crafted = K.rows_with_top(300, TOP, kinds, nullable, seed)
    # different rows with one 64-bit hash, so one home and one tag: only the ordered compare of the key words parts them
    eq_seed = {2: [1.5, 5], 3: [5, 2.5, 9], 4: [5, 2.5, 9, -2]}[ncols]
    eq = K.equal_hash_rows(40, eq_seed, kinds, nullable)
    tops = [(TOP, 300), (K.hash_words(K.key_words(eq[0], kinds, nullable)) >> 32, 40)]
    extra = []
    if nullable:   # (NULL, a, b, c) beside (0, a, b, c), and their equal-hash neighbours
        z = list(eq_seed)
        z[0] = 0.0 if kinds[0] == "f" else 0
        extra = [tuple(z), tuple([None] + z[1:])]
    first = K.first_slots(N_BG + 2 * (len(crafted) + len(eq) + len(extra)))
    chunks, crows = mk_chunks(np.random.default_rng(700 + ncols + 10 * nullable), ncols, nullable, crafted + eq + extra, tops, first)
    for plan in mk_plans(ncols, nullable):
        rows, st = run_host(plan, chunks)
        groups = R.check(plan, chunks, rows)
        assert st.groups == groups
        assert st.paths & P.AGG_PATH_MULTI_KEY and not st.paths & (P.AGG_PATH_V2_GLOBAL | P.AGG_PATH_V1_GLOBAL)
        assert st.table_slots <= K.slots_bound(first, groups + crows), st.table_slots


# ---- DISTINCT ---------------------------------------------------------------------------------------------------------
# columns: 0 g BIGINT (nullable) | 1 x BIGINT (nullable): the DISTINCT argument
D_TYPES = [INT, INT]


def d_plans(group_by):
    """the second list keeps to 4 state words, so the CTA-local level takes it"""
    fr = [AggFunc(P.AGG_FIRSTROW, 0)] if group_by else []
    return [AggPlan(D_TYPES, list(group_by), fr + [cnt(1), dsum(1), davg(1, 4), AggFunc(P.AGG_COUNT, 1)]),
            AggPlan(D_TYPES, list(group_by), fr + [cnt(1), davg(1, 4)])]


def d_run(plan, vals, first, entries):
    chunk = Chunk([Column(vals[c][0], vals[c][1]) for c in range(2)])
    rows, st, ds = run_host_distinct(plan, chunk.split(1 << 15))
    groups = DR.check(plan, vals, rows)
    assert st.groups == groups
    pairs = DR.pair_count(plan, vals, 1)
    assert ds.pairs == pairs, (ds.pairs, pairs)
    assert ds.set_slots <= K.slots_bound(first, pairs + entries), ds.set_slots
    return ds


def d_vals(rng, crafted, group_by, tops, first):
    """background (group, value) rows whose set hash keeps out of the windows, plus each crafted pair twice"""
    n = N_BG
    g = rng.integers(0, 300, 3 * n).astype(np.int64)
    gn = rng.random(3 * n) < 0.01
    v = rng.integers(-(1 << 40), 1 << 40, 3 * n)
    words = ([np.where(gn, 0, g), gn.astype(np.int64)] if group_by else []) + [v]
    ok = np.nonzero(K.outside_window_h(K.hash_words_np(words), tops, first))[0][:n]
    g, gn, v = g[ok], gn[ok], v[ok]
    vn = rng.random(len(v)) < 0.03
    cg = np.array([0 if p[0] is None else p[0] for p in crafted for _ in range(2)], dtype=np.int64)
    cgn = np.array([p[0] is None for p in crafted for _ in range(2)], dtype=bool)
    cv = np.array([p[1] for p in crafted for _ in range(2)], dtype=np.int64)
    perm = rng.permutation(len(g) + len(cg))
    cat = lambda a, b: np.concatenate([a, b])[perm]
    return {0: (cat(g, cg), cat(gn, cgn)), 1: (cat(v, cv), cat(vn, np.zeros(len(cv), dtype=bool)))}


@pytest.mark.parametrize("group_by", [(), (0,)])
def test_distinct_clustered_values(group_by):
    # 300 values of one group (or of no GROUP BY) share the set home at every size, and 40 pairs of different groups, the
    # NULL group among them, share one 64-bit set hash
    gw = lambda g: K.key_words([g], ["i"], True)
    if group_by:
        crafted = [(42, x) for x in K.values_with_set_top(300, gw(42), TOP)]
        eq = K.equal_hash_pairs(40, gw, [None] + list(range(1000, 1039)), 77)
        tops = [(TOP, 300), (K.hash_words(K.pair_words(gw(None), 77)) >> 32, 40)]
    else:
        crafted = [(0, x) for x in K.values_with_set_top(300, [], TOP)]
        eq = []
        tops = [(TOP, 300)]
    rows = N_BG + 2 * (len(crafted) + len(eq))
    first = K.first_slots(rows)
    vals = d_vals(np.random.default_rng(800 + len(group_by)), crafted + eq, group_by, tops, first)
    for plan in d_plans(group_by):
        d_run(plan, vals, first, 2 * (len(crafted) + len(eq)))
