"""Unique-key join tables at high load factors: long linear-probe runs (probed by 32-byte pairs), runs that wrap past the
last slot, the sentinel key, every probe path, and the densified default table.  Every output row is compared with a numpy
reference."""
import numpy as np
import pytest

from test_join_slice_sizing import table_slots
from test_oracle_join import INT_NN
from tidb_b200 import abi
from tidb_b200.chunk import Chunk, Column
from tidb_b200.executor import HashJoinExec, MockDataSource
from tidb_b200.plan import FilterItem, JoinPlan

pytestmark = pytest.mark.gpu

SENTINEL = -(1 << 63)
MUL = 0x9E3779B97F4A7C15
MUL_INV = pow(MUL, -1, 1 << 64)
PART = dict(TG_PROBE_PARTITION="1", TG_PROBE_PARTS="8", TG_PROBE_PART_MIN_MB="0", TG_PROBE_PART_MIN_ROWS="0")


def keys_hashing_to_the_end(n):
    """n keys whose hash64 is within 2^40 of 2^64: their home is one of the last slots of any table below 2^24 slots, so their
    runs wrap to slot 0.  hash64(k) = (k ^ k >> 32) * MUL: invert the multiply, then the xor-fold."""
    h = [(1 << 64) - 1 - i * 7919 for i in range(n)]
    f = [(x * MUL_INV) % (1 << 64) for x in h]
    k = [x ^ (x >> 32) for x in f]
    return np.array(k, dtype=np.uint64).view(np.int64)


def make_sides(nb, npr, match, seed):
    rng = np.random.default_rng(seed)
    bk = rng.permutation(nb).astype(np.int64) * 2654435761 + 3
    bk[:200] = keys_hashing_to_the_end(200)
    bk[200] = SENTINEL
    bv = np.arange(nb, dtype=np.int64) * 3 + 1
    miss = rng.integers(0, 1 << 62, npr).astype(np.int64) * 2 + 1       # odd: never a build key (build keys are even below)
    bk[201:] += bk[201:] & 1
    pk = np.where(rng.random(npr) < match, bk[rng.integers(0, nb, npr)], miss)
    pk[:500] = bk[rng.integers(0, 201, 500)] if match > 0 else miss[:500]   # wrapped runs and the sentinel key
    if match == 0:
        pk[500] = SENTINEL
        bk[200] = 6                                                         # the sentinel is on the probe side only
    return bk, bv, pk


def check(got, bk, bv, pk, pv=None):
    """got = (probe key, probe payload, build key, build payload) with probe payload = the probe row index"""
    pv = np.arange(len(pk), dtype=np.int64) if pv is None else pv
    order = np.argsort(bk)
    sb = bk[order]
    pos = np.minimum(np.searchsorted(sb, pk), len(bk) - 1)
    hit = sb[pos] == pk
    assert len(got[0]) == int(hit.sum())
    rows = np.searchsorted(pv, got[1])
    assert np.array_equal(np.sort(rows), np.nonzero(hit)[0])              # each matching probe row exactly once
    assert np.array_equal(got[0], pk[rows]) and np.array_equal(got[2], got[0])
    assert np.array_equal(got[3], bv[order[pos[rows]]])


def run_host(bk, bv, pk, lf, filt=None):
    plan = JoinPlan(abi.JOIN_INNER, [INT_NN, INT_NN], [INT_NN, INT_NN], [0], [0], load_factor=lf, probe_filter=filt or [])
    e = HashJoinExec(plan, MockDataSource(plan.left_types, [Chunk([Column(pk), Column(np.arange(len(pk), dtype=np.int64))])]),
                     MockDataSource(plan.right_types, [Chunk([Column(bk), Column(bv)])]))
    e.open()
    chunks = []
    while True:
        c = e.next(1 << 22)
        if c.num_rows() == 0:
            break
        chunks.append(c)
    st = e.stats()
    e.close()
    return [np.concatenate([c.columns[i].data for c in chunks] + [np.zeros(0, np.int64)]) for i in range(4)], st


def setenv(monkeypatch, env):
    for k in ("TG_PROBE_PARTITION", "TG_PROBE_PARTS", "TG_PROBE_UQ"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


@pytest.mark.parametrize("lf", [0.35, 0.8, 0.95])
@pytest.mark.parametrize("match", [1.0, 0.5, 0.0])
def test_dense_table_segment_probe(lf, match, monkeypatch):
    setenv(monkeypatch, PART)
    nb, npr = 100_003, 700_001
    bk, bv, pk = make_sides(nb, npr, match, seed=int(lf * 100))
    got, st = run_host(bk, bv, pk, lf)
    check(got, bk, bv, pk)
    assert st.table_slots == table_slots(nb, 50 << 20, load_factor=lf)
    assert st.paths & abi.JOIN_PATH_PROBE_SEG, hex(st.paths)


@pytest.mark.parametrize("path,env,filt,bit", [
    ("direct", dict(TG_PROBE_PARTITION="0"), None, abi.JOIN_PATH_PROBE_DIRECT),
    ("segment", PART, None, abi.JOIN_PATH_PROBE_SEG),
    ("unique key", {}, [FilterItem(abi.CMP_GE, 1, const_i64=0)], abi.JOIN_PATH_PROBE_UQ),
    ("general", dict(TG_PROBE_UQ="0"), [FilterItem(abi.CMP_GE, 1, const_i64=0)], abi.JOIN_PATH_PROBE_GENERAL),
])
def test_dense_table_every_probe_path(path, env, filt, bit, monkeypatch):
    setenv(monkeypatch, env)
    bk, bv, pk = make_sides(60_001, 500_001, 0.5, seed=7)
    got, st = run_host(bk, bv, pk, 0.9, filt)
    check(got, bk, bv, pk)
    assert st.paths & bit == bit, (path, hex(st.paths))


def test_dense_table_skewed_probe_takes_the_fallback(monkeypatch):
    # 70 % of the probe rows carry one key: a segment overflows and the gated direct launch probes the dense table
    setenv(monkeypatch, PART)
    bk, bv, pk = make_sides(80_001, 1_000_000, 1.0, seed=5)
    pk[np.random.default_rng(1).random(len(pk)) < 0.7] = bk[0]
    got, st = run_host(bk, bv, pk, 0.9)
    check(got, bk, bv, pk)
    assert st.paths & abi.JOIN_PATH_PROBE_DIRECT


def _device_join(nb, npr, lf, dup=False):
    import torch
    from tidb_b200.device import DeviceJoin, fetch_device
    from tidb_b200.plan import FieldType
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev); g.manual_seed(11)
    bk = torch.randperm(nb, device=dev, generator=g, dtype=torch.int64) * (2 * 0x9E3779B1) + 5
    if dup:
        bk[: nb // 10] = bk[nb // 10: 2 * (nb // 10)]
    bv = torch.arange(nb, device=dev, dtype=torch.int64) * 3
    pk = torch.where(torch.rand(npr, device=dev, generator=g) < 0.5, bk[torch.randint(0, nb, (npr,), device=dev, generator=g)],
                     torch.randint(0, 1 << 60, (npr,), device=dev, generator=g) * 2)   # misses: even, build keys are odd
    pv = torch.arange(npr, device=dev, dtype=torch.int64)
    torch.cuda.synchronize(dev)   # the join reads its inputs on a stream of its own: they must be written first
    INT = FieldType(abi.TYPE_LONGLONG, abi.FLAG_NOT_NULL)
    plan = JoinPlan(abi.JOIN_INNER, [INT, INT], [INT, INT], [0], [0], build_is_right=True, device=0, load_factor=lf)
    j = DeviceJoin(plan)
    j.build([bk, bv])
    rows, cols, _ = j.probe([pk, pv], sync=True)
    st = j.stats()
    got = [fetch_device(p, rows * 8).view(np.int64) for p in cols]
    j.close()
    return [x.cpu().numpy() for x in (bk, bv, pk)], got, st, torch.cuda.get_device_properties(0).L2_cache_size


def test_densified_default_table_device_input(monkeypatch):
    # 6 M unique keys at the default load factor: the U1 table is rebuilt for 16 L2-sized slices, device-resident input
    setenv(monkeypatch, {})
    (bk, bv, pk), got, st, l2 = _device_join(6_000_000, 20_000_000, 0.0)
    assert st.table_mode == 1 and st.table_slots == table_slots(6_000_000, l2) < table_slots(6_000_000, l2, u1=False)
    assert st.paths & (abi.JOIN_PATH_PROBE_SEG | abi.JOIN_PATH_SCATTER_BULK) == abi.JOIN_PATH_PROBE_SEG | abi.JOIN_PATH_SCATTER_BULK
    check(got, bk, bv, pk)


def test_dense_table_explicit_load_factor_device_input(monkeypatch):
    setenv(monkeypatch, {})
    (bk, bv, pk), got, st, l2 = _device_join(6_000_000, 20_000_000, 0.9)
    assert st.table_slots == table_slots(6_000_000, l2, load_factor=0.9)
    check(got, bk, bv, pk)


def test_g_table_keeps_its_sizing(monkeypatch):
    # duplicate build keys: a G table at the default load factor is not densified
    setenv(monkeypatch, {})
    (bk, bv, pk), got, st, l2 = _device_join(6_000_000, 1_000_000, 0.0, dup=True)
    assert st.table_mode == 2 and st.table_slots == table_slots(6_000_000, l2, u1=False)
