"""Tile size of the join's L2 partition pass (k_partition_scatter_bulk): dense probe input with one or two scattered columns
takes 4096-row tiles, segmented input (capacities in multiples of 1024 rows) and three or more columns take 1024-row tiles,
and the rows behind the last whole tile ride on the gated direct launch.  Every case compares every output row with the
numpy reference as a sorted multiset and asserts which tile size ran (JOIN_SCATTER_TILE_4K)."""
import numpy as np
import pytest

from tidb_b200 import abi
from test_gpu_join_inplace import INT, assert_mode, check, expected, make_sides, run_dev, setenv

pytestmark = pytest.mark.gpu

NB = 40_000
TILE = 4096
BULK, TILE_4K = abi.JOIN_PATH_SCATTER_BULK, abi.JOIN_SCATTER_TILE_4K


def assert_tiles(st, npr, big):
    """fewer than one 4096-row tile: the direct probe alone; else the bulk scatter with the tiles `big` says"""
    if npr < TILE:
        assert not st.paths & (BULK | TILE_4K | abi.JOIN_PATH_PROBE_SEG), hex(st.paths)
    else:
        assert st.paths & BULK and st.paths & abi.JOIN_PATH_PROBE_SEG, hex(st.paths)
        assert bool(st.paths & TILE_4K) == big, (hex(st.paths), big)
    assert st.paths & abi.JOIN_PATH_PROBE_DIRECT, hex(st.paths)


@pytest.mark.parametrize("npr", [2047, 2048, 3072, 4095, 4096, 4097, 6144, 150 * TILE - 1, 150 * TILE + 1, 500 * TILE - 1, 500 * TILE + 1])
@pytest.mark.parametrize("match,mode", [(1.0, "1"), (0.6, "0"), (0.6, "1")])   # in place, lean, in place with misses
def test_probe_sizes_around_the_tile(npr, match, mode, monkeypatch):
    setenv(monkeypatch, mode)
    bk, bv, pcols = make_sides(NB, npr, match, seed=npr % 1009)
    got, names, launches, st = run_dev(bk, bv, pcols)
    check(got, expected(bk, bv, pcols, [0, 1], [0, 1]))
    assert_tiles(st, npr, True)
    if npr >= TILE:   # one tail behind the 4096-row tiles costs no launch of its own
        assert_mode(names, launches, mode == "1")


def test_skewed_probe_overflows_a_segment(monkeypatch):
    # 70 % of the rows carry one key: a segment overflows the 4096-row scatter, the in-place probe exits and the gated direct
    # launch probes the original input, the < 4096-row tail with it
    setenv(monkeypatch, "1")
    npr = 100 * TILE + 3999
    bk, bv, pcols = make_sides(NB, npr, 1.0, seed=51)
    pcols[0][np.random.default_rng(51).random(npr) < 0.7] = bk[5]
    got, _, _, st = run_dev(bk, bv, pcols)
    check(got, expected(bk, bv, pcols, [0, 1], [0, 1]))
    assert_tiles(st, npr, True)


@pytest.mark.parametrize("ncols,lused,rused", [(3, [0, 1, 2], [0]), (4, [0, 1, 2, 3], [1])])
def test_three_or_four_columns_take_1024_row_tiles(ncols, lused, rused, monkeypatch):
    # a 4096-row tile of 3-4 columns does not fit in shared memory: the scatter keeps 1024-row tiles, and its tail stays < 1024 rows
    setenv(monkeypatch, "1")
    npr = 100 * TILE + 1500
    bk, bv, pcols = make_sides(NB, npr, 1.0, seed=52, ncols=ncols)
    got, names, launches, st = run_dev(bk, bv, pcols, lused, rused)
    check(got, expected(bk, bv, pcols, lused, rused))
    assert_tiles(st, npr, False)
    assert_mode(names, launches, True)


@pytest.mark.parametrize("nseg,cap,fill", [
    (3, 301 * 1024, [301 * 1024, 12_345, 301 * 1024 - 1]),   # an odd multiple of 1024: 4096-row tiles would straddle segments
    (2, 1024, [1024, 1000]),                                 # one tile per segment
])
def test_segmented_input_takes_1024_row_tiles(nseg, cap, fill, monkeypatch):
    import torch
    from tidb_b200.device import DeviceJoin, fetch_device
    from tidb_b200.plan import JoinPlan
    setenv(monkeypatch, None)
    monkeypatch.setenv("TG_PROBE_PARTS", "6")
    rng = np.random.default_rng(53)
    bk, bv, _ = make_sides(NB, 1, 1.0, seed=53)
    kcol, vcol = np.full(nseg * cap, -7, dtype=np.int64), np.full(nseg * cap, -9, dtype=np.int64)   # padding never matches
    pk, pv = [], []
    for s, f in enumerate(fill):
        k = np.where(rng.random(f) < 0.9, bk[rng.integers(0, NB, f)], rng.integers(0, 1 << 61, f) * 2)
        v = np.arange(f, dtype=np.int64) + s * 10_000_000
        kcol[s * cap:s * cap + f], vcol[s * cap:s * cap + f] = k, v
        pk.append(k), pv.append(v)
    pcols = [np.concatenate(pk), np.concatenate(pv)]
    t = lambda a: torch.from_numpy(a).cuda()
    j = DeviceJoin(JoinPlan(abi.JOIN_INNER, [INT, INT], [INT, INT], [0], [0], build_is_right=True))
    try:
        j.build([t(bk), t(bv)])
        rows, cols, _ = j.probe_segments([t(kcol), t(vcol)], t(np.array(fill, dtype=np.int64)), cap, sync=True)
        torch.cuda.synchronize()
        got = [fetch_device(p, rows * 8).view(np.int64) for p in cols]
        st = j.stats()
    finally:
        j.close()
    check(got, expected(bk, bv, pcols, [0, 1], [0, 1]))
    assert st.paths & BULK and not st.paths & TILE_4K, hex(st.paths)
