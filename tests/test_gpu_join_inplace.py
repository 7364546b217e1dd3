"""The in-place segment probe of the partitioned unique-key join: the partition pass scatters the probe columns straight into
the output columns, the probe writes the build side in place (compacting tiles with misses) and a hole fill makes the
output dense.  Every output row is compared with a numpy reference as a sorted multiset, in the forced modes
(TG_PROBE_INPLACE=1 / 0) and in the automatic one.  The mode a call took is read from the library's launch count and, when
the capture holds the kernel records, from torch.profiler's kernel names."""
import numpy as np
import pytest

from tidb_b200 import abi
from tidb_b200.chunk import Chunk, Column
from tidb_b200.executor import HashJoinExec, MockDataSource
from tidb_b200.plan import FieldType, JoinPlan

pytestmark = pytest.mark.gpu

SENTINEL = -(1 << 63)
INT = FieldType(abi.TYPE_LONGLONG, abi.FLAG_NOT_NULL)
PART = dict(TG_PROBE_PARTITION="1", TG_PROBE_PARTS="8", TG_PROBE_PART_MIN_MB="0", TG_PROBE_PART_MIN_ROWS="0")
INPLACE, LEAN, FILL, SCATTER = "k_probe_inner_u1_seg_inplace", "k_probe_inner_u1_seg_lean", "k_inplace_fill", "k_partition_scatter_bulk"
PIDX = "k_probe_inner_u1_seg_inplace_pidx"   # the in-place probe through the slice index (its name contains INPLACE)
# kernels one partitioned probe of dense input enqueues (stats.kernel_launches): k_segment_bases, the scatter, the segment
# probe and the gated k_probe_inner_u1_w; in place adds k_inplace_holes, the three scan kernels and k_inplace_fill
LAUNCHES = {True: 9, False: 4}


def setenv(monkeypatch, mode):
    for k in ("TG_PROBE_PARTITION", "TG_PROBE_PARTS", "TG_PROBE_UQ", "TG_PROBE_INPLACE", "TG_PROBE_CTAS_PER_SM"):
        monkeypatch.delenv(k, raising=False)
    for k, v in PART.items():
        monkeypatch.setenv(k, v)
    if mode is not None:
        monkeypatch.setenv("TG_PROBE_INPLACE", mode)


def make_sides(nb, npr, match, seed, ncols=2):
    """unique odd build keys (the sentinel among them); probe key = a build key with probability `match`, else an even miss;
    probe column c > 0 = row * (c + 1) + c, so every probe row is distinct in every column"""
    rng = np.random.default_rng(seed)
    bk = rng.permutation(nb).astype(np.int64) * 2 * 0x9E3779B1 + 1
    bk[0] = SENTINEL
    bv = np.arange(nb, dtype=np.int64) * 3 + 7
    miss = rng.integers(0, 1 << 61, npr).astype(np.int64) * 2
    pk = np.where(rng.random(npr) < match, bk[rng.integers(0, nb, npr)], miss)
    rows = np.arange(npr, dtype=np.int64)
    return bk, bv, [pk] + [rows * (c + 1) + c for c in range(1, ncols)]


def expected(bk, bv, pcols, lused, rused):
    order = np.argsort(bk)
    sb = bk[order]
    pos = np.minimum(np.searchsorted(sb, pcols[0]), len(bk) - 1)
    hit = sb[pos] == pcols[0]
    bcols = [bk[order[pos[hit]]], bv[order[pos[hit]]]]
    return [pcols[c][hit] for c in lused] + [bcols[c] for c in rused]


def sorted_rows(cols):
    a = np.stack(cols, axis=1) if cols[0].size else np.zeros((0, len(cols)), np.int64)
    return a[np.lexsort(a.T[::-1])] if len(a) else a


def check(got, exp):
    assert len(got) == len(exp)
    assert len(got[0]) == len(exp[0]), (len(got[0]), len(exp[0]))
    assert np.array_equal(sorted_rows(got), sorted_rows(exp))


def kernels_of(fn):
    """(fn's result, names of the CUDA kernels it launched)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        r = fn()
        torch.cuda.synchronize()
    return r, {e.name for e in prof.events()}


def ran(names, kernel):
    return any(kernel in n for n in names)


def assert_mode(names, launches, inplace, index=False):
    """the call took the in-place probe (else the lean one); in place, through the table's slice index (PIDX) or not"""
    assert launches == LAUNCHES[inplace], (launches, inplace)
    # a torch.profiler capture can come back without its kernel records (only the runtime API calls): the scatter runs in
    # both modes, so a capture that names it holds the kernels; test_profiler_names_the_mode_kernels requires one
    if ran(names, SCATTER):
        linear = any(INPLACE in n and PIDX not in n for n in names)
        assert linear == (inplace and not index) and ran(names, PIDX) == (inplace and index), names
        assert ran(names, FILL) == inplace and ran(names, LEAN) != inplace, names


class Dev:
    """one device-resident join handle (tg_join_probe_dev)"""

    def __init__(self, bk, bv, ncols, lused=None, rused=None):
        import torch
        from tidb_b200.device import DeviceJoin
        self.torch = torch
        self.lused = list(range(ncols)) if lused is None else lused
        self.rused = [0, 1] if rused is None else rused
        plan = JoinPlan(abi.JOIN_INNER, [INT] * ncols, [INT, INT], [0], [0], build_is_right=True, lused=lused, rused=rused)
        self.j = DeviceJoin(plan)
        self.j.build([torch.from_numpy(bk).cuda(), torch.from_numpy(bv).cuda()])
        torch.cuda.synchronize()

    def probe(self, pcols):
        from tidb_b200.device import fetch_device
        t = [self.torch.from_numpy(c).cuda() for c in pcols]
        self.torch.cuda.synchronize()
        l0 = self.j.stats().kernel_launches
        (rows, cols, _), names = kernels_of(lambda: self.j.probe(t, sync=True))
        return [fetch_device(p, rows * 8).view(np.int64) for p in cols], names, self.j.stats().kernel_launches - l0

    def close(self):
        self.j.close()


def run_dev(bk, bv, pcols, lused=None, rused=None):
    d = Dev(bk, bv, len(pcols), lused, rused)
    got, names, launches = d.probe(pcols)
    st = d.j.stats()
    d.close()
    return got, names, launches, st


@pytest.mark.parametrize("mode", ["1", "0", None])
@pytest.mark.parametrize("npr", [300_001, 262_144])   # with and without a < 1024-row tail behind the scatter
def test_full_match(mode, npr, monkeypatch):
    setenv(monkeypatch, mode)
    bk, bv, pcols = make_sides(40_000, npr, 1.0, seed=1)
    got, names, launches, st = run_dev(bk, bv, pcols)
    check(got, expected(bk, bv, pcols, [0, 1], [0, 1]))
    assert_mode(names, launches, mode != "0")   # auto: the first call of a handle takes the in-place probe
    assert st.paths & abi.JOIN_PATH_PROBE_SEG


@pytest.mark.parametrize("mode", ["1", "0"])
def test_profiler_names_the_mode_kernels(mode, monkeypatch):
    setenv(monkeypatch, mode)
    bk, bv, pcols = make_sides(40_000, 300_001, 1.0, seed=9)
    for _ in range(3):   # a capture without kernel records is taken again (a fresh handle: the same call)
        got, names, launches, _ = run_dev(bk, bv, pcols)
        check(got, expected(bk, bv, pcols, [0, 1], [0, 1]))
        if ran(names, SCATTER):
            break
    assert ran(names, SCATTER), names
    assert_mode(names, launches, mode == "1")


@pytest.mark.parametrize("match", [0.0, 0.5, 0.99, "one miss"])
def test_partial_match_forced_in_place(match, monkeypatch):
    setenv(monkeypatch, "1")
    bk, bv, pcols = make_sides(40_000, 300_001, 1.0 if match == "one miss" else match, seed=2)
    if match == "one miss":
        pcols[0][123_457] = 2
    got, names, launches, _ = run_dev(bk, bv, pcols)
    check(got, expected(bk, bv, pcols, [0, 1], [0, 1]))
    assert_mode(names, launches, True)


@pytest.mark.parametrize("mode", ["1", "0"])
def test_sentinel_probe_keys(mode, monkeypatch):
    # the key value that marks empty slots: matched through the side slot, in full tiles and in a segment's partial tile
    setenv(monkeypatch, mode)
    bk, bv, pcols = make_sides(40_000, 300_001, 1.0, seed=3)
    pcols[0][np.random.default_rng(3).integers(0, len(pcols[0]), 2000)] = SENTINEL
    got, _, _, _ = run_dev(bk, bv, pcols)
    check(got, expected(bk, bv, pcols, [0, 1], [0, 1]))
    bk2 = bk.copy()
    bk2[0] = 5                                                  # the sentinel on the probe side only: a miss
    got, _, _, _ = run_dev(bk2, bv, pcols)
    check(got, expected(bk2, bv, pcols, [0, 1], [0, 1]))


def test_skewed_probe_overflows_a_segment(monkeypatch):
    # 70 % of the rows carry one key: a segment overflows, the in-place probe and the hole fill exit, the gated direct
    # launch probes the original input
    setenv(monkeypatch, "1")
    bk, bv, pcols = make_sides(40_000, 400_000, 1.0, seed=4)
    pcols[0][np.random.default_rng(4).random(len(pcols[0])) < 0.7] = bk[5]
    got, _, _, st = run_dev(bk, bv, pcols)
    check(got, expected(bk, bv, pcols, [0, 1], [0, 1]))
    assert st.paths & abi.JOIN_PATH_PROBE_DIRECT


OUTPUT_SHAPES = [   # (probe columns, lused, rused); test_gpu_slice_index runs them through the slice index
    (2, None, None),            # NPC 1, NKD 2 (probe and build key), NMD 1
    (2, [0, 1], [1]),           # the pruned 3-column plan: NKD 1
    (2, [1], [0, 1]),           # NKD 1 fed by the build key only
    (2, [0], [0, 1]),           # NPC 0
    (3, [0, 1, 2], [0]),        # NPC 2, NMD 0
    (4, [0, 1, 2, 3], [1]),     # NPC 3, NKD 1
    (2, [1], [1]),              # no output fed by the key (NKD 0): not eligible
]


def run_shape(ncols, lused, rused, match, nb, npr, seed):
    """one forced in-place call of the output shape against its reference -> (kernel names, launches, stats, whether the
    shape is eligible for the in-place probe: an output fed by the join key)"""
    bk, bv, pcols = make_sides(nb, npr, match, seed=seed, ncols=ncols)
    got, names, launches, st = run_dev(bk, bv, pcols, lused, rused)
    lu = list(range(ncols)) if lused is None else lused
    ru = [0, 1] if rused is None else rused
    check(got, expected(bk, bv, pcols, lu, ru))
    return names, launches, st, 0 in lu or 0 in ru


@pytest.mark.parametrize("ncols,lused,rused", OUTPUT_SHAPES)
@pytest.mark.parametrize("match", [1.0, 0.6])
def test_output_shapes(ncols, lused, rused, match, monkeypatch):
    setenv(monkeypatch, "1")
    names, launches, _, eligible = run_shape(ncols, lused, rused, match, 30_000, 200_003, seed=5)
    assert_mode(names, launches, eligible)


@pytest.mark.parametrize("mode", ["1", "0", None])
def test_host_pushed_input(mode, monkeypatch):
    # tg_join_probe_push / tg_join_next: the result batches carry the segment-sized output columns
    setenv(monkeypatch, mode)
    bk, bv, pcols = make_sides(40_000, 700_001, 1.0, seed=6)
    plan = JoinPlan(abi.JOIN_INNER, [INT, INT], [INT, INT], [0], [0])
    e = HashJoinExec(plan, MockDataSource(plan.left_types, [Chunk([Column(c) for c in pcols])]),
                     MockDataSource(plan.right_types, [Chunk([Column(bk), Column(bv)])]))
    e.open()
    chunks = []
    while True:
        c = e.next(100_000)
        if c.num_rows() == 0:
            break
        chunks.append(c)
    st = e.stats()
    e.close()
    got = [np.concatenate([c.columns[i].data for c in chunks]) for i in range(4)]
    check(got, expected(bk, bv, pcols, [0, 1], [0, 1]))
    assert st.paths & abi.JOIN_PATH_PROBE_SEG


def test_mode_follows_the_last_match_fraction(monkeypatch):
    setenv(monkeypatch, None)
    bk, bv, full = make_sides(40_000, 300_001, 1.0, seed=7)
    _, _, half = make_sides(40_000, 300_001, 0.5, seed=8)
    d = Dev(bk, bv, 2)
    try:
        # first call: in place; the next call follows the match fraction of the one before it
        for pcols, inplace in ((full, True), (half, True), (full, False), (full, True)):
            got, names, launches = d.probe(pcols)
            check(got, expected(bk, bv, pcols, [0, 1], [0, 1]))
            assert_mode(names, launches, inplace)
    finally:
        d.close()
