"""The slice index of a big unique-key table (SliceIndex, join_kernels.cuh): a U1 table the partitioned probe slices gets a
per-slice hash-and-displace index, and the in-place segment probe looks each row up with one pilot byte and one 16-byte
slot.  Every output row is compared with a numpy reference as a sorted multiset, with the in-place probe (which takes the
index) and the lean one (which keeps the linear-probe table) forced.  The table needs about 4.6 M keys before the build
densifies it for slicing, so these tests build 4.7 M to 10 M,
some of them crafted key by key (slice_index_model.craft_build)."""
import numpy as np
import pytest

from tidb_b200 import abi
from test_gpu_join_inplace import SENTINEL, Dev, check, expected, make_sides, setenv

pytestmark = pytest.mark.gpu

NB, NPR = 5_000_000, 2_000_001
GOLD = 0x9E3779B97F4A7C15
M64 = (1 << 64) - 1


def run(bk, bv, pcols):
    d = Dev(bk, bv, len(pcols))
    got, _, _ = d.probe(pcols)
    st = d.j.stats()
    d.close()
    return got, st


def key_of_hash(h):
    """the int64 key whose hash64 (k ^ (k >> 32)) * GOLD is h"""
    kp = (h * pow(GOLD, -1, 1 << 64)) & M64
    hi, lo = kp >> 32, kp & 0xFFFFFFFF
    k = (hi << 32) | (lo ^ hi)
    assert (((k ^ (k >> 32)) * GOLD) & M64) == h
    return k - (1 << 64) if k >= 1 << 63 else k


@pytest.mark.parametrize("mode", ["1", "0"])
@pytest.mark.parametrize("match", [1.0, 0.5, 0.0])
def test_match_fractions(mode, match, monkeypatch):
    setenv(monkeypatch, mode)
    bk, bv, pcols = make_sides(NB, NPR, match, seed=11)
    got, st = run(bk, bv, pcols)
    check(got, expected(bk, bv, pcols, [0, 1], [0, 1]))
    assert st.paths & abi.JOIN_PATH_PROBE_SEG


@pytest.mark.parametrize("mode", ["1", "0"])
def test_sentinel_probe_keys(mode, monkeypatch):
    # the key value that marks empty slots is never in the index: its tiles take the linear-probe table's side slot
    setenv(monkeypatch, mode)
    bk, bv, pcols = make_sides(NB, NPR, 1.0, seed=12)
    pcols[0][np.random.default_rng(12).integers(0, NPR, 3000)] = SENTINEL
    got, st = run(bk, bv, pcols)
    check(got, expected(bk, bv, pcols, [0, 1], [0, 1]))
    assert st.paths & abi.JOIN_PATH_PROBE_SEG


@pytest.mark.parametrize("mode", ["1", "0"])
def test_unplaced_bucket(mode, monkeypatch):
    # 40 keys with one partition and one bucket (the same top and low hash bits): more than a bucket may hold, so the bucket
    # gets no pilot and its keys are found through the linear-probe table
    setenv(monkeypatch, mode)
    bk, bv, pcols = make_sides(NB, NPR, 1.0, seed=13)
    crafted = np.array([key_of_hash(((0x01000000 + 977 * i) << 32) | 0x5A5A5A5A) for i in range(40)], dtype=np.int64)
    bk[1:41] = crafted
    rng = np.random.default_rng(13)
    pcols[0][rng.integers(0, NPR, 20_000)] = crafted[rng.integers(0, 40, 20_000)]
    got, st = run(bk, bv, pcols)
    check(got, expected(bk, bv, pcols, [0, 1], [0, 1]))
    assert st.paths & abi.JOIN_PATH_PROBE_SEG


def test_skewed_probe_overflows_a_segment(monkeypatch):
    # 70 % of the rows carry one key: a segment overflows, the index probe exits and the gated direct launch probes the
    # original input
    setenv(monkeypatch, "1")
    bk, bv, pcols = make_sides(NB, NPR, 1.0, seed=14)
    pcols[0][np.random.default_rng(14).random(NPR) < 0.7] = bk[5]
    got, st = run(bk, bv, pcols)
    check(got, expected(bk, bv, pcols, [0, 1], [0, 1]))
    assert st.paths & abi.JOIN_PATH_PROBE_DIRECT


# ---- the index path, observed: every case below compares every output row with the numpy reference and asserts, from
# JOIN_PATH_PROBE_INDEX on a fresh handle or from the kernel names of one call, whether the in-place probe took the index;
# slice_index_model says when it must.

import slice_index_model as M
from test_gpu_join_inplace import OUTPUT_SHAPES, assert_mode, run_shape
from test_join_slice_sizing import H100_L2, probe_slices, table_slots

INDEX = abi.JOIN_PATH_PROBE_INDEX


def auto_parts(nb):
    """the slice count the build and the probe pick without TG_PROBE_PARTS (16 for every size here)"""
    return probe_slices(table_slots(nb, H100_L2) * 16, H100_L2)


def index_expected(bk, p_build, p_probe=None):
    """the in-place probe of a fresh handle takes the slice index: the build rebuilt the table dense for slicing, sized
    the index for the P the probe uses, and its pilots fit in shared memory"""
    p_probe = p_build if p_probe is None else p_probe
    sliced = table_slots(len(bk), H100_L2) < table_slots(len(bk), H100_L2, u1=False)
    return sliced and p_build == p_probe and M.index_params(M.part_counts(bk, p_build), p_build)[2]


def assert_index(st, want):
    assert bool(st.paths & INDEX) == want, (hex(st.paths), want)
    assert st.paths & abi.JOIN_PATH_PROBE_SEG


def setparts(monkeypatch, parts):
    if parts is None:
        monkeypatch.delenv("TG_PROBE_PARTS", raising=False)
    else:
        monkeypatch.setenv("TG_PROBE_PARTS", str(parts))


def probe_side(bk, npr, match, seed, ncols=2):
    """probe key = a build key with probability `match`, else a random int64 (a miss unless it hits by chance: the
    reference decides); column c > 0 = row * (c + 1) + c"""
    rng = np.random.default_rng(seed)
    pk = np.where(rng.random(npr) < match, bk[rng.integers(0, len(bk), npr)],
                  rng.integers(-(1 << 63), (1 << 63) - 1, npr, dtype=np.int64))
    rows = np.arange(npr, dtype=np.int64)
    return [pk] + [rows * (c + 1) + c for c in range(1, ncols)]


def payload(bk):
    return np.arange(len(bk), dtype=np.int64) * 3 + 7


@pytest.mark.parametrize("parts", [2, 4, 7, 8, 9, 11, 13, 16, None])
@pytest.mark.parametrize("match", [1.0, 0.6])
def test_slice_counts(parts, match, monkeypatch):
    # non-power-of-two P cut the hash range unevenly (mulhi32): the scatter and the index must cut it alike
    setenv(monkeypatch, "1")
    setparts(monkeypatch, parts)
    bk, bv, pcols = make_sides(NB, NPR, match, seed=21)
    P = parts or auto_parts(NB)
    want = index_expected(bk, P)
    assert want == (P >= 8)
    got, st = run(bk, bv, pcols)
    check(got, expected(bk, bv, pcols, [0, 1], [0, 1]))
    assert_index(st, want)


@pytest.mark.parametrize("mx", [655_356, 655_357])
def test_pilot_byte_boundary(mx, monkeypatch):
    # the fullest of 8 slices at the last key count whose pilots fit kPidxMaxPilotBytes, and one key beyond it
    setenv(monkeypatch, "1")
    counts = [600_000 + 1000 * p for p in range(8)]
    counts[3] = mx
    bk, _ = M.craft_build(counts, 8, seed=mx)
    assert M.index_params(counts, 8)[1:] == ((163_840, True) if mx == 655_356 else (163_856, False))
    assert index_expected(bk, 8) == (mx == 655_356)
    bv = payload(bk)
    pcols = probe_side(bk, NPR, 1.0, seed=22)
    got, st = run(bk, bv, pcols)
    check(got, expected(bk, bv, pcols, [0, 1], [0, 1]))
    assert_index(st, mx == 655_356)


def in_buckets(keys, P, B, buckets):
    """keys whose (slice, bucket) is one of `buckets`"""
    h = M.hash64(keys)
    gid = M.slot32(h, P).astype(np.int64) * B + M.pidx_bucket(h, B).astype(np.int64)
    return np.isin(gid, [p * B + b for p, b in buckets])


CRAFTED = {
    # name: (P, keys per slice, crafted buckets (slice, bucket, size), slice that gets no key or None)
    "bucket of 32": (8, [600_000] * 8, [(2, None, M.MAX_BUCKET)], None),
    "bucket of 33": (8, [600_000] * 8, [(5, None, M.MAX_BUCKET + 1)], None),
    # 550 buckets of 33 keys per slice: 3 % of the keys unplaced, so nearly every full tile takes inplace_tile_generic
    "oversized everywhere": (8, [600_000] * 8, [(p, None, 33) for p in range(8) for _ in range(550)], None),
    "empty slice": (16, [330_000] * 5 + [0] + [330_000] * 10, [], 5),
    "one slice twice the mean": (16, [312_500] * 9 + [625_000] + [312_500] * 6, [], None),
}


@pytest.mark.parametrize("case", list(CRAFTED))
def test_crafted_buckets(case, monkeypatch):
    setenv(monkeypatch, "1")
    P, counts, buckets, empty = CRAFTED[case]
    setparts(monkeypatch, P)
    bk, chosen = M.craft_build(counts, P, buckets, seed=23)
    _, B, built = M.index_params(counts, P)
    assert built and index_expected(bk, P)
    bv = payload(bk)
    pcols = probe_side(bk, NPR, 1.0, seed=24)
    rng = np.random.default_rng(25)
    if chosen:
        # a tenth of the probe rows take keys of the crafted buckets
        crafted = bk[in_buckets(bk, P, B, [(p, b) for p, b, _ in chosen])]
        assert len(crafted) == sum(size for _, _, size in chosen)
        rows = rng.choice(NPR, NPR // 10, replace=False)
        pcols[0][rows] = crafted[rng.integers(0, len(crafted), len(rows))]
    if empty is not None:
        # a tenth of the probe rows hash into the slice without build keys: all misses
        rows = rng.choice(NPR, NPR // 10, replace=False)
        pcols[0][rows] = M.key_of_hash(M.hashes_in_slice(rng, empty, P, len(rows)))
    got, st = run(bk, bv, pcols)
    exp = expected(bk, bv, pcols, [0, 1], [0, 1])
    check(got, exp)
    if empty is not None:
        assert len(exp[0]) < NPR * 0.95
    assert_index(st, True)


@pytest.mark.parametrize("ncols,lused,rused", OUTPUT_SHAPES)
@pytest.mark.parametrize("match", [1.0, 0.6])
def test_output_shapes_through_the_index(ncols, lused, rused, match, monkeypatch):
    # the shapes of test_gpu_join_inplace.test_output_shapes at index scale: each eligible shape runs its own
    # instantiation of the index kernel; the ineligible one (no output fed by the key) takes the lean probe
    setenv(monkeypatch, "1")
    names, launches, st, eligible = run_shape(ncols, lused, rused, match, NB, NPR, seed=26)
    assert_mode(names, launches, eligible, index=eligible)
    assert bool(st.paths & INDEX) == eligible, hex(st.paths)


@pytest.mark.parametrize("npr", [0, 1000, 1000 * 1024, 1000 * 1024 + 1023])
def test_probe_sizes(npr, monkeypatch):
    # 0 rows launch nothing; fewer than 1024 rows leave the partition pass nothing to scatter and take the direct probe
    # (through the partition pass they were all lost: the gated launch reads a tail that starts at row 0 as no tail); a
    # multiple of 1024 has no tail; 1023 rows is the longest tail, probed by the gated launch behind the index probe
    setenv(monkeypatch, "1")
    bk, bv, pcols = make_sides(NB, npr, 1.0, seed=27)
    assert index_expected(bk, 8)
    d = Dev(bk, bv, 2)
    try:
        if npr:
            got, names, launches = d.probe(pcols)
            if npr >= 1024:
                assert_mode(names, launches, True, index=True)
        else:
            import torch
            rows, _, _ = d.j.probe([torch.empty(0, dtype=torch.int64, device="cuda")] * 2, sync=True)
            assert rows == 0
            got = [np.zeros(0, np.int64)] * 4
        check(got, expected(bk, bv, pcols, [0, 1], [0, 1]))
        st = d.j.stats()
        assert bool(st.paths & INDEX) == bool(st.paths & abi.JOIN_PATH_PROBE_SEG) == (npr >= 1024), hex(st.paths)
        assert bool(st.paths & abi.JOIN_PATH_PROBE_DIRECT) == (npr > 0), hex(st.paths)
    finally:
        d.close()


def test_unaligned_probe_column(monkeypatch):
    # a key column that starts 8 bytes into its allocation is not 16-byte aligned: no partition pass, no index, the
    # direct probe, the same rows
    import torch
    from tidb_b200.device import fetch_device
    setenv(monkeypatch, "1")
    bk, bv, pcols = make_sides(NB, NPR, 1.0, seed=28)
    d = Dev(bk, bv, 2)
    try:
        base = torch.empty(NPR + 1, dtype=torch.int64, device="cuda")
        key = base[1:]
        key.copy_(torch.from_numpy(pcols[0]))
        assert key.data_ptr() % 16 == 8
        rows, cols, _ = d.j.probe([key, torch.from_numpy(pcols[1]).cuda()], sync=True)
        got = [fetch_device(p, rows * 8).view(np.int64) for p in cols]
        check(got, expected(bk, bv, pcols, [0, 1], [0, 1]))
        st = d.j.stats()
        assert st.paths & abi.JOIN_PATH_PROBE_DIRECT and not st.paths & (INDEX | abi.JOIN_PATH_PROBE_SEG), hex(st.paths)
    finally:
        d.close()


def test_mode_sequence_through_the_index(monkeypatch):
    # test_gpu_join_inplace.test_mode_follows_the_last_match_fraction at index scale: in place (through the index) while
    # the last call matched in full, lean after the half-matched one.  assert_mode reads the kernel names when the
    # capture holds its kernel records; the path bit shows that the handle's first call took the index.
    setenv(monkeypatch, None)
    bk, bv, full = make_sides(NB, NPR, 1.0, seed=29)
    half = probe_side(bk, NPR, 0.5, seed=30)
    assert index_expected(bk, 8)
    d = Dev(bk, bv, 2)
    try:
        for i, (pcols, inplace) in enumerate(((full, True), (half, True), (full, False), (full, True))):
            got, names, launches = d.probe(pcols)
            check(got, expected(bk, bv, pcols, [0, 1], [0, 1]))
            assert_mode(names, launches, inplace, index=inplace)
            if i == 0:
                assert d.j.stats().paths & INDEX
    finally:
        d.close()


def seg_capacity(n, P, fills=None, n_learned=None):
    """inplace_seg_cap (join.cu): C0 = 1.05·n_main/P + 16 K, or from the largest fill a synced call learned"""
    n_main = n // 1024 * 1024
    c0 = (int(n_main / P * 1.05) + 16384 + 127) // 128 * 128
    if fills is None:
        return c0
    f = max(fills) * n_main / n_learned
    return min((int(f + 8.0 * f ** 0.5) + 4096 + 127) // 128 * 128, c0)


def test_learned_capacity_then_overflow(monkeypatch):
    # call 2 sizes its segments from call 1's fills and takes the index; call 3 puts 20 K extra rows on one key, beyond
    # the learned capacity but within the first call's: its segment overflows, the index probe exits and the gated
    # direct launch probes the original input
    setenv(monkeypatch, "1")
    P = 8
    bk, bv, first = make_sides(NB, NPR, 1.0, seed=31)
    second = probe_side(bk, NPR, 1.0, seed=32)
    third = probe_side(bk, NPR, 1.0, seed=33)
    third[0][np.random.default_rng(33).choice(NPR, 20_000, replace=False)] = bk[11]
    # fills of the P segments: the scatter takes the first n_main rows, the sentinel key included
    fills = [np.bincount(M.slot32(M.hash64(c[0][:NPR // 1024 * 1024]), P).astype(np.int64), minlength=P) for c in (first, second, third)]
    learned = seg_capacity(NPR, P, fills[0], NPR // 1024 * 1024)
    assert max(fills[1]) <= learned < seg_capacity(NPR, P)
    assert learned < max(fills[2]) <= seg_capacity(NPR, P)
    d = Dev(bk, bv, 2)
    try:
        for i, pcols in enumerate((first, second, third)):
            got, names, launches = d.probe(pcols)
            check(got, expected(bk, bv, pcols, [0, 1], [0, 1]))
            assert_mode(names, launches, True, index=True)
            if i == 0:
                assert d.j.stats().paths & INDEX
        assert d.j.stats().paths & abi.JOIN_PATH_PROBE_DIRECT
    finally:
        d.close()


@pytest.mark.parametrize("p_build,p_probe", [(8, 16), (16, 8)])
def test_parts_changed_after_the_build(p_build, p_probe, monkeypatch):
    # the index is cut for the P of the build: a probe with another P must keep to the linear-probe table
    setenv(monkeypatch, "1")
    setparts(monkeypatch, p_build)
    bk, bv, pcols = make_sides(NB, NPR, 1.0, seed=34)
    assert index_expected(bk, p_build) and not index_expected(bk, p_build, p_probe)
    d = Dev(bk, bv, 2)
    try:
        setparts(monkeypatch, p_probe)
        got, names, launches = d.probe(pcols)
        check(got, expected(bk, bv, pcols, [0, 1], [0, 1]))
        assert_mode(names, launches, True, index=False)
        assert_index(d.j.stats(), False)
    finally:
        d.close()


@pytest.mark.parametrize("mode", ["1", None])
def test_host_pushed_input_through_the_index(mode, monkeypatch):
    from tidb_b200.chunk import Chunk, Column
    from tidb_b200.executor import HashJoinExec, MockDataSource
    from tidb_b200.plan import JoinPlan
    from test_gpu_join_inplace import INT
    setenv(monkeypatch, mode)
    bk, bv, pcols = make_sides(NB, NPR, 1.0, seed=35)
    assert index_expected(bk, 8)
    plan = JoinPlan(abi.JOIN_INNER, [INT, INT], [INT, INT], [0], [0])
    e = HashJoinExec(plan, MockDataSource(plan.left_types, [Chunk([Column(c) for c in pcols])]),
                     MockDataSource(plan.right_types, [Chunk([Column(bk), Column(bv)])]))
    e.open()
    chunks = []
    while True:
        c = e.next(100_000)
        if c.num_rows() == 0:
            break
        assert c.num_rows() <= 100_000
        chunks.append(c)
    st = e.stats()
    e.close()
    got = [np.concatenate([c.columns[i].data for c in chunks]) for i in range(4)]
    check(got, expected(bk, bv, pcols, [0, 1], [0, 1]))
    assert_index(st, True)


@pytest.mark.parametrize("nb", [4_700_000, 5_000_000, 10_000_000])
@pytest.mark.parametrize("seed", range(5))
def test_placement_keeps_the_index(nb, seed, monkeypatch):
    # the verify pass (k_pidx_write, check = 1) drops the index when a placed key is not at its slot: a placement race
    # in k_pidx_place would show here as a missing bit.  Automatic P (16 slices).
    setenv(monkeypatch, "1")
    setparts(monkeypatch, None)
    bk, bv, pcols = make_sides(nb, NPR, 1.0, seed=100 + seed)
    assert index_expected(bk, auto_parts(nb))
    got, st = run(bk, bv, pcols)
    check(got, expected(bk, bv, pcols, [0, 1], [0, 1]))
    assert_index(st, True)


def test_two_devices(monkeypatch):
    # the index kernel's shared-memory limit is a per-device attribute: a join on a second device of the same process
    # must launch it as well as the first
    import torch
    from tidb_b200.device import DeviceJoin, fetch_device
    from tidb_b200.plan import JoinPlan
    from test_gpu_join_inplace import INT
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two CUDA devices")
    setenv(monkeypatch, "1")
    for dev in (0, 1):
        bk, bv, pcols = make_sides(NB, NPR, 1.0, seed=40 + dev)
        assert index_expected(bk, 8)
        j = DeviceJoin(JoinPlan(abi.JOIN_INNER, [INT, INT], [INT, INT], [0], [0], build_is_right=True, device=dev))
        try:
            j.build([torch.from_numpy(bk).to(f"cuda:{dev}"), torch.from_numpy(bv).to(f"cuda:{dev}")])
            with torch.cuda.device(dev):
                rows, cols, _ = j.probe([torch.from_numpy(c).to(f"cuda:{dev}") for c in pcols], sync=True)
            got = [fetch_device(p, rows * 8, device=dev).view(np.int64) for p in cols]
            check(got, expected(bk, bv, pcols, [0, 1], [0, 1]))
            assert_index(j.stats(), True)
        finally:
            j.close()
