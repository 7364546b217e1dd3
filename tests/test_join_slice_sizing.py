"""The sizing rule of the join table and of the L2 partition pass (tidb_b200/csrc/join.cu: build_table, l2_slice_target,
probe_slices), restated in Python.  The GPU tests check the library's table_slots against table_slots() below; the tests
in this file pin the rule's values for the H100's L2."""
import math

SLOT = 16                  # bytes per table slot {int64 key, u64 meta}
MAX_PARTS = 16             # TG_MAX_PARTS
MAX_DENSE_LOAD = 0.5       # kMaxDenseLoad
PART_MIN_MB = 64           # TG_PROBE_PART_MIN_MB default
HOME_WIDTH = 4             # kHomeWidth: the slot count is a multiple of it
H100_L2 = 50 << 20         # cudaDevAttrL2CacheSize of an H100 SXM


def slice_target(l2_bytes):
    return l2_bytes // 4


def probe_slices(table_bytes, l2_bytes):
    return min(-(-table_bytes // slice_target(l2_bytes)), MAX_PARTS)


def table_slots(n, l2_bytes, load_factor=None, u1=True):
    """slots of the table a build of n rows gets (load_factor None = the default)"""
    default = load_factor is None
    nslots = int(max(n, 1) / (0.35 if default else load_factor)) + 32
    if default and nslots > MAX_PARTS * (33 << 20) // SLOT:
        nslots = max(MAX_PARTS * (33 << 20) // SLOT, int(max(n, 1) / 0.5) + 32)
    nslots &= ~(HOME_WIDTH - 1)
    if u1 and default and n > 0:
        dense = max(MAX_PARTS * slice_target(l2_bytes) // SLOT, int(n / MAX_DENSE_LOAD) + 32) & ~(HOME_WIDTH - 1)
        part_min = PART_MIN_MB << 20
        if nslots * SLOT > part_min and dense < nslots and dense * SLOT > part_min:
            nslots = dense
    return nslots


def test_bench_shape_on_h100():
    # 10 M unique keys, one payload: load factor 0.5 (the cap), 16 slices of 19.1 MiB instead of 14 of 31 MiB
    n = 10_000_000
    s = table_slots(n, H100_L2)
    assert s == 20_000_032
    assert abs(n / s - MAX_DENSE_LOAD) < 1e-5
    assert probe_slices(s * SLOT, H100_L2) == 16
    assert round(s * SLOT / 16 / 2**20, 1) == 19.1
    # the same build side without the rule (a G table): 28.6 M slots
    old = table_slots(n, H100_L2, u1=False)
    assert old == 28_571_460 and probe_slices(old * SLOT, H100_L2) == 16


def test_dense_enough_for_the_target_below_the_cap():
    # 6 M keys: 16 slices of exactly the target (12.5 MiB) need load factor 0.46 only
    s = table_slots(6_000_000, H100_L2)
    assert s == MAX_PARTS * slice_target(H100_L2) // SLOT == 13_107_200
    assert probe_slices(s * SLOT, H100_L2) == 16 and s * SLOT // 16 == 12.5 * 2**20


def test_tables_that_stay_as_they_are():
    # small tables (no partition pass), tables already within 16 target slices, explicit load factors, G tables
    assert table_slots(1_000_000, H100_L2) == int(1_000_000 / 0.35) + 32 & ~3
    assert table_slots(4_000_000, H100_L2) == int(4_000_000 / 0.35) + 32 & ~3          # 183 MB <= 16 x 12.5 MiB
    assert table_slots(10_000_000, H100_L2, load_factor=0.35) == 28_571_460
    assert table_slots(10_000_000, H100_L2, u1=False) == 28_571_460
    assert table_slots(101, H100_L2) % 4 == 0


def test_slices_follow_l2():
    # a device with half the L2 gets slices of half the size and a table twice as dense, up to the cap
    assert slice_target(H100_L2 // 2) == slice_target(H100_L2) // 2
    assert probe_slices(457 << 20, H100_L2 // 2) == 16
    assert probe_slices(100 << 20, H100_L2) == math.ceil((100 << 20) / (12.5 * 2**20)) == 8
