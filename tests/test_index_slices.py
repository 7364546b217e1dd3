"""The slice count of a sliced unique-key table's index and the pilot buffers of the index probe (tidb_b200/csrc/join.cu:
probe_slices, build_slice_index), restated in Python and pinned at the bench shape on an H100: 10 M build keys id * ODD."""
import numpy as np

import slice_index_model as M
from test_join_slice_sizing import H100_L2, probe_slices, table_slots

MAX_SLICES = 32                  # TG_MAX_SLICES
SHARED_OPTIN = 227 << 10         # cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100
ODD = 0x9E3779B97F4A7C15         # bench.py's key multiplier


def index_slices(table_bytes, l2_bytes, parts_override=0):
    """the index is cut for the partitioned probe's P: probe_slices, TG_PROBE_PARTS up to TG_MAX_SLICES"""
    if parts_override > 0:
        return min(parts_override, MAX_SLICES)
    return probe_slices(table_bytes, l2_bytes)


def pilot_buffers(B):
    """SliceIndex.nbuf: two when two slices' pilots fit kPidxMaxPilotBytes (and, with their mbarriers, shared memory)"""
    return 2 if 2 * B <= M.MAX_PILOT_BYTES and 2 * (B + 8) <= SHARED_OPTIN else 1


def bench_keys(n=10_000_000):
    with np.errstate(over="ignore"):
        return (np.arange(n, dtype=np.uint64) * np.uint64(ODD)).view(np.int64)


def test_bench_shape_keeps_16_slices_with_one_pilot_buffer():
    bk = bench_keys()
    slots = table_slots(len(bk), H100_L2)
    P = index_slices(slots * 16, H100_L2)
    assert P == 16
    S, B, built = M.index_params(M.part_counts(bk, P), P)
    assert built and (S, B) == (894_713, 156_576)            # 13.7 MiB slices, 152.9 KiB of pilots per slice
    assert pilot_buffers(B) == 1
    # at 32 slices (TG_PROBE_PARTS=32) two buffers of 76.6 KiB fit
    _, B32, built32 = M.index_params(M.part_counts(bk, 32), 32)
    assert built32 and B32 == 78_432 and pilot_buffers(B32) == 2


def test_override_sets_the_index_slices():
    slots = table_slots(10_000_000, H100_L2)
    assert [index_slices(slots * 16, H100_L2, p) for p in (8, 16, 17, 24, 32, 40)] == [8, 16, 17, 24, 32, 32]


def test_pilot_buffer_boundary():
    half = M.MAX_PILOT_BYTES // 2
    assert pilot_buffers(half) == 2 and pilot_buffers(half + 16) == 1
