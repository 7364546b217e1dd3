"""The slice-index rules of slice_index_model.py pinned at the values the GPU tests and the benchmark rely on: the
pilot-byte limit, the slice counts that get an index for a 5 M-key table and for the benchmark's 10 M keys, and build
sides crafted to put chosen numbers of keys in chosen slices and buckets."""
import os
import re

import numpy as np
import pytest

import slice_index_model as M
from tidb_b200 import abi
from test_join_slice_sizing import H100_L2, probe_slices, table_slots

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def uniform_keys(n, seed):
    # the build keys of test_gpu_join_inplace.make_sides: unique odd multiples, the sentinel among them
    k = np.random.default_rng(seed).permutation(n).astype(np.int64) * 2 * 0x9E3779B1 + 1
    k[0] = M.SENTINEL
    return k


def test_header_probe_index_path_bit():
    # tg_join_stats.paths bit 8 marks the index probe; the Python mirror carries the header's value, and bit 4 stays free
    hdr = open(os.path.join(ROOT, "include", "tidbgpu.h")).read()
    m = re.search(r"\bTG_JOIN_PATH_PROBE_INDEX = (0x[0-9a-fA-F]+|\d+)", hdr)
    assert m and int(m.group(1), 0) == 1 << 8 == abi.JOIN_PATH_PROBE_INDEX
    others = [int(h, 16) if h else 1 << int(s)
              for h, s in re.findall(r"\bTG_JOIN_PATH_(?!PROBE_INDEX\b)[A-Z0-9_]+ = (?:0x([0-9a-fA-F]+)|1 << (\d+))", hdr)]
    assert len(others) == 7 and abi.JOIN_PATH_PROBE_INDEX not in others and 1 << 4 not in others


def test_hash_matches_the_scalar_definition():
    rng = np.random.default_rng(1)
    keys = np.concatenate([rng.integers(-(1 << 63), (1 << 63) - 1, 1000, dtype=np.int64),
                           np.array([0, 1, -1, M.SENTINEL, (1 << 63) - 1], np.int64)])
    M64 = (1 << 64) - 1
    for k, h in zip(keys.tolist(), M.hash64(keys).tolist()):
        u = k & M64
        assert h == ((u ^ (u >> 32)) * M.GOLD) & M64
        assert int(M.slot32(np.array([h], np.uint64), 13)[0]) == ((h >> 32) * 13) >> 32
        assert int(M.pidx_bucket(np.array([h], np.uint64), 163_840)[0]) == ((h & 0xFFFFFFFF) * 163_840) >> 32


def test_key_of_hash_inverts_the_hash():
    rng = np.random.default_rng(2)
    h = rng.integers(0, 1 << 64, 100_000, dtype=np.uint64)
    assert np.array_equal(M.hash64(M.key_of_hash(h)), h)
    keys = rng.integers(-(1 << 63), (1 << 63) - 1, 100_000, dtype=np.int64)
    assert np.array_equal(M.key_of_hash(M.hash64(keys)), keys)


def test_pilot_byte_boundary():
    # B = (ceil(mx / 4) + 16) & ~15 reaches kPidxMaxPilotBytes at 655,356 keys in the fullest slice
    assert M.index_params([655_356] + [600_000] * 7, 8) == (936_224, 163_840, True)
    S, B, built = M.index_params([600_000] * 7 + [655_357], 8)
    assert (B, built) == (163_856, False) and S == 936_226
    assert M.index_params([655_356], 1)[2] is False   # one slice: no partitioned probe, no index


def test_5m_uniform_keys_get_an_index_from_8_slices():
    keys = uniform_keys(5_000_000, 11)
    for P in range(2, 17):
        c = M.part_counts(keys, P)
        assert c.sum() == len(keys) - 1
        S, B, built = M.index_params(c, P)
        assert built == (P >= 8), (P, c.max(), B)
    # the table is sliced (rebuilt dense) at this size, and the automatic slice count is 16
    assert table_slots(5_000_000, H100_L2) < table_slots(5_000_000, H100_L2, u1=False)
    assert probe_slices(table_slots(5_000_000, H100_L2) * 16, H100_L2) == 16


def test_bench_shape_is_about_4_percent_under_the_limit():
    keys = uniform_keys(10_000_000, 0)
    P = probe_slices(table_slots(10_000_000, H100_L2) * 16, H100_L2)
    assert P == 16
    S, B, built = M.index_params(M.part_counts(keys, P), P)
    assert built and 0.03 < 1 - B / M.MAX_PILOT_BYTES < 0.06, B
    # the build side at which the mean slice alone reaches the limit: about 10.5 M keys
    assert 10_400_000 < 16 * 655_356 < 10_500_000


@pytest.mark.parametrize("P", [8, 13, 16])
def test_crafted_keys_land_in_the_slice_and_bucket_asked_for(P):
    counts = [40_000 + 1000 * p for p in range(P)]
    counts[P // 2] = 0
    buckets = [(0, None, 32), (1, None, 33), (2, 7, 1), (P - 1, None, 50)]
    keys, chosen = M.craft_build(counts, P, buckets, seed=P)
    assert len(np.unique(keys)) == len(keys) == sum(counts) and not (keys == M.SENTINEL).any()
    assert np.array_equal(M.part_counts(keys, P), counts)
    _, B, _ = M.index_params(counts, P)
    sizes = M.bucket_sizes(keys, P, B)
    for p, b, size in chosen:
        assert sizes[p, b] == size
    assert (2, 7, 1) in chosen
    assert sizes[P // 2].sum() == 0
