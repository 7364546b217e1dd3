"""The slice index of a big unique-key table (SliceIndex, join_kernels.cuh): a U1 table the partitioned probe slices gets a
per-slice hash-and-displace index, and the in-place segment probe looks each row up with one pilot byte and one 16-byte
slot.  Every output row is compared with a numpy reference as a sorted multiset, with the in-place probe (which takes the
index) and the lean one (which keeps the linear-probe table) forced.  The table needs about 4.6 M keys before the build
densifies it for slicing, so these tests build 5 M."""
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
