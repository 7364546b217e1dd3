"""The slice index at more than 16 slices, where the index probe holds two slices' pilots and sweeps them without a
CTA-wide barrier (k_probe_inner_u1_seg_inplace_pidx with SliceIndex.nbuf = 2): every output row is compared with the
exact numpy reference as a sorted multiset, at P = 17, 24 and 32 and at the automatic P (16 slices, where a 5 M-key
table's pilots also fit twice), with a segment overflow, a bucket without a pilot, and probes whose P is not the
index's."""
import numpy as np
import pytest

from tidb_b200 import abi
import slice_index_model as M
from test_gpu_join_inplace import Dev, assert_mode, check, expected, make_sides, setenv
from test_gpu_slice_index import NB, NPR, payload, probe_side, setparts
from test_index_slices import index_slices, pilot_buffers
from test_join_slice_sizing import H100_L2, table_slots

pytestmark = pytest.mark.gpu

INDEX = abi.JOIN_PATH_PROBE_INDEX


def run(bk, bv, pcols, monkeypatch=None, probe_parts=None):
    """build, then probe once (with TG_PROBE_PARTS = probe_parts, unset for None, when monkeypatch is given)"""
    d = Dev(bk, bv, len(pcols))
    try:
        if monkeypatch is not None:
            setparts(monkeypatch, probe_parts)
        got, names, launches = d.probe(pcols)
        return got, names, launches, d.j.stats()
    finally:
        d.close()


def two_buffers(bk, P):
    _, B, built = M.index_params(M.part_counts(bk, P), P)
    return built and pilot_buffers(B) == 2


@pytest.mark.parametrize("parts", [17, 24, 32, None])
@pytest.mark.parametrize("match", [1.0, 0.6])
def test_slice_counts_beyond_16(parts, match, monkeypatch):
    setenv(monkeypatch, "1")
    setparts(monkeypatch, parts)
    bk, bv, pcols = make_sides(NB, NPR, match, seed=51)
    P = parts or index_slices(table_slots(NB, H100_L2) * 16, H100_L2)
    assert P == (parts or 16) and two_buffers(bk, P)
    got, names, launches, st = run(bk, bv, pcols)
    check(got, expected(bk, bv, pcols, [0, 1], [0, 1]))
    assert_mode(names, launches, True, index=True)
    assert st.paths & INDEX, hex(st.paths)


@pytest.mark.parametrize("parts", [32, None])
def test_skewed_probe_overflows_a_segment(parts, monkeypatch):
    # 60 % of the rows carry one key: its segment overflows, the index probe exits before it loads any pilots and the
    # gated direct launch probes the original input
    setenv(monkeypatch, "1")
    setparts(monkeypatch, parts)
    bk, bv, pcols = make_sides(NB, NPR, 1.0, seed=52)
    pcols[0][np.random.default_rng(52).random(NPR) < 0.6] = bk[7]
    got, _, _, st = run(bk, bv, pcols)
    check(got, expected(bk, bv, pcols, [0, 1], [0, 1]))
    assert st.paths & abi.JOIN_PATH_PROBE_DIRECT, hex(st.paths)


@pytest.mark.parametrize("size", [M.MAX_BUCKET, M.MAX_BUCKET + 1])
def test_bucket_without_a_pilot_at_32_slices(size, monkeypatch):
    # one bucket of 33 keys gets pilot 255: tiles with its keys take the linear-probe table; a bucket of 32 is placed
    setenv(monkeypatch, "1")
    P = 32
    setparts(monkeypatch, P)
    counts = [156_000] * P
    bk, chosen = M.craft_build(counts, P, [(9, None, size)], seed=53)
    _, B, built = M.index_params(counts, P)
    assert built and pilot_buffers(B) == 2
    bv = payload(bk)
    pcols = probe_side(bk, NPR, 1.0, seed=54)
    h = M.hash64(bk)
    (p, b, _), = chosen
    crafted = bk[(M.slot32(h, P) == p) & (M.pidx_bucket(h, B) == b)]
    assert len(crafted) == size
    rng = np.random.default_rng(55)
    rows = rng.choice(NPR, NPR // 10, replace=False)
    pcols[0][rows] = crafted[rng.integers(0, size, len(rows))]
    got, names, launches, st = run(bk, bv, pcols)
    check(got, expected(bk, bv, pcols, [0, 1], [0, 1]))
    assert_mode(names, launches, True, index=True)


@pytest.mark.parametrize("p_build,p_probe", [(None, 24), (24, 32), (32, 24), (32, None), (16, None)])
def test_probe_with_another_p_than_the_index(p_build, p_probe, monkeypatch):
    # the index is cut for the P of the build: a probe with another P keeps to the linear-probe table.  (16, None): the
    # automatic P of the probe is 16 as well, so it takes the index
    setenv(monkeypatch, "1")
    setparts(monkeypatch, p_build)
    bk, bv, pcols = make_sides(NB, NPR, 1.0, seed=56)
    got, names, launches, st = run(bk, bv, pcols, monkeypatch, p_probe)
    check(got, expected(bk, bv, pcols, [0, 1], [0, 1]))
    index = (p_build or 16) == (p_probe or 16)
    assert_mode(names, launches, True, index=index)
    assert bool(st.paths & INDEX) == index, hex(st.paths)


def test_mode_sequence_at_the_automatic_p(monkeypatch):
    # at 60 % match the handle turns to the lean probe, which keeps the linear-probe table
    setenv(monkeypatch, None)
    setparts(monkeypatch, None)
    bk, bv, full = make_sides(NB, NPR, 1.0, seed=57)
    part = probe_side(bk, NPR, 0.6, seed=58)
    d = Dev(bk, bv, 2)
    try:
        for pcols, inplace in ((full, True), (part, True), (part, False), (full, False), (full, True)):
            got, names, launches = d.probe(pcols)
            check(got, expected(bk, bv, pcols, [0, 1], [0, 1]))
            assert_mode(names, launches, inplace, index=inplace)
    finally:
        d.close()
