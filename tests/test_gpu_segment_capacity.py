"""Segment capacity of the in-place segment probe, learned per handle: after a partitioned call whose row count the host read,
the next in-place call of the same handle sizes its segments from that call's fills instead of 1.05·n/P + 16 K.  One handle
probes a sequence of batches that tighten the capacity, reuse it without a host read, overflow it, change the row count
and drop the match fraction; every output row of every call is compared with a numpy reference as a sorted multiset."""
import numpy as np
import pytest

from test_gpu_join_inplace import INT, check, expected, make_sides, setenv
from tidb_b200 import abi
from tidb_b200.plan import JoinPlan

pytestmark = pytest.mark.gpu

NB = 40_000
PARTS = 8   # TG_PROBE_PARTS of test_gpu_join_inplace.PART


class Handle:
    """one device-resident join handle (tg_join_probe_dev); probe() with or without the host reading the row count"""

    def __init__(self, bk, bv):
        import torch
        from tidb_b200.device import DeviceJoin
        self.torch = torch
        self.j = DeviceJoin(JoinPlan(abi.JOIN_INNER, [INT, INT], [INT, INT], [0], [0], build_is_right=True))
        self.j.build([torch.from_numpy(bk).cuda(), torch.from_numpy(bv).cuda()])
        torch.cuda.synchronize()

    def probe(self, pcols, want_rows, sync):
        from tidb_b200.device import fetch_device
        t = [self.torch.from_numpy(c).cuda() for c in pcols]
        rows, cols, _ = self.j.probe(t, sync=sync)
        self.torch.cuda.synchronize()
        if sync:
            assert rows == want_rows, (rows, want_rows)
        # without a host read the output is still dense in [0, rows): its first want_rows rows are the whole result
        return [fetch_device(p, want_rows * 8).view(np.int64) for p in cols]

    def close(self):
        self.j.close()


def hot_key(pcols, bk, extra, seed):
    """`extra` random probe rows take one build key: its segment holds about n/P + extra rows, beyond a capacity learned
    from uniform fills (n/P + a few sqrt(n/P) + 4 K) but within 1.05·n/P + 16 K"""
    out = [c.copy() for c in pcols]
    out[0][np.random.default_rng(seed).choice(len(out[0]), extra, replace=False)] = bk[11]
    return out


def run_sequence(h, bk, bv, calls):
    for pcols, sync in calls:
        exp = expected(bk, bv, pcols, [0, 1], [0, 1])
        check(h.probe(pcols, len(exp[0]), sync), exp)


@pytest.mark.parametrize("overflow_sync", [True, False])
def test_learned_capacity_sequence(overflow_sync, monkeypatch):
    setenv(monkeypatch, None)
    npr = 600_000   # 75 K rows per segment: sigma of a fill ~ 270 rows
    bk, bv, uni_a = make_sides(NB, npr, 1.0, seed=21)
    _, _, uni_b = make_sides(NB, npr, 1.0, seed=22)
    _, _, uni_c = make_sides(NB, npr, 1.0, seed=23)
    _, _, other_n = make_sides(NB, 417_793, 1.0, seed=24)    # a different n, with a < 1024-row tail
    _, _, half = make_sides(NB, npr, 0.5, seed=25)
    skew = hot_key(uni_c, bk, 12_000, seed=26)
    h = Handle(bk, bv)
    try:
        run_sequence(h, bk, bv, [
            (uni_a, True),               # formula capacity; the host reads the fills: the next call's capacity tightens
            (uni_b, False),              # learned capacity, no host read
            (skew, overflow_sync),       # one segment overflows the learned capacity: the gated direct probe does the work
            (uni_c, True),               # after a read overflow: the formula again, and the fills are learned anew
            (other_n, True),             # the learned fill scaled to another n
            (half, True),                # 50 % match, still in place (the last call matched in full), learned capacity
            (uni_a, True),               # the lean segment probe (the last call matched half), formula capacity
            (uni_a, True),               # in place again
        ])
    finally:
        h.close()


@pytest.mark.parametrize("sync_between", [True, False])
def test_tail_not_a_multiple_of_the_tile(sync_between, monkeypatch):
    setenv(monkeypatch, None)
    bk, bv, a = make_sides(NB, 500_001, 1.0, seed=31)
    _, _, b = make_sides(NB, 500_001 + 777, 1.0, seed=32)
    _, _, c = make_sides(NB, 499_713, 1.0, seed=33)
    h = Handle(bk, bv)
    try:
        run_sequence(h, bk, bv, [(a, True), (b, sync_between), (c, True), (a, False), (b, True)])
    finally:
        h.close()


def test_skewed_key_set_learned(monkeypatch):
    # a systematically skewed probe side: the learned capacity carries the skew, so the same kind of batch fits again
    setenv(monkeypatch, None)
    bk, bv, a = make_sides(NB, 600_000, 1.0, seed=41)
    _, _, b = make_sides(NB, 600_000, 1.0, seed=42)
    a, b = hot_key(a, bk, 9_000, seed=43), hot_key(b, bk, 9_000, seed=44)
    h = Handle(bk, bv)
    try:
        run_sequence(h, bk, bv, [(a, True), (b, False), (b, True), (a, True)])
    finally:
        h.close()
