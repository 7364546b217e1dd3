"""The repartition and exchange kernels of the multi-GPU path, run on ONE device against exact numpy references:
tg_partition_by_key / tg_partition_count, the counted exchange (tg_partition_exchange), the count-free exchange with and
without a spill area (tg_partition_exchange_cf / _cf_ex / _cf_spill), tg_peer_copy_regions and the mailboxes
(tg_mail_signal / tg_mail_wait).  A simulated world of W senders writes into W local "peer" receive buffers, so everything
but the NVLink transport (tests/test_gpu_multigpu.py) runs on a one-GPU machine.

Data conventions: column c of sender s holds gid * MUL[c] + ADD[c] with gid = s << 24 | row, so every output row can be
traced to its source row; a lost, duplicated or mixed row fails.  Order inside a destination run is undefined (the CTAs
reserve their runs with atomics): runs are compared as multisets, counts, offsets and flags exactly.  Every destination
buffer, region and spill area is followed by GUARD rows of SENT that must stay untouched."""
import ctypes as C
import threading

import numpy as np
import pytest

from tidb_b200 import abi
from tidb_b200.parallel import exchange_by_key_host, exchange_segments_host, partition_of_keys_np, recv_bases, region_capacity

pytestmark = pytest.mark.gpu

SENT = -0x2152411021524111
GUARD = 2048
MUL = [3, 5, 7, 9, 11, 13, 15, 17]
ADD = [101, 202, 303, 404, 505, 606, 707, 808]
HOT = 0x5DEECE66D          # the key a skewed input puts on 60 % of its rows
M40 = (1 << 40) - 1


def torch():
    import torch as t
    return t


def lib():
    return abi.load_lib()


def ptr(t):
    return C.c_void_p(t.data_ptr())


def parr(ts):
    return (C.c_void_p * len(ts))(*[t.data_ptr() for t in ts])


def payload(s, rows, ncols):
    gid = (np.int64(s) << 24) | np.arange(rows, dtype=np.int64)
    return [gid * MUL[c] + ADD[c] for c in range(ncols)]


def skewed(cols, seed):
    """cols with the key column rewritten to HOT on 60 % of the rows"""
    rng = np.random.default_rng(seed)
    return [np.where(rng.random(len(cols[0])) < 0.6, np.int64(HOT), cols[0])] + cols[1:]


def guarded(n, shift=0):
    """a device column of n legal rows followed by GUARD rows of SENT; shift=1 starts it one element (8 bytes) past a 16-byte
    boundary.  -> (the column view, the whole buffer)"""
    buf = torch().full((n + shift + GUARD,), SENT, dtype=torch().int64, device="cuda")
    return buf[shift:shift + n], buf


def upload(a, shift=0):
    view, buf = guarded(len(a), shift)
    if len(a):
        view.copy_(torch().from_numpy(np.ascontiguousarray(a)))
    return view, buf


def host(t):
    return t.cpu().numpy()


def assert_guard(tail, what):
    g = host(tail)
    assert np.all(g == SENT), f"{what}: {int(np.sum(g != SENT))} guard rows written"


def rows_of(cols):
    """rows of a column set, lexicographically sorted (multiset comparison)"""
    a = np.stack([np.asarray(c) for c in cols], axis=1) if len(cols[0]) else np.zeros((0, len(cols)), np.int64)
    return a[np.lexsort(a.T[::-1])] if len(a) else a


def same_rows(got, exp, what=""):
    assert len(got[0]) == len(exp[0]), (what, len(got[0]), len(exp[0]))
    assert np.array_equal(rows_of(got), rows_of(exp)), what


def row_index(got, cols_in, s):
    """source row of every output row, identified by column 1 (column 0 when it is the only one); every other column must
    be that row's value too.  -> local row indices"""
    c = 1 if len(cols_in) > 1 else 0
    g = np.asarray(got[c])
    ok = (g - ADD[c]) % MUL[c] == 0
    gid = (g - ADD[c]) // MUL[c]
    i = gid - (np.int64(s) << 24)
    ok &= (i >= 0) & (i < len(cols_in[0]))
    assert ok.all(), f"{int((~ok).sum())} output rows are no source row (sentinel or corrupted)"
    for k in range(len(cols_in)):
        assert np.array_equal(np.asarray(got[k]), cols_in[k][i]), f"column {k} does not travel with its row"
    return i


def destinations(key, nparts, notnull=None):
    """destination of every row: hash of the key, of the row index for a NULL key (row_part in partition_kernels.cuh)"""
    d = partition_of_keys_np(key, nparts)
    if notnull is not None:
        nul = ~notnull
        d[nul] = partition_of_keys_np(np.nonzero(nul)[0].astype(np.int64), nparts)
    return d


def kernels_of(fn):
    """(fn's result, names of the CUDA kernels it launched)"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        r = fn()
        torch().cuda.synchronize()
    return r, {e.name for e in prof.events()}


def routes(names):
    r = set()
    for n in names:
        if "k_partition_count4" in n:
            r.add("count4")
        elif "k_partition_count" in n:
            r.add("count")
        elif "k_partition_scatter_bulk" in n:
            r.add("bulk")
        elif "k_partition_scatter" in n:
            r.add("lsu")
    return r


def assert_routes(names, want):
    # a torch.profiler capture can come back without its kernel records; one that holds any partition kernel holds them all
    got = routes(names)
    if got:
        assert got == want, (sorted(got), sorted(want))


# ---- A. tg_partition_by_key and tg_partition_count -----------------------------------------------------------------------

BY_KEY = [
    # (P, rows, ncols, route)
    (1, 1025, 1, "aligned"), (2, 1024, 2, "aligned"), (3, 2049, 3, "aligned"), (7, 1_000_003, 4, "aligned"),
    (8, 1023, 2, "aligned"), (13, 1, 1, "aligned"), (16, 0, 4, "aligned"), (16, 2049, 5, "aligned"),
    (13, 1_000_003, 8, "aligned"), (3, 1024, 8, "aligned"),
    (2, 2049, 2, "src_shift"), (16, 1_000_003, 3, "src_shift"), (7, 1023, 5, "src_shift"), (1, 1024, 1, "src_shift"),
    (3, 1025, 4, "dst_shift"), (13, 1024, 2, "dst_shift"), (8, 1_000_003, 1, "dst_shift"),
    (7, 2049, 1, "key_sep"), (16, 1025, 3, "key_sep"), (2, 1_000_003, 8, "key_sep"),
    (8, 2049, 2, "null10"), (13, 1_000_003, 4, "null10"), (1, 1023, 5, "null10"),
    (16, 1025, 1, "null100"), (3, 1_000_003, 2, "null100"), (2, 1, 3, "null100"),
]


class ByKeyCase:
    """inputs, destination buffers and reference of one tg_partition_by_key call"""

    def __init__(self, P, rows, ncols, route, seed):
        rng = np.random.default_rng(seed)
        self.P, self.rows, self.ncols, self.route = P, rows, ncols, route
        self.cols = payload(0, rows, ncols)
        src_shift = 1 if route == "src_shift" else 0
        self.src = [upload(c, src_shift) for c in self.cols]
        if route == "key_sep":              # the key is not among the moved columns
            self.key_np = rng.integers(-(1 << 62), 1 << 62, rows).astype(np.int64)
            self.key = upload(self.key_np)[0]
        else:
            self.key_np, self.key = self.cols[0], self.src[0][0]
        self.notnull, self.nulls = None, None
        if route.startswith("null"):
            self.notnull = rng.random(rows) >= (0.1 if route == "null10" else 1.0)
            bm = np.packbits(self.notnull, bitorder="little") if rows else np.zeros(1, np.uint8)
            self.nulls = torch().from_numpy(np.concatenate([bm, np.zeros(16, np.uint8)])).cuda()
        self.dst = [guarded(rows, 1 if (route == "dst_shift" and c == 0) else 0) for c in range(ncols)]
        self.offs = guarded(P + 1)
        self.counts = guarded(P)
        self.dest = destinations(self.key_np, P, self.notnull)

    def call(self, stream=None):
        return lib().tg_partition_by_key(0, ptr(self.key), ptr(self.nulls) if self.nulls is not None else None, C.c_int64(self.rows),
                                         self.P, self.ncols, parr([v for v, _ in self.src]), parr([v for v, _ in self.dst]),
                                         ptr(self.offs[0]), stream)

    def count(self):
        return lib().tg_partition_count(0, ptr(self.key), C.c_int64(self.rows), self.P, ptr(self.counts[0]), None)

    def want_routes(self):
        if self.rows == 0:
            return set()
        count = "count4" if self.nulls is None and self.route != "src_shift" else "count"
        bulk = self.nulls is None and self.ncols <= 4 and self.route == "aligned"
        if not bulk:
            return {count, "lsu"}
        return {count} | ({"bulk"} if self.rows >= 1024 else set()) | ({"lsu"} if self.rows % 1024 else set())

    def check(self):
        P, n = self.P, self.rows
        o = host(self.offs[0])
        exp_cnt = np.bincount(self.dest, minlength=P)
        assert o[0] == 0 and o[P] == n, o
        assert np.array_equal(np.diff(o), exp_cnt), (np.diff(o), exp_cnt)
        assert_guard(self.offs[1][P + 1:], "offsets")
        got = [host(v) for v, _ in self.dst]
        for c, (v, buf) in enumerate(self.dst):
            assert_guard(buf[buf.numel() - GUARD:], f"destination column {c}")
        i = row_index(got, self.cols, 0)
        assert np.array_equal(np.sort(i), np.arange(n)), "not a permutation of the input rows"
        part_at = np.searchsorted(o, np.arange(n), side="right") - 1
        assert np.array_equal(self.dest[i], part_at), "a row sits outside its destination's range"


@pytest.mark.parametrize("P,rows,ncols,route", BY_KEY)
def test_partition_by_key_vs_reference(P, rows, ncols, route):
    case = ByKeyCase(P, rows, ncols, route, seed=P * 1000 + ncols)
    torch().cuda.synchronize()
    codes, names = kernels_of(lambda: (case.call(), case.count() if case.nulls is None else 0))
    assert codes == (0, 0), (codes, lib().tg_last_error())
    case.check()
    assert_routes(names, case.want_routes())
    if case.nulls is None:
        assert np.array_equal(host(case.counts[0]), np.bincount(case.dest, minlength=P))
        assert_guard(case.counts[1][P:], "counts")


def test_partition_count_packed_counters_flush():
    """k_partition_count4 packs 8 counters of 8 bits per register and flushes them at pending > 240.  With
    n = 2 * 32 * 4 * (SMs * 8 * 256) + 1 rows every thread of the full grid runs exactly 32 iterations of 8 rows, reaching the
    flush threshold with 248 rows in one lane; the odd n takes the last-key branch."""
    t = torch()
    sms = t.cuda.get_device_properties(0).multi_processor_count
    n = 2 * 32 * 4 * (sms * 8 * 256) + 1
    counts = guarded(16)
    key = t.arange(n, dtype=t.int64, device="cuda")
    t.cuda.synchronize()
    code, names = kernels_of(lambda: lib().tg_partition_count(0, ptr(key), C.c_int64(n), 1, ptr(counts[0]), None))
    assert code == 0
    assert_routes(names, {"count4"})
    assert int(host(counts[0])[0]) == n
    del key
    k = 0x123456789
    key = t.full((n,), k, dtype=t.int64, device="cuda")
    t.cuda.synchronize()
    assert lib().tg_partition_count(0, ptr(key), C.c_int64(n), 16, ptr(counts[0]), None) == 0
    want = np.zeros(16, np.int64)
    want[partition_of_keys_np(np.array([k], np.int64), 16)[0]] = n
    assert np.array_equal(host(counts[0]), want)
    assert_guard(counts[1][16:], "counts")


def test_partition_by_key_two_threads():
    """two host threads, two streams, 8 calls each: the counted calls share one per-device scratch behind a mutex"""
    t = torch()
    cases = [[ByKeyCase(5, 200_003 + 1000 * i, 2, "aligned", seed=i) for i in range(8)],
             [ByKeyCase(16, 150_001 + 777 * i, 6, "null10", seed=100 + i) for i in range(8)]]
    streams = [t.cuda.Stream(), t.cuda.Stream()]
    t.cuda.synchronize()
    codes = [[], []]

    def run(k):
        for case in cases[k]:
            codes[k].append(case.call(C.c_void_p(streams[k].cuda_stream)))

    th = [threading.Thread(target=run, args=(k,)) for k in range(2)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    t.cuda.synchronize()
    assert codes == [[0] * 8, [0] * 8]
    for row in cases:
        for case in row:
            case.check()


# ---- B. counted exchange, simulated world --------------------------------------------------------------------------------

def counted_exchange(senders, W):
    """tg_partition_count + tg_partition_exchange for every sender (senders[s] = device columns, key first) into W local
    receive buffers.  -> (recv[p] = list of (view, buffer) per column, count matrix, totals)"""
    L = lib()
    ncols = len(senders[0])
    M = np.zeros((W, W), np.int64)
    for s, cols in enumerate(senders):
        cnt = guarded(W)
        assert L.tg_partition_count(0, ptr(cols[0]), C.c_int64(cols[0].numel()), W, ptr(cnt[0]), None) == 0
        M[s] = host(cnt[0])
        assert_guard(cnt[1][W:], "counts")
    total = M.sum(axis=0)
    recv = [[guarded(int(total[p])) for _ in range(ncols)] for p in range(W)]
    peers = (C.c_void_p * (W * ncols))(*[recv[p][c][0].data_ptr() for p in range(W) for c in range(ncols)])
    for s, cols in enumerate(senders):
        base, _ = recv_bases(M, s)
        base_dev = upload(base)[0]
        cnt_dev = upload(M[s])[0]
        assert L.tg_partition_exchange(0, ptr(cols[0]), C.c_int64(cols[0].numel()), W, ncols, parr(cols), peers, ptr(cnt_dev),
                                       ptr(base_dev), None) == 0, L.tg_last_error()
    torch().cuda.synchronize()
    return recv, M, total


@pytest.mark.parametrize("W,ncols,rows", [(2, 2, 100_003), (5, 4, 50_001), (16, 6, 20_011), (5, 6, 3000), (16, 2, 7 * 1024),
                                          (2, 4, 1000)])
def test_counted_exchange_simulated_world(W, ncols, rows):
    ins = [payload(s, rows + 131 * s, ncols) for s in range(W)]
    senders = [[upload(c)[0] for c in cols] for cols in ins]
    torch().cuda.synchronize()
    recv, M, total = counted_exchange(senders, W)
    pieces = []        # pieces[s][p] = columns sender s sends to p, from the host rendering of the exchange
    for cols in ins:
        got = []
        exchange_by_key_host(cols[0], cols, W, lambda ps: got.append(ps) or ps)
        pieces.append([[got[c][p] for c in range(ncols)] for p in range(W)])
    for s, cols in enumerate(ins):
        assert np.array_equal(M[s], np.bincount(partition_of_keys_np(cols[0], W), minlength=W))
    for p in range(W):
        cols_p = [host(v) for v, _ in recv[p]]
        for c, (_, buf) in enumerate(recv[p]):
            assert_guard(buf[int(total[p]):], f"receiver {p} column {c}")
        base = 0
        for s in range(W):
            run = [x[base:base + M[s, p]] for x in cols_p]
            same_rows(run, pieces[s][p], f"receiver {p}, sender {s}")
            base += M[s, p]


# ---- C. count-free exchange, simulated world -----------------------------------------------------------------------------

class CfWorld:
    """W senders, W receivers; receiver p's buffers hold W regions of `cap` rows at s * stride, separated by >= GUARD rows of
    sentinel; sender s writes with region_base = s * stride"""

    def __init__(self, W, ncols, cap, spill_cap=0):
        self.W, self.ncols, self.cap = W, ncols, cap
        self.stride = (cap + GUARD + 1) // 2 * 2
        self.recv = [[guarded(W * self.stride) for _ in range(ncols)] for _ in range(W)]
        self.peers = (C.c_void_p * (W * ncols))(*[self.recv[p][c][0].data_ptr() for p in range(W) for c in range(ncols)])
        self.sent = [guarded(16) for _ in range(W)]
        self.ovf = [upload(np.zeros(1, np.int64)) for _ in range(W)]
        self.spill_cap = spill_cap
        if spill_cap:
            self.spill = [[guarded(spill_cap) for _ in range(ncols)] for _ in range(W)]
            self.cursor = [upload(np.zeros(1, np.int64)) for _ in range(W)]

    def send(self, s, cols, fn="cf", ctas=0):
        L, W = lib(), self.W
        n = cols[0].numel()
        head = (0, ptr(cols[0]), C.c_int64(n), W, self.ncols, parr(cols), self.peers, C.c_int64(s * self.stride), C.c_int64(self.cap),
                ptr(self.sent[s][0]), ptr(self.ovf[s][0]))
        if fn == "cf":
            code = L.tg_partition_exchange_cf(*head, None)
        elif fn == "cf_ex":
            code = L.tg_partition_exchange_cf_ex(*head, C.c_int32(ctas), None)
        else:
            code = L.tg_partition_exchange_cf_spill(*head, parr([v for v, _ in self.spill[s]]), C.c_int64(self.spill_cap),
                                                    ptr(self.cursor[s][0]), C.c_int32(ctas), None)
        assert code == 0, L.tg_last_error()

    def region(self, p, s, rows):
        return [host(self.recv[p][c][0][s * self.stride:s * self.stride + rows]) for c in range(self.ncols)]

    def check_gaps(self, stored):
        """stored[s][p] = rows region s of receiver p holds: everything after them up to the next region is sentinel"""
        for p in range(self.W):
            for c in range(self.ncols):
                b = host(self.recv[p][c][1])
                for s in range(self.W):
                    g = b[s * self.stride + stored[s][p]:(s + 1) * self.stride]
                    assert np.all(g == SENT), f"receiver {p} col {c}: region {s} written past its {stored[s][p]} rows"
                assert np.all(b[self.W * self.stride:] == SENT)

    def flags(self, s):
        return int(host(self.ovf[s][0])[0])


def cf_cap(kind, rows, W):
    return region_capacity(rows, W) if kind == "region" else kind


CF_FITS = [
    # (W, rows, ncols, fn, ctas, cap)
    (2, 1000, 1, "cf", 0, 1001), (3, 1024, 2, "cf_ex", 1, 1001), (5, 4613, 3, "cf_spill", 0, "region"),
    (2, 1_000_003, 4, "cf_ex", 1, "region"), (16, 1_000_003, 2, "cf", 0, "region"), (7, 4613, 4, "cf_spill", 1, 1001),
    (13, 1024, 1, "cf_ex", 1, "region"), (4, 1_000_003, 3, "cf_spill", 1, "region"),
]


@pytest.mark.parametrize("W,rows,ncols,fn,ctas,cap", CF_FITS)
def test_count_free_exchange_fits(W, rows, ncols, fn, ctas, cap):
    cap = cf_cap(cap, rows, W)
    w = CfWorld(W, ncols, cap, spill_cap=rows if fn == "cf_spill" else 0)
    ins = [payload(s, rows, ncols) for s in range(W)]
    dev = [[upload(c)[0] for c in cols] for cols in ins]
    torch().cuda.synchronize()
    for s in range(W):
        w.send(s, dev[s], fn, ctas)
    torch().cuda.synchronize()
    stored = []
    for s, cols in enumerate(ins):
        seg, seg_cnt, overflow = exchange_segments_host(cols[0], cols, W, 0, cap, lambda x: x)
        assert not overflow, "the case is meant to fit"
        cnt = np.bincount(partition_of_keys_np(cols[0], W), minlength=W)
        assert np.array_equal(host(w.sent[s][0])[:W], cnt)
        assert np.all(host(w.sent[s][1])[W:] == SENT)
        assert w.flags(s) == 0
        for p in range(W):
            same_rows(w.region(p, s, cnt[p]), [x[p * cap:p * cap + seg_cnt[p]] for x in seg], f"sender {s} -> {p}")
        stored.append(cnt)
        if fn == "cf_spill":
            assert int(host(w.cursor[s][0])[0]) == 0
            for c in range(ncols):
                assert_guard(w.spill[s][c][1], "unused spill area")
    w.check_gaps(stored)


@pytest.mark.parametrize("W,rows,ncols,fn,ctas,cap,hot", [
    (2, 4613, 2, "cf", 0, 1001, False), (3, 1_000_003, 3, "cf_ex", 1, 1001, False),
    (5, 1_000_003, 2, "cf_ex", 0, "region", True), (2, 1000, 1, "cf", 0, 257, False), (4, 2049, 4, "cf_ex", 1, 1001, True),
])
def test_count_free_exchange_overflow_without_spill(W, rows, ncols, fn, ctas, cap, hot):
    """a destination gets more rows than its region holds: the region takes exactly `cap` of them, sent[p] still counts every
    row destined to p (receivers clamp it to the capacity), and the overflow flag is raised and stays raised"""
    cap = cf_cap(cap, rows, W)
    w = CfWorld(W, ncols, cap)
    ins = [payload(s, rows, ncols) for s in range(W)]
    if hot:
        ins = [skewed(cols, 7 + s) for s, cols in enumerate(ins)]
    dev = [[upload(c)[0] for c in cols] for cols in ins]
    torch().cuda.synchronize()
    for s in range(W):
        w.send(s, dev[s], fn, ctas)
    torch().cuda.synchronize()
    stored = []
    for s, cols in enumerate(ins):
        dest = partition_of_keys_np(cols[0], W)
        cnt = np.bincount(dest, minlength=W)
        assert cnt.max() > cap, "the case is meant to overflow"
        assert np.array_equal(host(w.sent[s][0])[:W], cnt)
        assert w.flags(s) == 1
        keep = np.minimum(cnt, cap)
        for p in range(W):
            i = row_index(w.region(p, s, keep[p]), cols, s)
            assert len(np.unique(i)) == keep[p], f"sender {s} -> {p}: a row stored twice"
            assert np.all(dest[i] == p), f"sender {s} -> {p}: a row of another destination"
        stored.append(keep)
    w.check_gaps(stored)
    # sticky: a following call that fits leaves the flag raised and resets sent
    small = payload(0, 300, ncols)
    w.send(0, [upload(c)[0] for c in small], fn, ctas)
    torch().cuda.synchronize()
    assert w.flags(0) == 1
    assert np.array_equal(host(w.sent[0][0])[:W], np.bincount(partition_of_keys_np(small[0], W), minlength=W))


@pytest.mark.parametrize("W,rows,ncols,ctas,cap", [(4, 1_000_003, 2, 0, "region"), (3, 4613, 4, 1, 1001), (2, 1000, 1, 0, 257),
                                                  (16, 1_000_003, 3, 1, "region")])
def test_count_free_exchange_spill(W, rows, ncols, ctas, cap):
    """a hot key on 60 % of the rows: what does not fit its region goes to the spill area; regions plus spill hold every row
    exactly once, the spill cursor is exactly the excess and keeps counting across calls, the overflow flag stays 0"""
    cap = cf_cap(cap, rows, W)
    w = CfWorld(W, ncols, cap, spill_cap=2 * rows)
    before = [0] * W
    high = np.zeros((W, W), np.int64)     # rows region s of receiver p has held in any call so far
    for call in range(2):
        ins = [skewed(payload(s, rows - 17 * call, ncols), 100 * call + s) for s in range(W)]
        dev = [[upload(c)[0] for c in cols] for cols in ins]
        torch().cuda.synchronize()
        for s in range(W):
            w.send(s, dev[s], "cf_spill", ctas)
        torch().cuda.synchronize()
        for s, cols in enumerate(ins):
            cnt = np.bincount(partition_of_keys_np(cols[0], W), minlength=W)
            excess = int(np.maximum(cnt - cap, 0).sum())
            assert excess > 0, "the case is meant to spill"
            assert np.array_equal(host(w.sent[s][0])[:W], cnt)
            assert w.flags(s) == 0
            cur = int(host(w.cursor[s][0])[0])
            assert cur == before[s] + excess, (cur, before[s], excess)
            keep = np.minimum(cnt, cap)
            got = [np.concatenate([w.region(p, s, keep[p])[c] for p in range(W)] + [host(w.spill[s][c][0][before[s]:cur])])
                   for c in range(ncols)]
            same_rows(got, cols, f"sender {s}: regions + spill")
            for c in range(ncols):
                assert_guard(w.spill[s][c][1][cur:], "spill area past its cursor")
            before[s] = cur
            high[s] = np.maximum(high[s], keep)
        w.check_gaps(high)


@pytest.mark.parametrize("W,rows,ncols,ctas,cap,spill_cap", [(4, 1_000_003, 2, 0, "region", 100_000), (2, 1000, 2, 0, 257, 100),
                                                             (3, 4613, 3, 1, 1001, 700)])
def test_count_free_exchange_spill_area_full(W, rows, ncols, ctas, cap, spill_cap):
    """the excess exceeds the spill area: overflow is raised, no row is placed twice and nothing is written at or past
    spill_cap"""
    cap = cf_cap(cap, rows, W)
    w = CfWorld(W, ncols, cap, spill_cap=spill_cap)
    ins = [skewed(payload(s, rows, ncols), 50 + s) for s in range(W)]
    dev = [[upload(c)[0] for c in cols] for cols in ins]
    torch().cuda.synchronize()
    for s in range(W):
        w.send(s, dev[s], "cf_spill", ctas)
    torch().cuda.synchronize()
    stored = []
    for s, cols in enumerate(ins):
        dest = partition_of_keys_np(cols[0], W)
        cnt = np.bincount(dest, minlength=W)
        assert int(np.maximum(cnt - cap, 0).sum()) > spill_cap, "the case is meant to fill the spill area"
        assert w.flags(s) == 1
        keep = np.minimum(cnt, cap)
        placed = [row_index(w.region(p, s, keep[p]), cols, s) for p in range(W)]
        for p in range(W):
            assert np.all(dest[placed[p]] == p)
        sp = [host(w.spill[s][c][1]) for c in range(ncols)]
        for c in range(ncols):
            assert np.all(sp[c][spill_cap:] == SENT), "written at or past spill_cap"
        written = sp[1][:spill_cap] != SENT              # reservations that failed leave their rows unwritten
        placed.append(row_index([x[:spill_cap][written] for x in sp], cols, s))
        allp = np.concatenate(placed)
        assert len(np.unique(allp)) == len(allp), "a row placed twice"
        stored.append(keep)
    w.check_gaps(stored)


def test_count_free_exchange_gates():
    """every gate returns its code before anything is launched (sent and the receive buffers stay untouched)"""
    L = lib()
    W, ncols, n = 2, 2, 4096
    w = CfWorld(W, ncols, 2048, spill_cap=64)
    cols = [upload(c)[0] for c in payload(0, n, ncols)]
    shifted = [upload(c, 1)[0] for c in payload(0, n, ncols)]
    other_key = upload(payload(0, n, 1)[0])[0]
    odd_peer = (C.c_void_p * (W * ncols))(*[w.peers[i] + (8 if i == 1 else 0) for i in range(W * ncols)])
    torch().cuda.synchronize()
    spill = parr([v for v, _ in w.spill[0]])

    def cf(key=None, src=None, P=W, nc=ncols, peers=None, base=0, cap=2048):
        key = cols[0] if key is None else key
        src = parr(cols if src is None else src)
        return L.tg_partition_exchange_cf_ex(0, ptr(key), C.c_int64(n), P, nc, src, w.peers if peers is None else peers, C.c_int64(base),
                                             C.c_int64(cap), ptr(w.sent[0][0]), ptr(w.ovf[0][0]), C.c_int32(0), None)

    five = [upload(c)[0] for c in payload(0, n, 5)]
    assert cf(src=five, nc=5) == abi.TG_ERR_UNSUPPORTED
    assert cf(key=other_key) == abi.TG_ERR_INVALID                        # src[0] != key
    assert cf(key=shifted[0], src=shifted) == abi.TG_ERR_UNSUPPORTED     # unaligned source
    assert cf(peers=odd_peer) == abi.TG_ERR_UNSUPPORTED                  # unaligned receive column
    assert cf(base=2049) == abi.TG_ERR_UNSUPPORTED                       # odd region_base
    assert cf(cap=0) == abi.TG_ERR_INVALID
    assert cf(P=0) == abi.TG_ERR_UNSUPPORTED and cf(P=17) == abi.TG_ERR_UNSUPPORTED
    assert L.tg_partition_exchange_cf_spill(0, ptr(cols[0]), C.c_int64(n), W, ncols, parr(cols), w.peers, C.c_int64(0), C.c_int64(2048),
                                            ptr(w.sent[0][0]), ptr(w.ovf[0][0]), spill, C.c_int64(64), None, C.c_int32(0), None) == abi.TG_ERR_INVALID
    torch().cuda.synchronize()
    assert np.all(host(w.sent[0][1]) == SENT), "a gated call launched its kernels"
    assert w.flags(0) == 0
    w.check_gaps([[0] * W for _ in range(W)])


# ---- D. tg_peer_copy_regions on one device -------------------------------------------------------------------------------

@pytest.mark.parametrize("nreg,ctas", [(1, 0), (7, 1), (20, 7), (64, 0), (64, 7), (64, 1)])
def test_peer_copy_regions(nreg, ctas):
    """region r: the first min(count, cap) rows move; an odd count may carry its one padding row along (the kernel copies
    16-byte units and regions hold an even number of rows); everything from round_up_even(min(count, cap)) on is untouched"""
    L, t = lib(), torch()
    cap = 4096
    span = cap + GUARD
    vals = [0, 1, 7, 10, cap, cap + 5, 3001, 2, cap - 1, 1 << 40]
    counts = np.array([vals[k % len(vals)] for k in range(nreg + 3)], np.int64)
    counts_dev = upload(counts)[0]
    idx = np.random.default_rng(nreg).permutation(nreg + 3)[:nreg].astype(np.int32)
    src = t.arange(nreg * span, dtype=t.int64, device="cuda") * 3 + 1
    dst = t.full((nreg * span,), SENT, dtype=t.int64, device="cuda")
    t.cuda.synchronize()
    sp = (C.c_void_p * nreg)(*[src.data_ptr() + r * span * 8 for r in range(nreg)])
    dp = (C.c_void_p * nreg)(*[dst.data_ptr() + r * span * 8 for r in range(nreg)])
    ci = (C.c_int32 * nreg)(*idx.tolist())
    assert L.tg_peer_copy_regions(0, nreg, sp, dp, ci, ptr(counts_dev), C.c_int64(cap), ctas, None) == 0
    t.cuda.synchronize()
    s, d = host(src), host(dst)
    for r in range(nreg):
        m = int(min(counts[idx[r]], cap))
        sr, dr = s[r * span:(r + 1) * span], d[r * span:(r + 1) * span]
        assert np.array_equal(dr[:m], sr[:m]), f"region {r}: {m} rows"
        e = m + (m & 1)
        if m & 1:
            assert dr[m] in (SENT, sr[m])                 # the padding row of an odd count may be copied
        assert np.all(dr[e:] == SENT), f"region {r}: written past round_up_even({m})"


def test_peer_copy_regions_gates():
    L, t = lib(), torch()
    buf = t.full((4 * 8192,), SENT, dtype=t.int64, device="cuda")
    cnt = upload(np.array([100], np.int64))[0]
    t.cuda.synchronize()

    def call(n, src_off=0, dst_off=0, cap=4096):
        sp = (C.c_void_p * max(n, 1))(*([buf.data_ptr() + src_off] * max(n, 1)))
        dp = (C.c_void_p * max(n, 1))(*([buf.data_ptr() + 16384 * 8 + dst_off] * max(n, 1)))
        ci = (C.c_int32 * max(n, 1))(*([0] * max(n, 1)))
        return L.tg_peer_copy_regions(0, n, sp, dp, ci, ptr(cnt), C.c_int64(cap), 0, None)

    assert call(1, cap=4095) == abi.TG_ERR_INVALID
    assert call(0) == abi.TG_ERR_INVALID and call(65) == abi.TG_ERR_INVALID
    assert call(1, src_off=8) == abi.TG_ERR_UNSUPPORTED and call(1, dst_off=8) == abi.TG_ERR_UNSUPPORTED
    t.cuda.synchronize()
    assert np.all(host(buf) == SENT)


# ---- E. mailboxes on one device ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("W", [1, 5, 16])
def test_mailbox_signal_and_wait(W):
    """signal W slots of a local block, then wait on them on the same stream (the wait never spins: its signals are ordered
    before it; timeout_ms is only a safety net): the words are epoch << 40 | min(v, 2^40 - 1), the wait returns the low 40
    bits and leaves the error flag at 0"""
    L, t = lib(), torch()
    mail = t.full((16 + GUARD,), SENT, dtype=t.int64, device="cuda")
    err = upload(np.zeros(1, np.int64))[0]
    out = guarded(16)
    tg = abi.TgMailTargets()
    tg.n = W
    for p in range(W):
        tg.slot[p] = mail.data_ptr() + p * 8
    pool = [0, M40, 1 << 40, 1 << 62, 12345]
    for k, epoch in enumerate([1, 2, 3, 7, 1000]):
        if k == 2:
            values = None
            v = np.zeros(W, np.uint64)
        else:
            v = np.array([pool[(p + k) % len(pool)] for p in range(W)], np.uint64)
            values = upload(v.view(np.int64))[0]
        t.cuda.synchronize()
        assert L.tg_mail_signal(0, C.byref(tg), ptr(values) if values is not None else None, C.c_int64(epoch), None) == 0
        for e in (epoch, max(1, epoch - 1)):
            assert L.tg_mail_wait(0, ptr(mail), W, C.c_int64(e), ptr(out[0]), ptr(err), C.c_int64(5000), None) == 0
            t.cuda.synchronize()
            clamped = np.minimum(v, np.uint64(M40))
            words = host(mail).view(np.uint64)
            assert np.array_equal(words[:W], (np.uint64(epoch) << np.uint64(40)) | clamped), (epoch, words[:W])
            assert np.all(host(mail)[W:] == SENT)
            assert np.array_equal(host(out[0])[:W].view(np.uint64), clamped)
            assert np.all(host(out[1])[W:] == SENT)
            assert int(host(err)[0]) == 0


def test_mailbox_gates():
    L, t = lib(), torch()
    mail = t.full((16,), SENT, dtype=t.int64, device="cuda")
    err = upload(np.zeros(1, np.int64))[0]
    t.cuda.synchronize()
    for n in (0, 17):
        tg = abi.TgMailTargets()
        tg.n = n
        for p in range(16):
            tg.slot[p] = mail.data_ptr() + p * 8
        assert L.tg_mail_signal(0, C.byref(tg), None, C.c_int64(1), None) == abi.TG_ERR_INVALID
        assert L.tg_mail_wait(0, ptr(mail), n, C.c_int64(1), None, ptr(err), C.c_int64(100), None) == abi.TG_ERR_INVALID
    assert L.tg_mail_signal(0, None, None, C.c_int64(1), None) == abi.TG_ERR_INVALID
    assert L.tg_mail_wait(0, None, 1, C.c_int64(1), None, ptr(err), C.c_int64(100), None) == abi.TG_ERR_INVALID
    assert L.tg_mail_wait(0, ptr(mail), 1, C.c_int64(1), None, None, C.c_int64(100), None) == abi.TG_ERR_INVALID
    t.cuda.synchronize()
    assert np.all(host(mail) == SENT) and int(host(err)[0]) == 0


# ---- F. the product path end to end, W ranks on one device ---------------------------------------------------------------

KEYMUL = np.int64(-7046029254386353131)


@pytest.mark.parametrize("W", [4, 16])
def test_product_path_simulated_world(W):
    """mirror of tests/mgpu_worker.py with W ranks on device 0: build shards through the counted exchange, three probe steps
    through tg_partition_exchange_cf_spill with the fill counts published through the mailboxes and probed as segments
    (step 1 skewed: 60 % of the rows on one key), then the spill drained through the counted exchange.  The union of every
    rank's output is the unique-key inner join of the global inputs."""
    from tidb_b200.device import DeviceJoin, fetch_device
    from tidb_b200.plan import FieldType, JoinPlan
    L, t = lib(), torch()
    nb, npr, steps = 20_000, 50_000, 3
    ids = [np.random.default_rng(10 + r).permutation(nb).astype(np.int64) + r * nb for r in range(W)]
    bks = [i * KEYMUL for i in ids]
    bvs = [i * 7 for i in ids]
    probes = []       # probes[step][rank] = (pk, pv)
    for st in range(steps):
        row = []
        for r in range(W):
            rng = np.random.default_rng(1000 * st + r)
            pk = np.where(rng.random(npr) < 0.3, rng.integers(1 << 40, 1 << 41, npr).astype(np.int64) * 2 + 1,
                          rng.integers(0, nb * W, npr).astype(np.int64) * KEYMUL)
            if st == 1:
                pk = np.where(rng.random(npr) < 0.6, (np.array([12345], np.int64) * KEYMUL)[0], pk)
            row.append((pk, np.arange(npr, dtype=np.int64) + (st * W + r) * npr))
        probes.append(row)
    # build side: counted exchange, one DeviceJoin per rank
    INT = FieldType(abi.TYPE_LONGLONG, abi.FLAG_NOT_NULL)
    plan = JoinPlan(abi.JOIN_INNER, [INT, INT], [INT, INT], [0], [0], build_is_right=True)
    bdev = [[upload(bks[r])[0], upload(bvs[r])[0]] for r in range(W)]
    t.cuda.synchronize()
    brecv, _, btotal = counted_exchange(bdev, W)
    joins = []
    for r in range(W):
        j = DeviceJoin(plan)
        j.build([brecv[r][0][0], brecv[r][1][0]])
        joins.append(j)
    outs = []

    def collect(rows, cols):
        if rows:
            outs.append([fetch_device(p, rows * 8).view(np.int64).copy() for p in cols])

    cap = region_capacity(npr, W)
    spill_cap = 2 * npr
    spill = [[guarded(spill_cap) for _ in range(2)] for _ in range(W)]
    cursor = [upload(np.zeros(1, np.int64))[0] for _ in range(W)]
    ovf = [upload(np.zeros(1, np.int64))[0] for _ in range(W)]
    err = upload(np.zeros(1, np.int64))[0]
    counts = [guarded(16) for _ in range(W)]          # receiver r's count mailboxes, one slot per sender
    sent = [guarded(16) for _ in range(W)]
    spilled = []
    for st in range(steps):
        recv = [[guarded(W * cap) for _ in range(2)] for _ in range(W)]
        peers = (C.c_void_p * (W * 2))(*[recv[p][c][0].data_ptr() for p in range(W) for c in range(2)])
        pdev = [[upload(probes[st][r][0])[0], upload(probes[st][r][1])[0]] for r in range(W)]
        t.cuda.synchronize()
        before = [int(host(c)[0]) for c in cursor]
        for s in range(W):
            assert L.tg_partition_exchange_cf_spill(0, ptr(pdev[s][0]), C.c_int64(npr), W, 2, parr(pdev[s]), peers, C.c_int64(s * cap),
                                                    C.c_int64(cap), ptr(sent[s][0]), ptr(ovf[s]), parr([v for v, _ in spill[s]]),
                                                    C.c_int64(spill_cap), ptr(cursor[s]), C.c_int32(0), None) == 0, L.tg_last_error()
            tg = abi.TgMailTargets()
            tg.n = W
            for p in range(W):
                tg.slot[p] = counts[p][0].data_ptr() + s * 8
            assert L.tg_mail_signal(0, C.byref(tg), ptr(sent[s][0]), C.c_int64(st + 1), None) == 0
        for r in range(W):
            seg_cnt = guarded(W)[0]
            assert L.tg_mail_wait(0, ptr(counts[r][0]), W, C.c_int64(st + 1), ptr(seg_cnt), ptr(err), C.c_int64(5000), None) == 0
            # the join reads seg_cnt on a stream of its own, unordered with the default stream the wait writes it on: let the
            # wait finish first (mgpu_worker.py enqueues the wait on the join's stream instead).  Safe: every signal the wait
            # needs was enqueued above
            t.cuda.synchronize()
            collect(*joins[r].probe_segments([recv[r][0][0], recv[r][1][0]], seg_cnt, cap, sync=True)[:2])
        spilled.append(sum(int(host(c)[0]) for c in cursor) - sum(before))
    assert spilled[0] == 0 and spilled[1] > 0, spilled
    assert all(int(host(o)[0]) == 0 for o in ovf) and int(host(err)[0]) == 0
    # drain: every sender's spill rows through the counted exchange, probed like any other batch
    drain = [[v[:int(host(cursor[s])[0])] for v, _ in spill[s]] for s in range(W)]
    rrecv, _, rtotal = counted_exchange(drain, W)
    for r in range(W):
        if rtotal[r]:
            collect(*joins[r].probe([rrecv[r][0][0], rrecv[r][1][0]], sync=True)[:2])
    for j in joins:
        j.close()
    got = [np.concatenate([o[c] for o in outs]) for c in range(4)]
    # reference: numpy unique-key inner join of the global inputs
    bk, bv = np.concatenate(bks), np.concatenate(bvs)
    pk = np.concatenate([probes[st][r][0] for st in range(steps) for r in range(W)])
    pv = np.concatenate([probes[st][r][1] for st in range(steps) for r in range(W)])
    order = np.argsort(bk)
    pos = np.minimum(np.searchsorted(bk[order], pk), len(bk) - 1)
    hit = bk[order][pos] == pk
    exp = [pk[hit], pv[hit], bk[order[pos[hit]]], bv[order[pos[hit]]]]
    by = np.argsort(got[1])
    assert len(got[1]) == len(exp[1]), (len(got[1]), len(exp[1]))
    for g, e in zip(got, exp):
        assert np.array_equal(g[by], e)        # pv is unique and exp is in pv order
