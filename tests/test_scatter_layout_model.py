"""Executable model of the staging layout of k_partition_scatter_bulk (tidb_b200/csrc/partition_kernels.cuh).

The kernel parks the run of destination p at a shared-memory offset whose parity equals the parity of the run's first GLOBAL
row, so that the 16-byte aligned middle of the run can leave as one cp.async.bulk store (both addresses 16-byte aligned, size
a multiple of 16) and at most one head and one tail element go out as scalar stores.  This test restates the index arithmetic
(same expressions, same names) and checks the invariants for random cursor positions and counts; it documents the layout
and catches an edit that breaks it — the kernel itself, with its head / tail stores, truncated runs and spill area, is
exercised on one GPU by tests/test_gpu_partition_exchange.py."""
import numpy as np


def layout(gbase, cnt, cap_left=None):
    """gbase[p]: first global row of the run, cnt[p]: rows of the tile going to p.  -> per destination (s_off, head, mid, tail, len)"""
    out, incl = [], 0
    for p, (g, c) in enumerate(zip(gbase, cnt)):
        ln = c if cap_left is None else min(c, cap_left[p])
        w = ((g & 1) + c + 1) & ~1          # padded width: the next run starts at an even staging index
        s_off = incl + (g & 1)
        incl += w
        head = (g & 1) & (1 if ln > 0 else 0)
        mid = (ln - head) & ~1
        tail = (ln - head) & 1
        out.append((s_off, head, mid, tail, ln))
    return out, incl


def test_layout_invariants():
    rng = np.random.default_rng(1)
    TILE, MAXP = 1024, 16
    for _ in range(2000):
        P = int(rng.integers(1, MAXP + 1))
        cnt = np.bincount(rng.integers(0, P, TILE), minlength=P)
        if rng.random() < 0.3:
            cnt[rng.integers(0, P)] = 0
        gbase = rng.integers(0, 1 << 40, P)
        cap_left = [int(c) if rng.random() < 0.8 else int(rng.integers(0, c + 1)) for c in cnt] if rng.random() < 0.3 else None
        runs, total = layout([int(g) for g in gbase], [int(c) for c in cnt], cap_left)
        assert total <= TILE + 2 * MAXP                      # SROWS = TILE + 2 * TG_MAX_PARTS
        used = np.zeros(total + 2, dtype=np.int32)
        for p, (so, head, mid, tail, ln) in enumerate(runs):
            g, c = int(gbase[p]), int(cnt[p])
            used[so:so + c] += 1                             # every row of the tile has its own staging slot
            assert head + mid + tail == ln                   # every surviving row leaves exactly once
            if mid:
                assert (so + head) % 2 == 0 and (g + head) % 2 == 0     # 16-byte aligned on both sides (8-byte elements)
                assert (mid * 8) % 16 == 0
            if head:
                assert so % 2 == 1 and g % 2 == 1            # the odd first element is the scalar head
            if tail:
                assert (g + ln - 1) == g + head + mid        # the scalar tail is the last surviving row
        assert used.max() <= 1


def test_segment_capacity_formula():
    # join.cu: C = round128(n_main / P * 1.05 + 16384); SegmentExchange: cap = round1024(rows / world * 1.06 + 8192)
    from tidb_b200.parallel import region_capacity
    for n, P in [(100_000_000, 12), (4_194_304, 2), (99_999_744, 16)]:
        C = (int(n / P * 1.05) + 16384 + 127) // 128 * 128
        assert C % 128 == 0 and C * P >= n and C * P / 128 < (1 << 31)
    for rows, world in [(100_000_000, 8), (100_000_000, 2), (1_000_000, 4)]:
        cap = region_capacity(rows, world)
        assert cap % 1024 == 0 and cap >= rows / world * 1.06


def test_spill_bookkeeping_model():
    """count-free scatter with a spill area (PartDst.spill_cursor, tg_partition_exchange_cf_spill): per (tile, destination) run
    the first `len` rows go to the region, the rest to spill rows [spg, spg + spn); over many tiles and CTAs in any order every
    row lands exactly once, a region never holds more than its capacity, and the cursors the receiver sees (clamped to the
    capacity) count exactly the rows stored.  Same expressions as the kernel's warp-0 block."""
    rng = np.random.default_rng(3)
    for trial in range(200):
        P, cap, spill_cap = int(rng.integers(1, 9)), int(rng.integers(0, 5000)), 1 << 20
        cursors, spill_cursor = np.zeros(P, dtype=np.int64), 0
        region = [[] for _ in range(P)]
        spill, total = [], 0
        hot = int(rng.integers(0, P))
        for tile in range(int(rng.integers(1, 40))):
            dest = np.where(rng.random(1024) < 0.5, hot, rng.integers(0, P, 1024))
            cnt = np.bincount(dest, minlength=P)
            for p in range(P):
                c = int(cnt[p])
                old = int(cursors[p]); cursors[p] += c                         # atomicAdd(&cursors[p], c)
                avail = cap - old if old < cap else 0
                ln, spn, spg = c, 0, 0
                if c > avail:
                    ln = avail
                    spn = c - ln
                    spg = spill_cursor; spill_cursor += spn                    # atomicAdd(spill_cursor, spn)
                    assert spg + spn <= spill_cap
                rows = [(tile, p, r) for r in range(c)]                        # staging slots so + r, r = rank inside the run
                region[p].extend(rows[:ln])                                    # head / bulk middle / tail stores
                assert spn == 0 or len(spill) == spg
                spill.extend(rows[ln:ln + spn])                                # scalar spill stores src[so + len + r]
                total += c
        assert all(len(region[p]) == min(int(cursors[p]), cap) for p in range(P))   # what the receiver reads: min(cursor, cap)
        placed = [x for r in region for x in r] + spill
        assert len(placed) == total == len(set(placed))
