"""Key-hash repartition across GPUs: the one exchange step of the partitioned hash join / aggregation.

Reference analogue: the MPP ExchangeSender with ExchangeType HashPartition that the planner emits for TiFlash
(pkg/planner/core/operator/physicalop/physical_exchange_sender.go:115; Q3 plan in
planner/core/casetest/tpch/testdata/tpch_suite_out.json:99-123) and, in process,
partitionHashSplitter.split (pkg/executor/shuffle.go:450).  One process per GPU (torch.distributed).

Two data paths, same partition function (tg_partition_of_key = low 32 bits of mix64(key), disjoint from the table
slot bits):
  * "nccl": k_partition_scatter into local per-destination regions, then all_to_all_single per column;
  * "p2p" : tg_partition_exchange — the scatter kernel stores each destination's runs straight into the peer's
            receive buffer over NVLink (buffers shared with cudaIpc handles), i.e. the repartition and its
            all-to-all are ONE kernel; only the 8×8 count matrix goes through a collective.
The host-side bookkeeping (counts → send/recv splits → bases) is shared with the CPU/gloo tests.
"""
from __future__ import annotations

import ctypes as C
from typing import Callable, List, Optional, Sequence, Tuple

import numpy as np

_C64 = np.uint64(0x9E3779B97F4A7C15)


def hash64_np(k: np.ndarray) -> np.ndarray:
    """numpy mirror of tg::hash64 (csrc/common.cuh): xor-fold + one 64-bit multiply"""
    k = k.astype(np.uint64, copy=True)
    with np.errstate(over="ignore"):
        k ^= k >> np.uint64(32)
        k *= _C64
    return k


def partition_of_keys_np(keys: np.ndarray, nparts: int) -> np.ndarray:
    """numpy mirror of tg_partition_of_key (tg::part_of): destination rank of every key"""
    h = hash64_np(keys.view(np.uint64) if keys.dtype != np.uint64 else keys)
    lo = (h & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    hi = (h >> np.uint64(32)).astype(np.uint32)
    with np.errstate(over="ignore"):
        g = lo ^ (hi * np.uint32(0x85EBCA6B))
        g = g * np.uint32(0xC2B2AE35)
        g ^= g >> np.uint32(16)
    return ((g.astype(np.uint64) * np.uint64(nparts)) >> np.uint64(32)).astype(np.int64)


def recv_bases(count_matrix: np.ndarray, rank: int) -> Tuple[np.ndarray, int]:
    """count_matrix[src, dst] = rows src sends to dst.
    -> (base[dst] = first row of `rank`'s region inside dst's receive buffer, rows this rank receives)"""
    base = count_matrix[:rank, :].sum(axis=0).astype(np.int64)
    return base, int(count_matrix[:, rank].sum())


def exchange_by_key_host(keys: np.ndarray, cols: Sequence[np.ndarray], world: int,
                         all_to_all: Callable[[List[np.ndarray]], List[np.ndarray]]) -> List[np.ndarray]:
    """CPU rendering of the exchange (gloo tests): split rows by destination, hand the per-destination pieces to
    `all_to_all`, concatenate what arrives.  Same function, same bookkeeping as the device path."""
    dest = partition_of_keys_np(keys, world)
    order = np.argsort(dest, kind="stable")
    counts = np.bincount(dest, minlength=world)
    offs = np.concatenate([[0], np.cumsum(counts)])
    out = []
    for c in cols:
        cs = c[order]
        pieces = [np.ascontiguousarray(cs[offs[d]:offs[d + 1]]) for d in range(world)]
        out.append(np.concatenate(all_to_all(pieces)))
    return out


def region_capacity(rows_per_step: int, world: int, slack: float = 1.06) -> int:
    """rows of one (sender, receiver) region of the count-free exchange: expected share + slack, a multiple of the
    1024-row scatter tile (tg_join_probe_dev_seg requires it)"""
    return ((int(rows_per_step / world * slack) + 8192 + 1023) // 1024) * 1024


def exchange_segments_host(keys: np.ndarray, cols: Sequence[np.ndarray], world: int, rank: int, cap: int,
                           all_to_all: Callable[[List], List], spill: Optional[List] = None):
    """CPU rendering of SegmentExchange (gloo tests): same region layout, same bookkeeping, same overflow rule.
    Every sender appends the rows of destination d to ITS region of d's receive buffer (at most `cap` rows, the excess is
    dropped and flagged); the receiver sees `world` segments of `cap` rows, segment s valid for seg_cnt[s] rows.
    With `spill` (a list) the excess is appended to it instead — one entry of columns per overflowing destination — and no
    overflow is flagged: the caller moves those rows with exchange_by_key_host afterwards (MailboxExchange.drain_spill).
    -> (received columns of world*cap rows each, seg_cnt[world], overflow flag)"""
    dest = partition_of_keys_np(keys, world)
    pieces, sent, overflow = [], np.zeros(world, dtype=np.int64), False
    for d in range(world):
        idx = np.nonzero(dest == d)[0]
        if len(idx) > cap:
            if spill is not None:      # tg_partition_exchange_cf_spill: the excess stays on the sender, in its spill area
                spill.append([np.ascontiguousarray(c[idx[cap:]]) for c in cols])
            else:
                overflow = True
            idx = idx[:cap]
        sent[d] = len(idx)
        pieces.append([np.ascontiguousarray(c[idx]) for c in cols])
    got = all_to_all(pieces)                      # got[s] = the columns sender s appended to my region s
    out = [np.zeros(world * cap, dtype=c.dtype) for c in cols]
    seg_cnt = np.zeros(world, dtype=np.int64)
    for s_, piece in enumerate(got):
        seg_cnt[s_] = len(piece[0])
        for c in range(len(cols)):
            out[c][s_ * cap:s_ * cap + len(piece[c])] = piece[c]
    return out, seg_cnt, overflow


def segments_to_dense(cols: Sequence[np.ndarray], seg_cnt: np.ndarray, cap: int) -> List[np.ndarray]:
    """the valid rows of a segmented column set, in segment order (what tg_join_probe_dev_seg probes)"""
    return [np.concatenate([c[s_ * cap:s_ * cap + int(n)] for s_, n in enumerate(seg_cnt)]) for c in cols]


class KeyExchange:
    """Device-side exchange for `ncols` 8-byte columns (key first) on one rank."""

    def __init__(self, rank: int, world: int, device: int, stream, ncols: int, capacity_rows: int, mode: str = "p2p"):
        import torch
        import torch.distributed as dist
        from . import abi
        self.torch, self.dist, self.abi = torch, dist, abi
        self.lib = abi.load_lib()
        self.rank, self.world, self.device, self.stream, self.ncols = rank, world, device, stream, ncols
        self.mode = mode
        self.dev = torch.device("cuda", device)
        self.capacity = int(capacity_rows)
        self.launches = 0
        self.counts = torch.zeros(world, dtype=torch.int64, device=self.dev)
        self.count_mat = torch.zeros(world * world, dtype=torch.int64, device=self.dev)
        self.base_dev = torch.zeros(world, dtype=torch.int64, device=self.dev)
        if mode == "p2p":
            self._alloc_symmetric()
        else:
            self.scratch = [torch.empty(0, dtype=torch.int64, device=self.dev) for _ in range(ncols)]
            self.offs = torch.zeros(world + 1, dtype=torch.int64, device=self.dev)

    # ---- p2p: symmetric receive buffers, IPC-mapped on every peer ------------------------------------------
    def _alloc_symmetric(self):
        lib, abi = self.lib, self.abi
        self.recv_ptrs = []
        handles = []
        for _ in range(self.ncols):
            p = C.c_void_p()
            abi.check(lib.tg_dev_alloc(self.device, C.c_size_t(self.capacity * 8), C.byref(p)))
            self.recv_ptrs.append(p.value)
            h = (C.c_uint8 * 64)()
            abi.check(lib.tg_ipc_export(self.device, p, h))
            handles.append(bytes(h))
        gathered = [None] * self.world
        self.dist.all_gather_object(gathered, handles)
        # peer_ptrs[p][c] = address, in THIS process, of column c's receive buffer on rank p
        self.peer_ptrs = []
        for p in range(self.world):
            row = []
            for c in range(self.ncols):
                if p == self.rank:
                    row.append(self.recv_ptrs[c])
                else:
                    mp = C.c_void_p()
                    hb = (C.c_uint8 * 64).from_buffer_copy(gathered[p][c])
                    abi.check(lib.tg_ipc_open(self.device, hb, C.byref(mp)))
                    row.append(mp.value)
            self.peer_ptrs.append(row)
        flat = [self.peer_ptrs[p][c] for p in range(self.world) for c in range(self.ncols)]
        self.peer_arr = (C.c_void_p * len(flat))(*flat)

    def _view(self, ptr: int, n: int):
        class _A:
            pass
        a = _A()
        a.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i8", "data": (ptr, False), "version": 3}
        return self.torch.as_tensor(a, device=self.dev)

    def exchange(self, key, cols):
        """cols[0] must be the key column.  -> list of received columns (torch int64 tensors on this device)"""
        torch, dist, lib, abi = self.torch, self.dist, self.lib, self.abi
        n = key.numel()
        st = C.c_void_p(self.stream.cuda_stream)
        if self.mode == "nccl":
            dst = []
            for i, c in enumerate(cols):
                if self.scratch[i].numel() < n:
                    self.scratch[i] = torch.empty(n, dtype=torch.int64, device=self.dev)
                dst.append(self.scratch[i][:n])
            src_p = (C.c_void_p * len(cols))(*[c.data_ptr() for c in cols])
            dst_p = (C.c_void_p * len(cols))(*[c.data_ptr() for c in dst])
            abi.check(lib.tg_partition_by_key(self.device, C.c_void_p(key.data_ptr()), None, C.c_int64(n), self.world, len(cols),
                                              src_p, dst_p, C.c_void_p(self.offs.data_ptr()), st))
            self.launches += 3
            send = torch.diff(self.offs)
            recv = torch.empty_like(send)
            dist.all_to_all_single(recv, send)
            send_l, recv_l = send.tolist(), recv.tolist()
            out = []
            for c in dst:
                r = torch.empty(sum(recv_l), dtype=torch.int64, device=self.dev)
                dist.all_to_all_single(r, c, recv_l, send_l)
                out.append(r)
            return out
        # p2p: counts → all-gather → bases → one scatter kernel that writes into the peers
        abi.check(lib.tg_partition_count(self.device, C.c_void_p(key.data_ptr()), C.c_int64(n), self.world,
                                         C.c_void_p(self.counts.data_ptr()), st))
        dist.all_gather_into_tensor(self.count_mat, self.counts)
        mat = self.count_mat.cpu().numpy().reshape(self.world, self.world)
        base, nrecv = recv_bases(mat, self.rank)
        if int(mat.sum(axis=0).max()) > self.capacity:
            raise RuntimeError("receive buffer capacity exceeded: re-create KeyExchange with a larger capacity_rows")
        self.base_dev.copy_(torch.from_numpy(base))
        dist.barrier()   # every peer is done reading what the previous exchange delivered into its receive buffers
        src_p = (C.c_void_p * len(cols))(*[c.data_ptr() for c in cols])
        abi.check(lib.tg_partition_exchange(self.device, C.c_void_p(key.data_ptr()), C.c_int64(n), self.world, len(cols), src_p,
                                            self.peer_arr, C.c_void_p(self.counts.data_ptr()), C.c_void_p(self.base_dev.data_ptr()), st))
        self.launches += 2
        dist.barrier()   # all peers' stores into my receive buffers have completed (kernel end + barrier)
        return [self._view(self.recv_ptrs[c], nrecv) for c in range(len(cols))]

    def close(self):
        if self.mode == "p2p":
            for p in range(self.world):
                if p == self.rank:
                    continue
                for c in range(self.ncols):
                    self.lib.tg_ipc_close(self.device, C.c_void_p(self.peer_ptrs[p][c]))
            for ptr in self.recv_ptrs:
                self.lib.tg_dev_free(self.device, C.c_void_p(ptr))
            self.recv_ptrs = []


class SegmentExchange:
    """Count-free key-hash exchange (tg_partition_exchange_cf): no histogram pass and NO host round trip per step.

    Every rank owns, inside each peer's receive buffers, one fixed-capacity region (region s of rank d's buffer belongs to
    sender s).  One kernel regroups 1024-row tiles by destination in shared memory and appends each destination's run to
    this rank's region on that peer with bulk stores over NVLink; the per-destination row counts stay on the device and
    are exchanged with ONE all-gather, which is also the barrier that makes the peer stores visible.  The receiver probes
    the `world` regions as segments (DeviceJoin.probe_segments), so nothing is compacted or counted on the host.
    Two alternating sets of receive buffers: a rank may start sending step k+1 while a peer still probes step k.
    The reference's analogue is the MPP HashPartition exchange (physical_exchange_sender.go:115)."""

    def __init__(self, rank: int, world: int, device: int, stream, ncols: int, rows_per_step: int, slack: float = 1.06, dma: bool = False):
        import torch
        import torch.distributed as dist
        from . import abi
        self.torch, self.dist, self.abi = torch, dist, abi
        self.lib = abi.load_lib()
        self.rank, self.world, self.device, self.stream, self.ncols = rank, world, device, stream, ncols
        self.dev = torch.device("cuda", device)
        self.dma = bool(dma) and world > 1
        self.cap = region_capacity(rows_per_step, world, slack)   # rows per (sender, receiver) region
        self.sets = 2
        self.step = 0
        self.launches = 0
        self.sent = [torch.zeros(16, dtype=torch.int64, device=self.dev) for _ in range(self.sets)]
        self.overflow = [torch.zeros(1, dtype=torch.int64, device=self.dev) for _ in range(self.sets)]
        self.count_mat = [torch.zeros(world * world, dtype=torch.int64, device=self.dev) for _ in range(self.sets)]
        self.seg_cnt = [torch.zeros(world, dtype=torch.int64, device=self.dev) for _ in range(self.sets)]
        lib = self.lib
        self.recv_ptrs = []      # [set][col]
        handles = []
        for _ in range(self.sets):
            row = []
            for _c in range(ncols):
                p = C.c_void_p()
                abi.check(lib.tg_dev_alloc(device, C.c_size_t(world * self.cap * 8 + 64), C.byref(p)))
                row.append(p.value)
                h = (C.c_uint8 * 64)()
                abi.check(lib.tg_ipc_export(device, p, h))
                handles.append(bytes(h))
            self.recv_ptrs.append(row)
        gathered = [None] * world
        dist.all_gather_object(gathered, handles)
        self.peer_ptrs = []      # [set][peer][col]
        self.peer_arr = []
        for s in range(self.sets):
            per_set = []
            for p in range(world):
                row = []
                for c in range(ncols):
                    if p == rank:
                        row.append(self.recv_ptrs[s][c])
                    else:
                        mp = C.c_void_p()
                        hb = (C.c_uint8 * 64).from_buffer_copy(gathered[p][s * ncols + c])
                        abi.check(lib.tg_ipc_open(device, hb, C.byref(mp)))
                        row.append(mp.value)
                per_set.append(row)
            self.peer_ptrs.append(per_set)
            flat = [per_set[p][c] for p in range(world) for c in range(ncols)]
            self.peer_arr.append((C.c_void_p * len(flat))(*flat))
        # dma=True: the kernel regroups into a LOCAL staging copy of the region layout (own rows go straight into the own
        # receive buffer) and copy engines push region p to peer p (tg_memcpy_d2d_async) — the NVLink transfer then needs
        # no SM and runs under the probe kernel of the previous step
        self.staging = []
        self.stage_arr = []
        self.copy_streams = []
        if self.dma:
            # one stream's copies run back to back on one copy engine; a few streams keep
            # several engines and NVLink paths busy
            self.copy_streams = [torch.cuda.Stream(device=self.dev) for _ in range(min(4, world - 1))]
            for c in range(ncols):
                p = C.c_void_p()
                abi.check(lib.tg_dev_alloc(device, C.c_size_t(world * self.cap * 8 + 64), C.byref(p)))
                self.staging.append(p.value)
            # exchange_async(): a second staging set and a dedicated transfer stream, so that the regrouping kernel of
            # step k+2 runs while the copy engines still move step k+1
            self.staging2 = []
            for s2 in range(self.sets):
                row = []
                for c in range(ncols):
                    p = C.c_void_p()
                    abi.check(lib.tg_dev_alloc(device, C.c_size_t(world * self.cap * 8 + 64), C.byref(p)))
                    row.append(p.value)
                self.staging2.append(row)
            self.stage2_arr = []
            for s2 in range(self.sets):
                flat = [self.recv_ptrs[s2][c] if p == rank else self.staging2[s2][c] + (p - rank) * self.cap * 8
                        for p in range(world) for c in range(ncols)]
                self.stage2_arr.append((C.c_void_p * len(flat))(*flat))
            self.dstream = torch.cuda.Stream(device=self.dev)
            self.got = [None] * self.sets
            for s in range(self.sets):
                # the kernel writes destination p at rows [rank*cap, ...) of the pointer it is given: bias the staging
                # pointer so that this lands in staging region p
                flat = [self.recv_ptrs[s][c] if p == rank else self.staging[c] + (p - rank) * self.cap * 8
                        for p in range(world) for c in range(ncols)]
                self.stage_arr.append((C.c_void_p * len(flat))(*flat))

    def _view(self, ptr: int, n: int):
        class _A:
            pass
        a = _A()
        a.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i8", "data": (ptr, False), "version": 3}
        return self.torch.as_tensor(a, device=self.dev)

    def exchange(self, key, cols, before_gather=None, trace=None):
        """cols[0] must be `key`.  Everything is enqueued on self.stream (the caller's current stream must be self.stream).
        `before_gather` (optional callable) runs between the scatter and the all-gather: a caller that probes on another
        stream makes self.stream wait there for its probe of the PREVIOUS step — the all-gather is what lets the peers
        move on to the step that overwrites the buffer set that probe is still reading, the scatter is not.
        -> (received columns: world*cap rows each, seg_cnt tensor [world], cap)"""
        torch, dist, lib, abi = self.torch, self.dist, self.lib, self.abi
        s = self.step % self.sets
        self.step += 1
        st = C.c_void_p(self.stream.cuda_stream)
        src_p = (C.c_void_p * len(cols))(*[c.data_ptr() for c in cols])

        def mark(name):
            if trace is not None:
                e = torch.cuda.Event(enable_timing=True); e.record(self.stream); trace.append((name, e))
        mark("x0")
        abi.check(lib.tg_partition_exchange_cf(self.device, C.c_void_p(key.data_ptr()), C.c_int64(key.numel()), self.world, len(cols), src_p,
                                               self.stage_arr[s] if self.dma else self.peer_arr[s], C.c_int64(self.rank * self.cap), C.c_int64(self.cap),
                                               C.c_void_p(self.sent[s].data_ptr()), C.c_void_p(self.overflow[s].data_ptr()), st))
        self.launches += 2
        if self.dma:
            # whole regions (capacity, not fill: the fill counts never reach the host), ring order so that the peers'
            # NVLink ingress is spread evenly
            regrouped = torch.cuda.Event(); regrouped.record(self.stream)
            for cs in self.copy_streams:
                cs.wait_event(regrouped)
            for k in range(1, self.world):
                p = (self.rank + k) % self.world
                cs = self.copy_streams[(k - 1) % len(self.copy_streams)]
                for c in range(len(cols)):
                    abi.check(lib.tg_memcpy_d2d_async(self.device, C.c_void_p(self.peer_ptrs[s][p][c] + self.rank * self.cap * 8),
                                                      C.c_void_p(self.staging[c] + p * self.cap * 8), C.c_size_t(self.cap * 8),
                                                      C.c_void_p(cs.cuda_stream)))
            for cs in self.copy_streams:
                sent = torch.cuda.Event(); sent.record(cs)
                self.stream.wait_event(sent)
        mark("scatter+dma enqueued-end")
        if before_gather is not None:
            before_gather()
        mark("after wait")
        # counts[src, dst] on every rank; completes only after every peer's scatter kernel (stream order) — the barrier
        dist.all_gather_into_tensor(self.count_mat[s], self.sent[s][:self.world])
        self.seg_cnt[s].copy_(self.count_mat[s].view(self.world, self.world)[:, self.rank])
        mark("gathered")
        return [self._view(self.recv_ptrs[s][c], self.world * self.cap) for c in range(len(cols))], self.seg_cnt[s], self.cap

    def exchange_async(self, key, cols, prev_probe_done=None, prev2_probe_done=None):
        """Pipelined form of exchange() (dma=True): three engines work on three different steps at once —
            self.stream : regroup step k into staging set k%2                         (SMs, HBM-bound)
            self.dstream: copy the regions of step k to the peers, then all-gather    (copy engines, NVLink-bound)
            caller      : probe step k-1                                              (SMs)
        `prev_probe_done`: event recorded after the caller's probe of the PREVIOUS step; the all-gather of this step waits
        for it (it releases the peers into the step that overwrites the receive set that probe reads).
        `prev2_probe_done`: event after the probe of the step BEFORE that one — it read the receive set this step's
        regrouping kernel writes its own rows into, so the kernel waits for it.
        -> (received columns, seg_cnt, cap, event to wait for before probing)"""
        assert self.dma, "exchange_async needs dma=True"
        torch, dist, lib, abi = self.torch, self.dist, self.lib, self.abi
        s = self.step % self.sets
        self.step += 1
        X, D = self.stream, self.dstream
        src_p = (C.c_void_p * len(cols))(*[c.data_ptr() for c in cols])
        with torch.cuda.stream(X):
            if self.got[s] is not None:
                X.wait_event(self.got[s])     # step k-2: its copies have left staging set s, its all-gather has read sent[s]
            if prev2_probe_done is not None:
                X.wait_event(prev2_probe_done)
            abi.check(lib.tg_partition_exchange_cf(self.device, C.c_void_p(key.data_ptr()), C.c_int64(key.numel()), self.world, len(cols), src_p,
                                                   self.stage2_arr[s], C.c_int64(self.rank * self.cap), C.c_int64(self.cap),
                                                   C.c_void_p(self.sent[s].data_ptr()), C.c_void_p(self.overflow[s].data_ptr()),
                                                   C.c_void_p(X.cuda_stream)))
            self.launches += 2
            regrouped = torch.cuda.Event(); regrouped.record(X)
        with torch.cuda.stream(D):
            D.wait_event(regrouped)
            for k in range(1, self.world):
                p = (self.rank + k) % self.world
                for c in range(len(cols)):
                    abi.check(lib.tg_memcpy_d2d_async(self.device, C.c_void_p(self.peer_ptrs[s][p][c] + self.rank * self.cap * 8),
                                                      C.c_void_p(self.staging2[s][c] + p * self.cap * 8), C.c_size_t(self.cap * 8),
                                                      C.c_void_p(D.cuda_stream)))
            if prev_probe_done is not None:
                D.wait_event(prev_probe_done)
            dist.all_gather_into_tensor(self.count_mat[s], self.sent[s][:self.world])
            self.seg_cnt[s].copy_(self.count_mat[s].view(self.world, self.world)[:, self.rank])
            got = torch.cuda.Event(); got.record(D)
            self.got[s] = got
        return [self._view(self.recv_ptrs[s][c], self.world * self.cap) for c in range(len(cols))], self.seg_cnt[s], self.cap, got

    def check_overflow(self):
        """host check (synchronises): raises when some step dropped rows because a region was too small"""
        bad = sum(int(o.item()) for o in self.overflow)
        flag = self.torch.tensor([bad], device=self.dev)
        self.dist.all_reduce(flag)
        if int(flag.item()):
            raise RuntimeError("count-free exchange overflowed a receive region: raise `slack` or use KeyExchange (counted)")

    def close(self):
        for s in range(self.sets):
            for p in range(self.world):
                if p == self.rank:
                    continue
                for c in range(self.ncols):
                    self.lib.tg_ipc_close(self.device, C.c_void_p(self.peer_ptrs[s][p][c]))
            for ptr in self.recv_ptrs[s]:
                self.lib.tg_dev_free(self.device, C.c_void_p(ptr))
        for ptr in self.staging + [q for row in getattr(self, "staging2", []) for q in row]:
            self.lib.tg_dev_free(self.device, C.c_void_p(ptr))
        self.recv_ptrs = []
        self.staging = []


class MailboxExchange:
    """Count-free key-hash exchange whose ONLY synchronisation is device-side mailboxes (tg_mail_signal / tg_mail_wait):
    no NCCL collective, no copy-engine call and no host wait inside a step, so a step is a fixed handful of kernel
    launches per rank (CUDA-graph capturable) and its cost does not depend on host-side enqueue latency.

      send()    on the exchange stream X:  wait for the peers' ACKs of the step that last used this buffer set,
                k_partition_scatter_bulk regroups 1024-row tiles by destination and appends each destination's run to
                this rank's region on that peer with bulk stores over NVLink (one kernel = repartition + all-to-all),
                then publishes the per-destination fill counts into every peer's COUNT mailbox;
      recv()    on the probe stream S: spin (on the device) until all `world` senders have published their count for
                this step; the counts land in seg_cnt, ready for tg_join_probe_dev_seg;
      release() on S after the probe: ACK to every sender that this buffer set may be overwritten.

    Two buffer sets: the exchange runs one step ahead of the probe.  PROTOCOL RULE: on every rank a wait may only depend
    on signals that were enqueued EARLIER in program order (send(k+1) waits for release(k-1), recv(k) for send(k)); a host
    call that synchronises the device can then never deadlock against a spinning wait kernel.
    dma=True keeps the SMs out of the transfer: the kernel regroups into a local staging copy of the region layout and
    copy engines push region p to peer p on several streams (fill is unknown to the host, so whole regions move).
    Reference analogue: MPP ExchangeSender/Receiver with HashPartition (physical_exchange_sender.go:115)."""

    KIND_COUNT, KIND_ACK = 0, 1
    SLOTS = 16   # TG_MAIL_MAX_PEERS

    def __init__(self, rank: int, world: int, device: int, xstream, ncols: int, rows_per_step: int, slack: float = 1.06,
                 dma: bool = False, ctas_per_sm: int = 0, timeout_ms: int = 10000, copy_streams: int = 0, direct_peers: int = 0,
                 sm_copy: bool = False, sm_copy_ctas: int = 0, spill_rows: int = 0):
        import torch
        import torch.distributed as dist
        from . import abi
        self.torch, self.dist, self.abi = torch, dist, abi
        self.lib = abi.load_lib()
        self.rank, self.world, self.device, self.stream, self.ncols = rank, world, device, xstream, ncols
        self.dev = torch.device("cuda", device)
        self.dma = bool(dma) and world > 1
        # dma + direct_peers = K: HYBRID transfer.  The regroup kernel stores the rows of the K next ranks (ring order) straight
        # into those peers over NVLink (SM bulk stores while the kernel runs) and stages the rest for the copy engines: the
        # two paths add up, the copy
        # engines' share shrinks until it hides behind the probe again
        self.direct = set(((rank + i) % world) for i in range(1, min(int(direct_peers), world - 1) + 1)) if self.dma else set()
        # dma + sm_copy: the staged regions are moved by tg_peer_copy_regions (an SM kernel small enough to sit next to the
        # persistent probe kernel: 128 threads x 32 registers, no shared memory) instead of the copy engines; it copies the
        # FILL of every region, read on the device
        self.sm_copy, self.sm_copy_ctas = bool(sm_copy) and self.dma, int(sm_copy_ctas)
        self.ctas_per_sm = int(ctas_per_sm)
        self.timeout_ms = int(timeout_ms)
        self.cap = region_capacity(rows_per_step, world, slack)
        self.sets = 2
        self.sent_steps = 0
        self.recv_steps = 0
        self.last_transfer = None    # event: the most recent step's transfer has been handed to the peers (dma mode)
        self.launches = 0
        lib = self.lib
        self.sent = [torch.zeros(self.SLOTS, dtype=torch.int64, device=self.dev) for _ in range(self.sets)]
        self.seg_cnt = [torch.zeros(world, dtype=torch.int64, device=self.dev) for _ in range(self.sets)]
        self.overflow = torch.zeros(1, dtype=torch.int64, device=self.dev)
        self.errflag = torch.zeros(1, dtype=torch.int64, device=self.dev)
        # spill_rows > 0: rows that do not fit their destination's region (skewed keys) are appended to a local spill area by
        # the regroup kernel instead of being dropped (tg_partition_exchange_cf_spill); drain_spill() hands them out after the
        # pipeline so the caller can move them with the counted exchange.  Skew then costs time, not rows.
        self.spill_rows = int(spill_rows)
        if self.spill_rows > 0:
            self.spill = [torch.empty(self.spill_rows + 2, dtype=torch.int64, device=self.dev) for _ in range(ncols)]
            self.spill_cursor = torch.zeros(1, dtype=torch.int64, device=self.dev)
            self.spill_arr = (C.c_void_p * ncols)(*[t.data_ptr() for t in self.spill])
        # receive buffers [set][col] and the mailbox block [kind][set][SLOTS] of this rank, all IPC-exported
        self.recv_ptrs, handles = [], []
        for _ in range(self.sets):
            row = []
            for _c in range(ncols):
                row.append(self._alloc(world * self.cap * 8 + 64, handles))
            self.recv_ptrs.append(row)
        self.mail_ptr = self._alloc(2 << 20, handles)   # a whole 2 MiB allocation: IPC handles map at allocation granularity
        abi.check(lib.tg_memcpy_h2d(device, C.c_void_p(self.mail_ptr), (C.c_uint64 * (2 * self.sets * self.SLOTS))(), C.c_size_t(2 * self.sets * self.SLOTS * 8)))
        gathered = [None] * world
        dist.all_gather_object(gathered, handles)
        self._mapped = []
        def peer_ptr(p, idx):
            if p == rank:
                return ([q for row in self.recv_ptrs for q in row] + [self.mail_ptr])[idx]
            mp = C.c_void_p()
            hb = (C.c_uint8 * 64).from_buffer_copy(gathered[p][idx])
            abi.check(lib.tg_ipc_open(device, hb, C.byref(mp)))
            self._mapped.append(mp.value)
            return mp.value
        self.peer_recv = [[[peer_ptr(p, s_ * ncols + c) for c in range(ncols)] for p in range(world)] for s_ in range(self.sets)]   # [set][peer][col]
        self.peer_mail = [peer_ptr(p, self.sets * ncols) for p in range(world)]
        self.peer_arr = []
        for s_ in range(self.sets):
            flat = [self.peer_recv[s_][p][c] for p in range(world) for c in range(ncols)]
            self.peer_arr.append((C.c_void_p * len(flat))(*flat))
        # where this rank's words live inside every peer's mailbox block
        self.targets = {}
        for kind in (self.KIND_COUNT, self.KIND_ACK):
            for s_ in range(self.sets):
                t = abi.TgMailTargets()
                t.n = world
                for p in range(world):
                    t.slot[p] = self.peer_mail[p] + ((kind * self.sets + s_) * self.SLOTS + rank) * 8
                self.targets[(kind, s_)] = t
        if self.dma:
            self.staging, self.stage_arr, self.staged_free = [], [], [None] * self.sets
            for s_ in range(self.sets):
                row = [self._alloc(world * self.cap * 8 + 64, None) for _c in range(ncols)]
                self.staging.append(row)
                # the kernel writes destination p at rows [rank*cap, ...) of the pointer it is given: bias the staging
                # pointer so that this lands in staging region p; own rows go straight into the own receive set
                flat = [self.recv_ptrs[s_][c] if p == rank else (self.peer_recv[s_][p][c] if p in self.direct else row[c] + (p - rank) * self.cap * 8)
                        for p in range(world) for c in range(ncols)]
                self.stage_arr.append((C.c_void_p * len(flat))(*flat))
            # one stream drives one copy engine at a time: the (world-1) x ncols region copies are spread over several streams
            # (default: one per copy, at most 16): with a few streams the transfer, not the SMs, bounds the step
            ncs = copy_streams if copy_streams > 0 else min(16, (world - 1) * ncols)
            self.copy_streams = [torch.cuda.Stream(device=self.dev) for _ in range(max(1, ncs))]
            self.dstream = torch.cuda.Stream(device=self.dev)
        torch.cuda.synchronize(self.dev)
        dist.barrier()    # every mailbox is zeroed and mapped before anybody signals

    def _alloc(self, nbytes, handles):
        p = C.c_void_p()
        self.abi.check(self.lib.tg_dev_alloc(self.device, C.c_size_t(nbytes), C.byref(p)))
        if handles is not None:
            h = (C.c_uint8 * 64)()
            self.abi.check(self.lib.tg_ipc_export(self.device, p, h))
            handles.append(bytes(h))
        return p.value

    def _mail(self, kind, s_):
        return self.mail_ptr + (kind * self.sets + s_) * self.SLOTS * 8

    def _view(self, ptr: int, n: int):
        class _A:
            pass
        a = _A()
        a.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i8", "data": (ptr, False), "version": 3}
        return self.torch.as_tensor(a, device=self.dev)

    def _scatter(self, key, ncols, src_p, dst_arr, s_, X):
        """the regroup kernel of one step: 1024-row tiles regrouped by destination rank, bulk stores into the regions"""
        lib, abi = self.lib, self.abi
        if self.spill_rows > 0:
            if ncols != self.ncols:
                raise ValueError("the spill area was sized for the exchange's column count")
            abi.check(lib.tg_partition_exchange_cf_spill(self.device, C.c_void_p(key.data_ptr()), C.c_int64(key.numel()), self.world, ncols, src_p,
                                                         dst_arr, C.c_int64(self.rank * self.cap), C.c_int64(self.cap),
                                                         C.c_void_p(self.sent[s_].data_ptr()), C.c_void_p(self.overflow.data_ptr()),
                                                         self.spill_arr, C.c_int64(self.spill_rows), C.c_void_p(self.spill_cursor.data_ptr()),
                                                         C.c_int32(self.ctas_per_sm), X))
        else:
            abi.check(lib.tg_partition_exchange_cf_ex(self.device, C.c_void_p(key.data_ptr()), C.c_int64(key.numel()), self.world, ncols, src_p,
                                                      dst_arr, C.c_int64(self.rank * self.cap), C.c_int64(self.cap),
                                                      C.c_void_p(self.sent[s_].data_ptr()), C.c_void_p(self.overflow.data_ptr()), C.c_int32(self.ctas_per_sm), X))

    def drain_spill(self):
        """host call after the pipelined steps (synchronises this device): the rows the regroup kernel could not place in
        their destination's region since the last drain, as column tensors (views of the spill area, valid until the next
        send) -> (rows, [col tensors]); the spill cursor is reset.  The caller moves them with the counted exchange
        (KeyExchange) and probes them like any other batch.  Collective-free; every rank must call the follow-up exchange
        even with 0 spilled rows."""
        if self.spill_rows <= 0:
            return 0, []
        self.torch.cuda.synchronize(self.dev)
        n = int(self.spill_cursor.item())
        if n > self.spill_rows:
            raise RuntimeError("count-free exchange: the spill area overflowed as well (raise spill_rows)")
        self.spill_cursor.zero_()
        return n, [t[:n] for t in self.spill]

    def send(self, key, cols, compute_stream=None):
        """enqueue step k's repartition + transfer + count publication; cols[0] must be `key`.
        The SM kernel (regroup / scatter) goes on `compute_stream` (default: the exchange stream given to the constructor).
        Putting it on the SAME stream as the probe keeps the shared-memory-heavy scatter and the L1-hungry probe kernel
        from ever sharing an SM (the probe slows down under a large shared-memory carve-out); with
        dma=True the NVLink transfer then overlaps the probe on the copy engines."""
        lib, abi, torch = self.lib, self.abi, self.torch
        k = self.sent_steps
        self.sent_steps += 1
        s_, epoch = k % self.sets, k + 1
        cs_ = compute_stream if compute_stream is not None else self.stream
        X = C.c_void_p(cs_.cuda_stream)
        src_p = (C.c_void_p * len(cols))(*[c.data_ptr() for c in cols])
        err = C.c_void_p(self.errflag.data_ptr())
        if not self.dma:
            if k >= self.sets:   # every peer has finished probing the step that used this buffer set
                abi.check(lib.tg_mail_wait(self.device, C.c_void_p(self._mail(self.KIND_ACK, s_)), self.world, C.c_int64(epoch - self.sets), None, err, C.c_int64(self.timeout_ms), X))
            self._scatter(key, len(cols), src_p, self.peer_arr[s_], s_, X)
            abi.check(lib.tg_mail_signal(self.device, C.byref(self.targets[(self.KIND_COUNT, s_)]), C.c_void_p(self.sent[s_].data_ptr()), C.c_int64(epoch), X))
            self.launches += 4 if k >= self.sets else 3
            return
        D = self.dstream
        with torch.cuda.stream(cs_):
            if self.staged_free[s_] is not None:
                cs_.wait_event(self.staged_free[s_])      # the copies of step k-2 have left staging set s_
            if k >= self.sets and (cs_ is self.stream or self.direct):
                # own rows go straight into the own receive set: the own probe of step k-2 must be done.  (On the probe's own
                # stream that is stream order; on a separate exchange stream it is the ACK mailbox, which includes this rank.)
                # Hybrid transfer: the kernel also stores into the direct peers, whose probes of step k-2 must be done.
                abi.check(lib.tg_mail_wait(self.device, C.c_void_p(self._mail(self.KIND_ACK, s_)), self.world, C.c_int64(epoch - self.sets), None, err, C.c_int64(self.timeout_ms), X))
            self._scatter(key, len(cols), src_p, self.stage_arr[s_], s_, X)
            regrouped = torch.cuda.Event(); regrouped.record(cs_)
        with torch.cuda.stream(D):
            D.wait_event(regrouped)
            if k >= self.sets:   # the peers have finished probing the step that used the receive set the copies overwrite
                abi.check(lib.tg_mail_wait(self.device, C.c_void_p(self._mail(self.KIND_ACK, s_)), self.world, C.c_int64(epoch - self.sets), None, err, C.c_int64(self.timeout_ms), C.c_void_p(D.cuda_stream)))
            ready = torch.cuda.Event(); ready.record(D)
        if self.sm_copy:
            with torch.cuda.stream(D):
                srcs, dsts, idx = [], [], []
                for i in range(1, self.world):
                    p = (self.rank + i) % self.world
                    if p in self.direct:
                        continue
                    for c in range(len(cols)):
                        srcs.append(self.staging[s_][c] + p * self.cap * 8); dsts.append(self.peer_recv[s_][p][c] + self.rank * self.cap * 8); idx.append(p)
                if srcs:
                    abi.check(lib.tg_peer_copy_regions(self.device, len(srcs), (C.c_void_p * len(srcs))(*srcs), (C.c_void_p * len(dsts))(*dsts),
                                                       (C.c_int32 * len(idx))(*idx), C.c_void_p(self.sent[s_].data_ptr()), C.c_int64(self.cap),
                                                       C.c_int32(self.sm_copy_ctas), C.c_void_p(D.cuda_stream)))
                abi.check(lib.tg_mail_signal(self.device, C.byref(self.targets[(self.KIND_COUNT, s_)]), C.c_void_p(self.sent[s_].data_ptr()), C.c_int64(epoch), C.c_void_p(D.cuda_stream)))
                done = torch.cuda.Event(); done.record(D)
                self.staged_free[s_] = done
                self.last_transfer = done
            self.launches += 5 if k >= self.sets else 4
            return
        for cs in self.copy_streams:
            cs.wait_event(ready)
        q = 0
        for i in range(1, self.world):
            p = (self.rank + i) % self.world      # ring order spreads the peers' NVLink ingress
            if p in self.direct:
                continue                          # already stored by the regroup kernel
            for c in range(len(cols)):
                cs = self.copy_streams[q % len(self.copy_streams)]; q += 1
                abi.check(lib.tg_memcpy_d2d_async(self.device, C.c_void_p(self.peer_recv[s_][p][c] + self.rank * self.cap * 8),
                                                  C.c_void_p(self.staging[s_][c] + p * self.cap * 8), C.c_size_t(self.cap * 8), C.c_void_p(cs.cuda_stream)))
        with torch.cuda.stream(D):
            for cs in self.copy_streams:
                e = torch.cuda.Event(); e.record(cs); D.wait_event(e)
            abi.check(lib.tg_mail_signal(self.device, C.byref(self.targets[(self.KIND_COUNT, s_)]), C.c_void_p(self.sent[s_].data_ptr()), C.c_int64(epoch), C.c_void_p(D.cuda_stream)))
            done = torch.cuda.Event(); done.record(D)
            self.staged_free[s_] = done
            self.last_transfer = done
        self.launches += 4 if k >= self.sets else 3

    def recv(self, probe_stream):
        """enqueue on `probe_stream` the wait for step k's counts -> (received columns, seg_cnt tensor, cap, set, epoch)"""
        k = self.recv_steps
        self.recv_steps += 1
        s_, epoch = k % self.sets, k + 1
        self.abi.check(self.lib.tg_mail_wait(self.device, C.c_void_p(self._mail(self.KIND_COUNT, s_)), self.world, C.c_int64(epoch),
                                             C.c_void_p(self.seg_cnt[s_].data_ptr()), C.c_void_p(self.errflag.data_ptr()), C.c_int64(self.timeout_ms),
                                             C.c_void_p(probe_stream.cuda_stream)))
        self.launches += 1
        return [self._view(self.recv_ptrs[s_][c], self.world * self.cap) for c in range(self.ncols)], self.seg_cnt[s_], self.cap, s_, epoch

    def release(self, probe_stream, s_, epoch):
        """enqueue on `probe_stream`, after the consumer of set `s_`: tell every sender the set may be overwritten"""
        self.abi.check(self.lib.tg_mail_signal(self.device, C.byref(self.targets[(self.KIND_ACK, s_)]), None, C.c_int64(epoch), C.c_void_p(probe_stream.cuda_stream)))
        self.launches += 1

    def discard_outstanding(self, probe_stream):
        """consume (without probing) every step that was sent but not received yet, e.g. the step a pipelined loop keeps in
        flight when it stops; afterwards sends and receives are level again"""
        while self.recv_steps < self.sent_steps:
            _c, _n, _cap, s_, ep = self.recv(probe_stream)
            self.release(probe_stream, s_, ep)

    def check(self):
        """host check (synchronises): a region overflow or a mailbox timeout anywhere fails the run on every rank"""
        self.torch.cuda.synchronize(self.dev)
        flag = self.torch.stack([self.overflow[0], self.errflag[0]]).clone()
        flag = (flag != 0).to(self.torch.int64)
        self.dist.all_reduce(flag)
        if int(flag[1].item()):
            raise RuntimeError("mailbox wait timed out on some rank: a peer never published its step (see tg_mail_wait)")
        if int(flag[0].item()):
            raise RuntimeError("count-free exchange overflowed a receive region: raise `slack` or use KeyExchange (counted)")

    def close(self):
        self.torch.cuda.synchronize(self.dev)
        self.dist.barrier()
        for mp in self._mapped:
            self.lib.tg_ipc_close(self.device, C.c_void_p(mp))
        for row in self.recv_ptrs + (self.staging if self.dma else []):
            for ptr in row:
                self.lib.tg_dev_free(self.device, C.c_void_p(ptr))
        self.lib.tg_dev_free(self.device, C.c_void_p(self.mail_ptr))
        self.recv_ptrs, self._mapped = [], []
