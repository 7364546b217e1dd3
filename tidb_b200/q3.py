"""TPC-H Q3-shape pipeline on device-resident synthetic columns (BASELINE.json configs[3]).

Plan shape follows the reference's TiFlash MPP plan for Q3 (pkg/planner/core/casetest/tpch/testdata/tpch_suite_out.json:99-123):

    HashAgg(group by l_orderkey, o_orderdate, o_shippriority; sum(l_extendedprice * (1 - l_discount)))
      HashJoin(lineitem.l_orderkey = orders.o_orderkey)            probe: Selection(l_shipdate > D) on lineitem
        HashJoin(orders.o_custkey = customer.c_custkey)            probe: Selection(o_orderdate < D) on orders
          Selection(c_mktsegment = S) on customer                  (build side)

Everything runs through the C-ABI operators: the three Selections are fused into the joins as build / probe
filters (tg_filter_item), and the
aggregation is tg_agg with all three GROUP BY columns (tag-claimed multi-word slots) and the projection
l_extendedprice * (1 - l_discount) fused into its update kernel (tg_agg_func.arg_expr), followed by tg_topn.

By default the prices are DOUBLE.  gen(..., decimal=True) gives l_extendedprice and l_discount TiDB's real type,
DECIMAL(15,2), as 40-byte MyDecimal cells; run() then carries the cells through J2, sums the exact DECIMAL revenue at
scale 4 and orders TopN by that DECIMAL column.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Dict

import torch

from . import abi
from .device import DeviceAgg, DeviceJoin
from .plan import AggFunc, AggPlan, FieldType, FilterItem, JoinPlan

INT = FieldType(abi.TYPE_LONGLONG, abi.FLAG_NOT_NULL)
DBL = FieldType(abi.TYPE_DOUBLE, abi.FLAG_NOT_NULL)
PRICE = FieldType(abi.TYPE_NEWDECIMAL, abi.FLAG_NOT_NULL, 15, 2)   # l_extendedprice / l_discount DECIMAL(15,2)
REVENUE_FRAC = 4                                                    # SUM(DECIMAL(15,2) * (1 - DECIMAL(15,2))): scale 2 + 2
SEGMENT, DATE = 1, 1168   # c_mktsegment = 1, o_orderdate < 1168 < l_shipdate  (SURVEY §8d)


@dataclass
class Q3Data:
    c_custkey: torch.Tensor; c_seg: torch.Tensor
    o_orderkey: torch.Tensor; o_custkey: torch.Tensor; o_date: torch.Tensor; o_prio: torch.Tensor
    l_orderkey: torch.Tensor; l_price: torch.Tensor; l_disc: torch.Tensor; l_ship: torch.Tensor

    def scanned_bytes(self) -> int:
        return sum(t.numel() * t.element_size() for t in self.__dict__.values())


def price_cells(cents: torch.Tensor) -> torch.Tensor:
    """int64 values * 100 -> DECIMAL(15,2) cells as MyDecimal.FromBin stores them (digitsInt 13: two integer words; one
    fraction word, left-aligned), an (n, 40) uint8 tensor; values are non-negative"""
    n = cents.numel()
    w = torch.zeros((n, 10), dtype=torch.int32, device=cents.device)
    w[:, 0] = 13 | (2 << 8)
    ip = cents // 100
    w[:, 1] = (ip // 10**9).to(torch.int32)
    w[:, 2] = (ip % 10**9).to(torch.int32)
    w[:, 3] = ((cents % 100) * 10**7).to(torch.int32)
    return w.view(torch.uint8).view(n, 40)


def cents_of(cells: torch.Tensor) -> torch.Tensor:
    """price_cells' inverse"""
    w = cells.view(torch.int32).view(-1, 10).to(torch.int64)
    return (w[:, 1] * 10**9 + w[:, 2]) * 100 + w[:, 3] // 10**7


def gen(dev, n_cust: int, n_orders: int, n_line: int, seed: int = 42, rank: int = 0, world: int = 1, decimal: bool = False) -> Q3Data:
    """rank's shard of the tables (world = 1: the whole tables).  Keys are global: customer / order keys are unique across
    ranks, foreign keys are uniform over the GLOBAL key sets, and rows land on ranks at random — nothing is co-partitioned,
    so the multi-GPU plan has to exchange.  decimal=True: l_price / l_disc are the same values as DECIMAL(15,2) cells
    (price_cells); every other column is as with DOUBLE prices."""
    g = torch.Generator(device=dev); g.manual_seed(seed + 1000 * rank)
    ri = lambda lo, hi, n: torch.randint(lo, hi, (n,), device=dev, generator=g, dtype=torch.int64)
    nc, no, nl = n_cust // world, n_orders // world, n_line // world
    n_cust, n_orders = nc * world, no * world
    d = Q3Data(
        c_custkey=torch.randperm(nc, device=dev, generator=g, dtype=torch.int64) + rank * nc, c_seg=ri(0, 5, nc),
        o_orderkey=(torch.randperm(no, device=dev, generator=g, dtype=torch.int64) + rank * no) * 4 + 1, o_custkey=ri(0, n_cust, no),
        o_date=ri(0, 2406, no), o_prio=ri(0, 5, no),
        l_orderkey=ri(0, n_orders, nl) * 4 + 1,
        l_price=torch.floor(torch.rand(nl, device=dev, generator=g, dtype=torch.float64) * 100000) / 100,
        l_disc=torch.floor(torch.rand(nl, device=dev, generator=g, dtype=torch.float64) * 11) / 100,
        l_ship=ri(0, 2406, nl))
    if decimal:
        d.l_price = price_cells(torch.round(d.l_price * 100).to(torch.int64))
        d.l_disc = price_cells(torch.round(d.l_disc * 100).to(torch.int64))
    return d


def _view(ptr: int, n: int, dev, dt="<i8"):
    """a device column as a tensor; dt "cell": (n, 40) uint8 DECIMAL cells"""
    class _A:
        pass
    a = _A()
    shape, dt = ((n, 40), "|u1") if dt == "cell" else ((n,), dt)
    a.__cuda_array_interface__ = {"shape": shape, "typestr": dt, "data": (ptr, False), "version": 3}
    return torch.as_tensor(a, device=dev)


def _col_struct(ptr: int, n: int, nulls: int = 0, elem: int = 8):
    c = abi.TgColumn(); c.length = n; c.data = ptr or None; c.elem_len = elem; c.null_bitmap = nulls or None; c.offsets = None
    return c


def run(d: Q3Data, dev, stream, topn: int = 10, timings: Dict[str, float] = None, keep_groups: bool = True, j1_out=None) -> Dict[str, torch.Tensor]:
    """The whole query on the device.  -> {orderkey, revenue, o_date, o_prio} of every group (unordered, device tensors) and,
    under "top", the TopN rows (host numpy arrays, ORDER BY revenue DESC, o_orderdate LIMIT topn).
    Operators: J1 = orders JOIN customer (Selections fused as build/probe filters), J2 = lineitem JOIN J1 (J1's device-resident
    output is the build side, borrowed, no copy), HashAgg GROUP BY (l_orderkey, o_orderdate, o_shippriority) with
    SUM(l_extendedprice * (1 - l_discount)) evaluated INSIDE the update kernel (tg_agg_func.arg_expr: no projected column,
    the constant is a scalar), TopN (tg_topn).
    With DECIMAL prices (gen(decimal=True)) the plan is the exact one: J2 carries the two DECIMAL(15,2) columns, the
    aggregation sums the exact DECIMAL products at scale 4 (TG_ARGEXPR_MUL_CSUB, ret_type DECIMAL), "revenue" is an
    (groups, 40) uint8 tensor of MyDecimal cells and TopN orders by that DECIMAL column."""
    import numpy as np
    from .chunk import DECIMAL_DTYPE
    lib = abi.load_lib()
    dec = d.l_price.dim() == 2
    PT = PRICE if dec else DBL
    st = stream.cuda_stream
    di = dev.index or 0
    marks = []

    def mark(name):
        if timings is not None:
            e = torch.cuda.Event(enable_timing=True); e.record(stream); marks.append((name, e))
    mark("start")
    if j1_out is not None:     # multi-GPU plan: J1 ran before the exchange, its (repartitioned) output is handed in
        n1, j1_cols, j1 = j1_out[0].numel(), list(j1_out), None
    else:
      # J1: orders (probe, filter o_date < D) JOIN customer (build, filter c_seg = S); keep o_orderkey, o_date, o_prio
      j1 = DeviceJoin(JoinPlan(abi.JOIN_INNER, [INT] * 4, [INT] * 2, [1], [0], build_is_right=True, lused=[0, 2, 3], rused=[],
                             build_filter=[FilterItem(abi.CMP_EQ, 1, const_i64=SEGMENT)], probe_filter=[FilterItem(abi.CMP_LT, 2, const_i64=DATE)],
                             device=di, stream=st))
      j1.build([d.c_custkey, d.c_seg])
      mark("J1 build (customer, c_mktsegment filter fused)")
      n1, c1, _ = j1.probe([d.o_orderkey, d.o_custkey, d.o_date, d.o_prio])
      mark("J1 probe (orders, o_orderdate filter fused)")
      j1_cols = [_view(p, n1, dev) for p in c1]
    # J2: lineitem (probe, filter l_ship > D) JOIN J1 (build on o_orderkey); keep l_orderkey, l_price, l_disc, o_date, o_prio
    j2 = DeviceJoin(JoinPlan(abi.JOIN_INNER, [INT, PT, PT, INT], [INT] * 3, [0], [0], build_is_right=True, lused=[0, 1, 2], rused=[1, 2],
                             probe_filter=[FilterItem(abi.CMP_GT, 3, const_i64=DATE)], device=di, stream=st))
    j2.build(j1_cols)     # borrowed until build_finish: J1's result buffers are read in place
    mark("J2 build (J1 output, in place)")
    if j1 is not None:
        j1.close()
    n2, c2, _ = j2.probe([d.l_orderkey, d.l_price, d.l_disc, d.l_ship])
    mark("J2 probe (lineitem, l_shipdate filter fused)")
    vdt = "cell" if dec else "<f8"
    lk = _view(c2[0], n2, dev); price = _view(c2[1], n2, dev, vdt); disc = _view(c2[2], n2, dev, vdt)
    jd = _view(c2[3], n2, dev); jp = _view(c2[4], n2, dev)
    # HashAgg: GROUP BY l_orderkey, o_orderdate, o_shippriority; SUM(l_extendedprice * (1 - l_discount)) fused
    revenue = (AggFunc(abi.AGG_SUM, 1, abi.TYPE_NEWDECIMAL, arg_col2=2, arg_expr=abi.ARGEXPR_MUL_CSUB, arg_const=1.0,
                       ret_type=abi.TYPE_NEWDECIMAL, ret_frac=REVENUE_FRAC) if dec else
               AggFunc(abi.AGG_SUM, 1, abi.TYPE_DOUBLE, arg_col2=2, arg_expr=abi.ARGEXPR_MUL_CSUB, arg_const=1.0))
    agg = DeviceAgg(AggPlan([INT, PT, PT, INT, INT], [0, 3, 4],
                            [AggFunc(abi.AGG_FIRSTROW, 0), revenue, AggFunc(abi.AGG_FIRSTROW, 3), AggFunc(abi.AGG_FIRSTROW, 4)],
                            device=di, stream=st, expected_groups=max(n1, 1)))
    agg.push([lk, price, disc, jd, jp])
    ng, ca, na = agg.finish()
    mark("HashAgg (3 GROUP BY columns, projection fused)")
    if timings is not None:
        ast_ = agg.stats()
        timings["agg_kernels_ms"] = {"update": round(ast_.update_ms, 3), "finalize": round(ast_.finalize_ms, 3), "table_slots": int(ast_.table_slots), "launches": int(ast_.kernel_launches)}
    out = {"groups": ng}
    if keep_groups:   # copies of the whole aggregate result (verification); the query's own result is the TopN below
        out.update({"orderkey": _view(ca[0], ng, dev).clone(), "revenue": _view(ca[1], ng, dev, vdt).clone(),
                    "o_date": _view(ca[2], ng, dev).clone(), "o_prio": _view(ca[3], ng, dev).clone()})
    # TopN: ORDER BY revenue DESC, o_orderdate LIMIT topn  (tpch_suite_out.json:102)
    if topn > 0:
        rev_elem = 40 if dec else 8
        cols = (abi.TgColumn * 4)(*[_col_struct(ca[k], ng, na[k], rev_elem if k == 1 else 8) for k in range(4)])
        ck = abi.TgChunk(); ck.ncols = 4; ck.cols = C.cast(cols, C.POINTER(abi.TgColumn)); ck.sel = None; ck.nsel = 0
        tps = (C.c_int32 * 4)(abi.TYPE_LONGLONG, abi.TYPE_NEWDECIMAL if dec else abi.TYPE_DOUBLE, abi.TYPE_LONGLONG, abi.TYPE_LONGLONG)
        fls = (C.c_uint32 * 4)(0, 0, 0, 0)
        items = (abi.TgSortItem * 2)(abi.TgSortItem(1, 1), abi.TgSortItem(2, 0))
        from .chunk import MutChunk
        oc = MutChunk([8, rev_elem, 8, 8], max(topn, 8), [np.int64, DECIMAL_DTYPE if dec else np.float64, np.int64, np.int64])
        got = C.c_int64(0)
        abi.check(lib.tg_topn(di, 1, C.byref(ck), tps, fls, items, 2, C.c_int64(0), C.c_int64(topn), C.byref(oc.struct), C.byref(got), C.c_void_p(st)))
        out["top"] = [v.copy() for v, _ in oc.columns(got.value)]
        mark("TopN")
    agg.close(); j2.close()
    if timings is not None:
        stream.synchronize()
        for (_, a), (name, b) in zip(marks[:-1], marks[1:]):
            timings[name] = timings.get(name, 0.0) + a.elapsed_time(b)
        timings["rows"] = {"j1_out": n1, "j2_out": n2, "groups": ng}
    return out


class Q3Distributed:
    """The Q3-shape plan on N GPUs (one process per GPU), the MPP shape of tpch_suite_out.json:99-123 / SURVEY 8e:
      1. customer is small: every rank all-gathers the customer columns (the broadcast side) and runs J1 on its own orders shard;
      2. the filtered orders (J1 output) and lineitem are REPARTITIONED by order key over NVLink (KeyExchange: scatter
         kernel storing into the peers, ExchangeType HashPartition in the reference plan), so equal order keys meet;
      3. J2, the aggregation and TopN run shard-locally — the GROUP BY key contains the partition key, so groups never span
         ranks and no partial -> final aggregate exchange is needed;
      4. the N local TopN results (N x topn rows) are gathered and reduced by one more tg_topn."""

    def __init__(self, rank: int, world: int, dev, stream, orders_rows: int, lineitem_rows: int):
        from .parallel import KeyExchange
        self.rank, self.world, self.dev, self.stream = rank, world, dev, stream
        di = dev.index or 0
        with torch.cuda.stream(stream):
            self.x_orders = KeyExchange(rank, world, di, stream, 3, int(orders_rows * 0.25) + 65536, "p2p")     # J1 keeps ~10 % of the orders
            self.x_line = KeyExchange(rank, world, di, stream, 4, int(lineitem_rows * 1.05) + 65536, "p2p")

    def run(self, d: Q3Data, topn: int = 10, timings: Dict[str, float] = None) -> Dict:
        import numpy as np
        import torch.distributed as dist
        dev, stream, world = self.dev, self.stream, self.world
        st, di = stream.cuda_stream, dev.index or 0
        marks = []

        def mark(name):
            if timings is not None:
                e = torch.cuda.Event(enable_timing=True); e.record(stream); marks.append((name, e))
        with torch.cuda.stream(stream):
            mark("start")
            nc = d.c_custkey.numel()
            ck = torch.empty(nc * world, dtype=torch.int64, device=dev); cs = torch.empty(nc * world, dtype=torch.int64, device=dev)
            dist.all_gather_into_tensor(ck, d.c_custkey); dist.all_gather_into_tensor(cs, d.c_seg)
            mark("broadcast customer (all-gather)")
            j1 = DeviceJoin(JoinPlan(abi.JOIN_INNER, [INT] * 4, [INT] * 2, [1], [0], build_is_right=True, lused=[0, 2, 3], rused=[],
                                     build_filter=[FilterItem(abi.CMP_EQ, 1, const_i64=SEGMENT)], probe_filter=[FilterItem(abi.CMP_LT, 2, const_i64=DATE)],
                                     device=di, stream=st))
            j1.build([ck, cs])
            n1, c1, _ = j1.probe([d.o_orderkey, d.o_custkey, d.o_date, d.o_prio])
            mark("J1 (local orders shard x all customers)")
            o_cols = [_view(p, n1, dev) for p in c1]
            ok, od, op = self.x_orders.exchange(o_cols[0], o_cols)
            j1.close()
            mark("repartition filtered orders by o_orderkey")
            lk, lp, ld, ls = self.x_line.exchange(d.l_orderkey, [d.l_orderkey, d.l_price.view(torch.int64), d.l_disc.view(torch.int64), d.l_ship])
            mark("repartition lineitem by l_orderkey")
            part = Q3Data(c_custkey=ck, c_seg=cs, o_orderkey=ok, o_custkey=ok, o_date=od, o_prio=op,
                          l_orderkey=lk, l_price=lp.view(torch.float64), l_disc=ld.view(torch.float64), l_ship=ls)
            t2 = {} if timings is not None else None
            out = run(part, dev, stream, topn=topn, timings=t2, keep_groups=False, j1_out=(ok, od, op))
            mark("local J2 + HashAgg + TopN")
            # global TopN over the N local results
            top = out.get("top", [np.zeros(0, dtype=np.int64), np.zeros(0), np.zeros(0, dtype=np.int64), np.zeros(0, dtype=np.int64)])
            gathered = [None] * world
            dist.all_gather_object(gathered, [t.tolist() for t in top])
            groups = torch.tensor([out["groups"]], dtype=torch.int64, device=dev); dist.all_reduce(groups)
            mark("gather local TopN")
        cols = [np.array(sum((g[c] for g in gathered), []), dtype=np.float64 if c == 1 else np.int64) for c in range(4)]
        n = len(cols[0])
        final = cols
        if n > 0:
            lib = abi.load_lib()
            from .chunk import Chunk, Column, MutChunk
            ck_ = Chunk([Column(c) for c in cols]).to_struct()
            tps = (C.c_int32 * 4)(abi.TYPE_LONGLONG, abi.TYPE_DOUBLE, abi.TYPE_LONGLONG, abi.TYPE_LONGLONG)
            fls = (C.c_uint32 * 4)(0, 0, 0, 0)
            items = (abi.TgSortItem * 2)(abi.TgSortItem(1, 1), abi.TgSortItem(2, 0))
            oc = MutChunk([8, 8, 8, 8], max(topn, 8), [np.int64, np.float64, np.int64, np.int64])
            got = C.c_int64(0)
            abi.check(lib.tg_topn(di, 0, C.byref(ck_), tps, fls, items, 2, C.c_int64(0), C.c_int64(topn), C.byref(oc.struct), C.byref(got), C.c_void_p(st)))
            final = [v.copy() for v, _ in oc.columns(got.value)]
        if timings is not None:
            stream.synchronize()
            for (_, a), (name, b) in zip(marks[:-1], marks[1:]):
                timings[name] = timings.get(name, 0.0) + a.elapsed_time(b)
            timings["local"] = t2
        return {"top": final, "groups": int(groups.item())}

    def close(self):
        self.x_orders.close(); self.x_line.close()


def reference(d: Q3Data) -> Dict[str, torch.Tensor]:
    """the same query with plain torch ops (verification only).  "revenue_s4" is the exact revenue as an integer at scale 4
    (the prices are whole cents in either form); with DECIMAL prices "revenue" is that value as a double."""
    cust_ok = torch.zeros(int(d.c_custkey.max().item()) + 1, dtype=torch.bool, device=d.c_custkey.device)
    cust_ok[d.c_custkey[d.c_seg == SEGMENT]] = True
    om = (d.o_date < DATE) & cust_ok[d.o_custkey]
    n_ok = int(d.o_orderkey.max().item()) + 1
    order_row = torch.full((n_ok,), -1, dtype=torch.int64, device=om.device)
    idx = torch.nonzero(om).flatten()
    order_row[d.o_orderkey[idx]] = idx
    lm = d.l_ship > DATE
    lk = d.l_orderkey[lm]
    orow = order_row[lk]
    keep = orow >= 0
    lk, orow = lk[keep], orow[keep]
    dec = d.l_price.dim() == 2
    price, disc = d.l_price[lm][keep], d.l_disc[lm][keep]
    pc, dc = (cents_of(price), cents_of(disc)) if dec else (torch.round(price * 100).to(torch.int64), torch.round(disc * 100).to(torch.int64))
    keys, inv = torch.unique(lk, return_inverse=True)
    s4 = torch.zeros(keys.numel(), dtype=torch.int64, device=lk.device).scatter_add_(0, inv, pc * (100 - dc))
    if dec:
        s = s4.to(torch.float64) / 10**REVENUE_FRAC
    else:
        rev = (price * (1 - disc))
        s = torch.zeros(keys.numel(), dtype=torch.float64, device=lk.device).scatter_add_(0, inv, rev)
    first = torch.zeros(keys.numel(), dtype=torch.int64, device=lk.device).scatter_(0, inv, orow)
    return {"orderkey": keys, "revenue": s, "revenue_s4": s4, "o_date": d.o_date[first], "o_prio": d.o_prio[first]}
