"""The DECIMAL VecEval calls against the same work over DOUBLE and against a plain device copy, on one GPU.

    python tools/bench_vec_decimal.py [--rows 100000000] [--rounds 5] [--warmup 2] [--steps 3]

Workload, all device-resident (`rows` rows, TPC-H Q6's lineitem columns):
  filter_dec   tg_vec_filter_ex: l_shipdate >= d0 AND l_shipdate < d1 (BIGINT items) AND l_discount BETWEEN 0.05 AND 0.07
               AND l_quantity < 24 (DECIMAL(15,2) items over 40-byte cells in MyDecimal.FromBin's form)
  filter_dbl   tg_vec_filter: the same predicate over DOUBLE l_discount / l_quantity columns
  cmp_const    tg_vec_compare_decimal: l_quantity < 24
  cmp_col      tg_vec_compare_decimal: l_discount < l_quantity
  copy         a device-to-device copy of one 40-byte cell column (cudaMemcpyAsync), the measured ceiling
Each step is one call timed with CUDA events; the plans alternate within each round in one process, so all see the same
clocks and neighbours on a shared machine.  Bytes per row come from the shapes (what a call must read and write); GB/s
is those bytes over the median call time, and `of_copy` its ratio to the copy's rate (a copy reads and writes its bytes).
A separate torch.profiler run (tracing slows the host) gives the kernels' own device time.  The summary line carries the
card's name and power limit, read in the same run.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import struct
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench_join_decimal import card   # noqa: E402  (tools/ is the script's directory)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--steps", type=int, default=3, help="timed calls per plan and round")
    args = ap.parse_args()

    import torch
    from tidb_b200 import abi
    from tidb_b200.device import dev_chunk
    from tidb_b200.plan import FilterItem, dec_const_array, filter_array
    from tidb_b200.q3 import price_cells

    if not torch.cuda.is_available():
        raise SystemExit("bench_vec_decimal.py needs a CUDA device")
    lib = abi.load_lib()
    dev = torch.device("cuda")
    n = args.rows
    g = torch.Generator(device=dev).manual_seed(6)
    ship = torch.randint(8000, 10600, (n,), device=dev, dtype=torch.int64, generator=g)
    disc = torch.randint(0, 11, (n,), device=dev, dtype=torch.int64, generator=g)          # 0.00 .. 0.10, * 100
    qty = torch.randint(100, 5001, (n,), device=dev, dtype=torch.int64, generator=g)       # 1.00 .. 50.00, * 100
    disc_c, qty_c = price_cells(disc), price_cells(qty)
    disc_f, qty_f = disc.to(torch.float64) / 100, qty.to(torch.float64) / 100
    want = int(((ship >= 8766) & (ship < 9131) & (disc >= 5) & (disc <= 7) & (qty < 2400)).sum())
    want_lt = int((qty < 2400).sum())
    del disc, qty
    copy_dst = torch.empty_like(qty_c)
    res = torch.empty(n, dtype=torch.int64, device=dev)
    res_nulls = torch.empty((n + 7) // 8 + 16, dtype=torch.uint8, device=dev)
    selected = torch.empty(n, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize()
    stream = torch.cuda.current_stream()
    st = C.c_void_p(stream.cuda_stream)

    def cell(text: str) -> bytes:
        """a non-negative literal with at most 2 fraction digits -> its cell: one integer word, one fraction word"""
        ip, _, fp = text.partition(".")
        return struct.pack("<bbbB9i", 9, 2, 2, 0, int(ip), int(fp.ljust(2, "0")) * 10 ** 7, *([0] * 7))

    ship_items = [FilterItem(abi.CMP_GE, 0, const_i64=8766), FilterItem(abi.CMP_LT, 0, const_i64=9131)]
    dec_items = ship_items + [FilterItem(abi.CMP_GE, 1, is_decimal=True, const_cell=cell("0.05")),
                              FilterItem(abi.CMP_LE, 1, is_decimal=True, const_cell=cell("0.07")),
                              FilterItem(abi.CMP_LT, 2, is_decimal=True, const_cell=cell("24"))]
    dbl_items = ship_items + [FilterItem(abi.CMP_GE, 1, is_real=True, const_f64=0.05), FilterItem(abi.CMP_LE, 1, is_real=True, const_f64=0.07),
                              FilterItem(abi.CMP_LT, 2, is_real=True, const_f64=24.0)]
    dec_chk, dbl_chk = dev_chunk([ship, disc_c, qty_c]), dev_chunk([ship, disc_f, qty_f])
    types = (C.c_int32 * 3)(abi.TYPE_LONGLONG, abi.TYPE_NEWDECIMAL, abi.TYPE_NEWDECIMAL)
    dec_arr, dec_consts, dbl_arr = filter_array(dec_items), dec_const_array(dec_items), filter_array(dbl_items)
    qcol, dcol = dec_chk.cols[2], dec_chk.cols[1]
    k24 = (C.c_uint8 * 40).from_buffer_copy(cell("24"))
    cnt = C.c_int64(0)
    rp, np_, sp = C.c_void_p(res.data_ptr()), C.c_void_p(res_nulls.data_ptr()), C.c_void_p(selected.data_ptr())

    def filter_dec():
        abi.check(lib.tg_vec_filter_ex(0, 1, C.byref(dec_chk), types, dec_arr, len(dec_items), dec_consts, sp, C.byref(cnt), st))
        return cnt.value == want

    def filter_dbl():
        abi.check(lib.tg_vec_filter(0, 1, C.byref(dbl_chk), dbl_arr, len(dbl_items), sp, C.byref(cnt), st))
        return cnt.value == want

    def cmp_const():
        abi.check(lib.tg_vec_compare_decimal(0, 1, abi.CMP_LT, C.byref(qcol), None, k24, rp, np_, st))
        return True

    def cmp_col():
        abi.check(lib.tg_vec_compare_decimal(0, 1, abi.CMP_LT, C.byref(dcol), C.byref(qcol), None, rp, np_, st))
        return True

    def copy():
        copy_dst.copy_(qty_c)
        return True

    # bytes a call must move per row, from the shapes: reads, then writes (1 byte of `selected`; 8 bytes + a bit of result)
    plans = {"filter_dec": (filter_dec, 8 + 40 + 40 + 1), "filter_dbl": (filter_dbl, 8 + 8 + 8 + 1),
             "cmp_const": (cmp_const, 40 + 8 + 1 / 8), "cmp_col": (cmp_col, 40 + 40 + 8 + 1 / 8), "copy": (copy, 40 + 40)}

    def step(fn) -> float:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(stream)
        ok = fn()
        e1.record(stream)
        torch.cuda.synchronize()
        assert ok, "wrong row count"
        return e0.elapsed_time(e1)

    for _ in range(args.warmup):
        for fn, _b in plans.values():
            step(fn)
    cmp_const()
    torch.cuda.synchronize()
    assert int(res.sum()) == want_lt, "l_quantity < 24 selected the wrong rows"

    times = {name: [] for name in plans}
    for r in range(args.rounds):
        names = list(plans) if r % 2 == 0 else list(reversed(plans))   # ABBA order across rounds
        row = {"round": r}
        for name in names:
            ts = [step(plans[name][0]) for _ in range(args.steps)]
            times[name].extend(ts)
            row[name + "_ms"] = [round(t, 3) for t in ts]
        print(json.dumps(row), flush=True)

    from torch.profiler import ProfilerActivity, profile as tprofile
    kernel_ms = {}
    for name, kernel in (("filter_dec", "k_vec_filter_dec"), ("filter_dbl", "k_vec_filter"), ("cmp_const", "k_vec_compare_dec"),
                         ("cmp_col", "k_vec_compare_dec")):
        with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                plans[name][0]()
            torch.cuda.synchronize()
        us = sum(e.device_time_total for e in prof.key_averages() if e.key.split("(")[0].split("<")[0].endswith(kernel)) / args.steps
        kernel_ms[name] = round(us / 1000, 3)

    med = {name: statistics.median(ts) for name, ts in times.items()}
    gbps = {name: plans[name][1] * n / (med[name] * 1e-3) / 1e9 for name in plans}
    summary = {"workload": "Q6 predicate / DECIMAL compares, device-resident DECIMAL(15,2) cells", "rows": n,
               "bytes_per_row": {k: round(v[1], 3) for k, v in plans.items()},
               "median_ms": {k: round(v, 3) for k, v in med.items()},
               "min_ms": {k: round(min(v), 3) for k, v in times.items()},
               "GBps": {k: round(v, 1) for k, v in gbps.items()},
               "of_copy": {k: round(v / gbps["copy"], 3) for k, v in gbps.items()},
               "kernel_ms": kernel_ms,
               "kernel_GBps": {k: round(plans[k][1] * n / (v * 1e-3) / 1e9, 1) if v else None for k, v in kernel_ms.items()}}
    summary.update(card())
    print(json.dumps(summary), flush=True)


if __name__ == "__main__":
    main()
