"""The string VecEval calls against a plain device copy of the same bytes, on one GPU.

    python tools/bench_vec_string.py [--rows 100000000] [--rounds 5] [--warmup 2] [--steps 3]

Workload, all device-resident (`rows` rows, seeded), TPC-H-like string columns:
  seg_eq       tg_vec_filter_ex2: c_mktsegment = 'BUILDING' under utf8mb4_bin over a 10-byte column (segment names padded
               with spaces to 10 bytes, which utf8mb4_bin ignores)
  seg_eq_col   tg_vec_compare_string: the same comparison as an int64 result column with its NULL bitmap
  type_like    tg_vec_filter_ex2: p_type LIKE 'PROMO%' over a 25-byte column
  comment_nlike  tg_vec_filter_ex2: o_comment NOT LIKE '%special%requests%' over comments of 20..80 bytes (about 50)
  cmp_col      tg_vec_compare_string: comment < comment2, a second comment column generated independently (its own
               vocabulary, offsets and bytes), so both operands come from DRAM
  copy         a device-to-device copy of the comment column's offsets and bytes (cudaMemcpyAsync), the ceiling
Each step is one call timed with CUDA events; the plans alternate within each round in one process, so all see the same
clocks and neighbours on a shared machine.  Bytes per row come from the shapes: offsets (8), the row's bytes, and what is
written (1 byte of `selected`, or 8 bytes and a bit of result).  GB/s is those bytes over the median call time, and
`of_copy` its ratio to the copy's rate.  A separate torch.profiler run (tracing slows the host) gives the kernels' own
device time (`kernel_ms`), which leaves out the host-side argument checks, the pattern upload and the flag read-back of
each call.  The summary line carries the card's name and power limit, read in the same run.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench_join_decimal import card   # noqa: E402  (tools/ is the script's directory)

SEGMENTS = [b"AUTOMOBILE", b"BUILDING", b"FURNITURE", b"HOUSEHOLD", b"MACHINERY"]
T1 = [b"STANDARD", b"SMALL", b"MEDIUM", b"LARGE", b"ECONOMY", b"PROMO"]
T2 = [b"ANODIZED", b"BURNISHED", b"PLATED", b"POLISHED", b"BRUSHED"]
T3 = [b"TIN", b"NICKEL", b"BRASS", b"STEEL", b"COPPER"]
WORDS = [b"carefully", b"final", b"deposits", b"detect", b"slyly", b"pending", b"packages", b"ironic", b"foxes", b"regular",
         b"accounts", b"haggle", b"quickly", b"blithely", b"express", b"theodolites", b"furiously", b"bold", b"requests",
         b"special"]


def fixed_width(names, width):
    return np.frombuffer(b"".join(s.ljust(width) for s in names), np.uint8).reshape(len(names), width)


def comment_vocab(rng, k=4096):
    out = []
    while len(out) < k:
        s = b" ".join(WORDS[j] for j in rng.integers(0, len(WORDS) - 2, 12))[: int(rng.integers(20, 81))]
        if rng.random() < 0.02:
            s = (s[:20] + b" special " + s[20:40] + b" requests")[:80]
        out.append(s)
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--steps", type=int, default=3, help="timed calls per plan and round")
    args = ap.parse_args()

    import torch
    from tidb_b200 import abi
    from tidb_b200.plan import FilterItem, filter_array, str_arg_array

    if not torch.cuda.is_available():
        raise SystemExit("bench_vec_string.py needs a CUDA device")
    lib = abi.load_lib()
    dev = torch.device("cuda")
    n = args.rows
    g = torch.Generator(device=dev).manual_seed(7)

    # fixed-width columns: one table row per value, gathered by a random id
    seg_tab = torch.from_numpy(fixed_width(SEGMENTS, 10)).to(dev)
    types = [a + b" " + b + b" " + c for a in T1 for b in T2 for c in T3]
    type_tab = torch.from_numpy(fixed_width(types, 25)).to(dev)
    seg_id = torch.randint(0, len(SEGMENTS), (n,), device=dev, generator=g)
    type_id = torch.randint(0, len(types), (n,), device=dev, generator=g)
    seg_data, type_data = seg_tab[seg_id].reshape(-1), type_tab[type_id].reshape(-1)
    seg_offs = torch.arange(0, n + 1, device=dev, dtype=torch.int64) * 10
    type_offs = torch.arange(0, n + 1, device=dev, dtype=torch.int64) * 25
    want_seg = int((seg_id == 1).sum())
    want_type = int(torch.tensor([t.startswith(b"PROMO") for t in types], device=dev)[type_id].sum())
    del seg_id, type_id

    # comments: two independent columns of n rows, each from its own 4096-entry vocabulary, built in batches
    def comments(seed):
        vocab = comment_vocab(np.random.default_rng(seed))
        vlen = torch.tensor([len(s) for s in vocab], device=dev, dtype=torch.int64)
        vstart = torch.zeros(len(vocab), device=dev, dtype=torch.int64)
        vstart[1:] = torch.cumsum(vlen, 0)[:-1]
        vblob = torch.from_numpy(np.frombuffer(b"".join(vocab), np.uint8).copy()).to(dev)
        vspecial = torch.tensor([(s.find(b"special") >= 0 and s.find(b"requests", s.find(b"special") + 7) >= 0) for s in vocab], device=dev)
        ids = torch.randint(0, len(vocab), (n,), device=dev, generator=g)
        offs = torch.zeros(n + 1, device=dev, dtype=torch.int64)
        offs[1:] = torch.cumsum(vlen[ids], 0)
        data = torch.empty(int(offs[-1]), device=dev, dtype=torch.uint8)
        batch = 1 << 22
        for lo in range(0, n, batch):
            b_ids = ids[lo:lo + batch]
            lens = vlen[b_ids]
            rel = torch.arange(int(lens.sum()), device=dev, dtype=torch.int64)
            first = torch.repeat_interleave(offs[lo:lo + len(b_ids)] - offs[lo], lens)
            src = torch.repeat_interleave(vstart[b_ids], lens) + rel - first
            data[int(offs[lo]):int(offs[lo]) + len(rel)] = vblob[src]
        return offs, data, n - int(vspecial[ids].sum())

    com_offs, com_data, want_com = comments(7)
    com2_offs, com2_data, _ = comments(8)
    avg_com = float(com_offs[n]) / n
    avg_com2 = float(com2_offs[n]) / n

    def column(data, offs, length):
        c = abi.TgColumn()
        c.length, c.null_bitmap, c.offsets, c.data, c.elem_len = length, None, offs.data_ptr(), data.data_ptr(), -1
        return c

    seg_c, type_c = column(seg_data, seg_offs, n), column(type_data, type_offs, n)
    com_a, com_b = column(com_data, com_offs, n), column(com2_data, com2_offs, n)

    def chunk(col):
        arr = (abi.TgColumn * 1)(col)
        ch = abi.TgChunk(); ch.ncols, ch.cols, ch.sel, ch.nsel = 1, C.cast(arr, C.POINTER(abi.TgColumn)), None, 0
        ch._keep = arr
        return ch

    seg_chk, type_chk, com_chk = chunk(seg_c), chunk(type_c), chunk(com_a)
    vc = (C.c_int32 * 1)(abi.TYPE_VARCHAR)
    items = {"seg": [FilterItem(abi.CMP_EQ, 0, is_string=True, const_bytes=b"BUILDING", collation=abi.COLLATION_UTF8MB4_BIN)],
             "type": [FilterItem(abi.CMP_EQ, 0, is_string=True, str_kind=abi.STR_LIKE, const_bytes=b"PROMO%")],
             "com": [FilterItem(abi.CMP_EQ, 0, is_string=True, str_kind=abi.STR_NOT_LIKE, const_bytes=b"%special%requests%")]}
    rendered = {k: (filter_array(v), str_arg_array(v)) for k, v in items.items()}
    copy_dst = torch.empty(com_data.numel() + com_offs.numel() * 8, device=dev, dtype=torch.uint8)
    res = torch.empty(n, dtype=torch.int64, device=dev)
    res_nulls = torch.empty((n + 7) // 8 + 16, dtype=torch.uint8, device=dev)
    selected = torch.empty(n, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize()
    stream = torch.cuda.current_stream()
    st = C.c_void_p(stream.cuda_stream)
    cnt = C.c_int64(0)
    rp, np_, sp = C.c_void_p(res.data_ptr()), C.c_void_p(res_nulls.data_ptr()), C.c_void_p(selected.data_ptr())
    kb = (C.c_uint8 * 8).from_buffer_copy(b"BUILDING")

    def filt(key, chk, want):
        def run():
            arr, sa = rendered[key]
            abi.check(lib.tg_vec_filter_ex2(0, 1, C.byref(chk), vc, arr, 1, None, sa, sp, C.byref(cnt), st))
            return cnt.value == want
        return run

    def seg_eq_col():
        abi.check(lib.tg_vec_compare_string(0, 1, abi.CMP_EQ, abi.COLLATION_UTF8MB4_BIN, C.byref(seg_c), None, kb, C.c_int64(8), rp, np_, st))
        return True

    def cmp_col():
        abi.check(lib.tg_vec_compare_string(0, 1, abi.CMP_LT, abi.COLLATION_UTF8MB4_BIN, C.byref(com_a), C.byref(com_b), None, C.c_int64(0), rp, np_, st))
        return True

    def copy():
        copy_dst[:com_data.numel()].copy_(com_data)
        copy_dst[com_data.numel():].copy_(com_offs.view(torch.uint8))
        return True

    plans = {"seg_eq": (filt("seg", seg_chk, want_seg), 8 + 10 + 1), "seg_eq_col": (seg_eq_col, 8 + 10 + 8 + 1 / 8),
             "type_like": (filt("type", type_chk, want_type), 8 + 25 + 1),
             "comment_nlike": (filt("com", com_chk, want_com), 8 + avg_com + 1),
             "cmp_col": (cmp_col, 8 + avg_com + 8 + avg_com2 + 8 + 1 / 8), "copy": (copy, 2 * (8 + avg_com))}

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
    seg_eq_col()
    torch.cuda.synchronize()
    assert int(res.sum()) == want_seg, "c_mktsegment = 'BUILDING' selected the wrong rows"

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
    for name in plans:
        if name == "copy":
            continue
        with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                plans[name][0]()
            torch.cuda.synchronize()
        us = sum(e.device_time_total for e in prof.key_averages() if "k_vec_string" in e.key) / args.steps
        kernel_ms[name] = round(us / 1000, 3)

    med = {name: statistics.median(ts) for name, ts in times.items()}
    gbps = {name: plans[name][1] * n / (med[name] * 1e-3) / 1e9 for name in plans}
    summary = {"workload": "string Selection / VecEval over device-resident TPC-H-like columns", "rows": n,
               "avg_comment_bytes": [round(avg_com, 2), round(avg_com2, 2)],
               "bytes_per_row": {k: round(v[1], 3) for k, v in plans.items()},
               "median_ms": {k: round(v, 3) for k, v in med.items()},
               "min_ms": {k: round(min(v), 3) for k, v in times.items()},
               "GBps": {k: round(v, 1) for k, v in gbps.items()},
               "of_copy": {k: round(v / gbps["copy"], 3) for k, v in gbps.items()},
               "kernel_ms": kernel_ms,
               "kernel_of_copy": {k: round(plans[k][1] * n / (v * 1e-3) / 1e9 / gbps["copy"], 3) if v else None
                                  for k, v in kernel_ms.items()}}
    summary.update(card())
    print(json.dumps(summary), flush=True)


if __name__ == "__main__":
    main()
