"""TopN over a DECIMAL ORDER BY column against the same plan over DOUBLE, on one GPU.

    python tools/bench_topn_decimal.py [--rows 100000000] [--rounds 5] [--warmup 2] [--steps 3]

Workload: device-resident tg_topn over `rows` rows, ORDER BY a DECIMAL(15,2) column DESC LIMIT 10, with one DECIMAL(15,2)
payload column and two 8-byte payload columns (BIGINT, DATETIME).  The DOUBLE plan holds the same values as DOUBLE in
both price columns.  The cells are in MyDecimal.FromBin's form (two integer words, one fraction word) with up to 15
significant digits, so every value has its own rank and the candidates are the 10 rows.  A step is one tg_topn call
(rank pass, 8 histogram passes, collect, gather, host sort), timed with CUDA events; the two plans alternate within each
round, in one process, so both see the same clocks and neighbours on a shared machine.  A separate torch.profiler run
(tracing slows the host) gives the device time of k_topn_rank_dec and its bandwidth at 48 B per row (a 40-byte cell read,
an 8-byte rank written) against the H100 SXM data-sheet 3.35 TB/s.  Prints one JSON line per round and a summary line
with the card's name and power limit.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench_join_decimal import card   # noqa: E402  (tools/ is the script's directory)

HBM_TBPS = 3.35   # H100 SXM data sheet


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--steps", type=int, default=3, help="timed calls per plan and round")
    ap.add_argument("--limit", type=int, default=10)
    args = ap.parse_args()

    import numpy as np
    import torch
    from tidb_b200 import abi
    from tidb_b200.chunk import DECIMAL_DTYPE, MutChunk
    from tidb_b200.device import dev_chunk
    from tidb_b200.q3 import price_cells

    if not torch.cuda.is_available():
        raise SystemExit("bench_topn_decimal.py needs a CUDA device")
    lib = abi.load_lib()
    dev = torch.device("cuda")
    n, k = args.rows, args.limit
    g = torch.Generator(device=dev).manual_seed(9)
    price = torch.randint(0, 10**15, (n,), device=dev, dtype=torch.int64, generator=g)   # DECIMAL(15,2) * 100
    other = torch.randint(0, 10**15, (n,), device=dev, dtype=torch.int64, generator=g)
    ints = torch.randint(-(1 << 62), 1 << 62, (n,), device=dev, dtype=torch.int64, generator=g)
    times8 = torch.randint(0, 1 << 62, (n,), device=dev, dtype=torch.int64, generator=g)
    plans = {
        "decimal": ([price_cells(price), price_cells(other), ints, times8], abi.TYPE_NEWDECIMAL, 40, DECIMAL_DTYPE),
        "double": ([price.to(torch.float64) / 100, other.to(torch.float64) / 100, ints, times8], abi.TYPE_DOUBLE, 8, np.float64),
    }
    del other
    torch.cuda.synchronize()
    stream = torch.cuda.current_stream()
    items = (abi.TgSortItem * 1)(abi.TgSortItem(0, 1))
    fls = (C.c_uint32 * 4)(0, 0, 0, 0)
    calls = {}
    for name, (cols, tp, el, dt) in plans.items():
        ck = dev_chunk(cols)
        tps = (C.c_int32 * 4)(tp, tp, abi.TYPE_LONGLONG, abi.TYPE_DATETIME)
        out = MutChunk([el, el, 8, 8], k, [dt, dt, np.int64, np.int64])
        calls[name] = (ck, tps, out)

    def call(name) -> int:
        ck, tps, out = calls[name]
        nr = C.c_int64(0)
        abi.check(lib.tg_topn(0, 1, C.byref(ck), tps, fls, items, 1, C.c_int64(0), C.c_int64(k), C.byref(out.struct), C.byref(nr),
                              C.c_void_p(stream.cuda_stream)))
        return nr.value

    def step(name) -> float:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(stream)
        assert call(name) == k
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    for _ in range(args.warmup):
        for name in calls:
            step(name)
    # both plans return the same rows: the same prices, and the same BIGINT payloads
    want = torch.topk(price, k).values.cpu().numpy()
    dcells = calls["decimal"][2].columns(k)[0][0]
    got_dec = dcells.view(np.int32).reshape(k, 10).astype(np.int64)
    got_dec = (got_dec[:, 1] * 10**9 + got_dec[:, 2]) * 100 + got_dec[:, 3] // 10**7
    got_dbl = np.round(calls["double"][2].columns(k)[0][0] * 100).astype(np.int64)
    same = bool(np.array_equal(got_dec, want) and np.array_equal(got_dbl, want)
                and np.array_equal(calls["decimal"][2].columns(k)[2][0], calls["double"][2].columns(k)[2][0]))

    times = {name: [] for name in calls}
    for r in range(args.rounds):
        names = list(calls) if r % 2 == 0 else list(reversed(calls))   # ABBA order across rounds
        row = {"round": r}
        for name in names:
            ts = [step(name) for _ in range(args.steps)]
            times[name].extend(ts)
            row[name + "_ms"] = [round(t, 3) for t in ts]
        print(json.dumps(row), flush=True)

    from torch.profiler import ProfilerActivity, profile as tprofile
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            call("decimal")
        torch.cuda.synchronize()
    rank_us = sum(e.device_time_total for e in prof.key_averages() if "k_topn_rank_dec" in e.key) / args.steps
    med = {name: statistics.median(ts) for name, ts in times.items()}
    summary = {"workload": "tg_topn device-resident, ORDER BY DECIMAL(15,2) DESC LIMIT %d, payload DECIMAL + 2 x 8-byte" % k,
               "rows": n, "same_rows": same,
               "median_ms": {kk: round(v, 3) for kk, v in med.items()},
               "min_ms": {kk: round(min(v), 3) for kk, v in times.items()},
               "decimal_over_double": round(med["decimal"] / med["double"], 3),
               "k_topn_rank_dec_ms": round(rank_us / 1000, 3),
               "k_topn_rank_dec_TBps_at_48B_per_row": round(48 * n / (rank_us * 1e-6) / 1e12, 3) if rank_us else None,
               "share_of_3.35_TBps": round(48 * n / (rank_us * 1e-6) / 1e12 / HBM_TBPS, 3) if rank_us else None}
    summary.update(card())
    print(json.dumps(summary), flush=True)


if __name__ == "__main__":
    main()
