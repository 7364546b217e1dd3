"""Probe time of the Q3 J2 join shape with DECIMAL payload columns against the same plan with DOUBLE columns, on one GPU.

    python tools/bench_join_decimal.py [--probe-rows 100000000] [--build-rows 10000000] [--rounds 5] [--warmup 2]

The shape is J2 of Q3, device-resident: probe (l_orderkey, l_extendedprice, l_discount) against unique build keys carrying
one payload column (o_totalprice), every probe row matching; output = probe key, both probe payload columns and the build
payload.  The DECIMAL plan carries 40-byte MyDecimal cells, the DOUBLE plan 8-byte values; both probe the same keys.  The
two plans alternate within each round, in one process, so both see the same clocks and neighbours on a shared machine.
A step is one tg_join_probe_dev call (build excluded), timed with CUDA events.  The DECIMAL plan's kernels move row ids
and k_gather_cells turns them into cells, so its extra cost per output row and DECIMAL column is the id traffic (about
24 B) plus the 40 B cell read and 40 B cell write any design pays.  A separate torch.profiler run (tracing slows the host)
gives the device time of k_gather_cells per step.  Prints one JSON line per round and a summary line with the card's name
and power limit.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as e:   # the numbers still stand; say that the card could not be read
        return {"gpu": "unknown", "power_limit": f"unknown ({e})"}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--probe-rows", type=int, default=100_000_000)
    ap.add_argument("--build-rows", type=int, default=10_000_000)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--steps", type=int, default=3, help="timed probes per plan and round")
    args = ap.parse_args()

    import torch
    from tidb_b200 import abi
    from tidb_b200.device import DeviceJoin
    from tidb_b200.plan import FieldType, JoinPlan

    if not torch.cuda.is_available():
        raise SystemExit("bench_join_decimal.py needs a CUDA device")
    dev = torch.device("cuda")
    nb, npr = args.build_rows, args.probe_rows
    g = torch.Generator(device=dev).manual_seed(7)
    bkey = torch.randperm(nb, device=dev, generator=g).to(torch.int64) * 4 + 1
    pkey = bkey[torch.randint(0, nb, (npr,), device=dev, generator=g)]
    INT = FieldType(abi.TYPE_LONGLONG, abi.FLAG_NOT_NULL)
    DBL = FieldType(abi.TYPE_DOUBLE, abi.FLAG_NOT_NULL)
    DEC = FieldType(abi.TYPE_NEWDECIMAL, abi.FLAG_NOT_NULL, 15, 2)
    cols = {
        "double": ([pkey] + [torch.rand(npr, device=dev, dtype=torch.float64, generator=g) for _ in range(2)],
                   [bkey, torch.rand(nb, device=dev, dtype=torch.float64, generator=g)], DBL),
        "decimal": ([pkey] + [torch.randint(0, 256, (npr, 40), device=dev, dtype=torch.uint8, generator=g) for _ in range(2)],
                    [bkey, torch.randint(0, 256, (nb, 40), device=dev, dtype=torch.uint8, generator=g)], DEC),
    }
    torch.cuda.synchronize()
    joins = {}
    for name, (pc, bc, t) in cols.items():
        j = DeviceJoin(JoinPlan(abi.JOIN_INNER, [INT, t, t], [INT, t], [0], [0], lused=[0, 1, 2], rused=[1]))
        j.build(bc)
        joins[name] = j

    def step(name) -> float:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        n, _, _ = joins[name].probe(cols[name][0])
        e1.record()
        torch.cuda.synchronize()
        assert n == npr
        return e0.elapsed_time(e1)

    for _ in range(args.warmup):
        for name in joins:
            step(name)
    times = {name: [] for name in joins}
    for r in range(args.rounds):
        names = list(joins) if r % 2 == 0 else list(reversed(joins))   # ABBA order across rounds
        row = {"round": r}
        for name in names:
            ts = [step(name) for _ in range(args.steps)]
            times[name].extend(ts)
            row[name + "_ms"] = [round(t, 3) for t in ts]
        print(json.dumps(row), flush=True)
    paths = {name: hex(j.stats().paths) for name, j in joins.items()}

    from torch.profiler import ProfilerActivity, profile as tprofile
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            joins["decimal"].probe(cols["decimal"][0])
        torch.cuda.synchronize()
    gather_us = sum(e.device_time_total for e in prof.key_averages() if "k_gather_cells" in e.key)
    for j in joins.values():
        j.close()
    med = {name: statistics.median(ts) for name, ts in times.items()}
    summary = {"workload": "join J2 shape, device-resident", "probe_rows": npr, "build_rows": nb, "decimal_columns": 3,
               "median_ms": {k: round(v, 3) for k, v in med.items()},
               "min_ms": {k: round(min(v), 3) for k, v in times.items()},
               "decimal_over_double": round(med["decimal"] / med["double"], 3),
               "gather_ms_per_step": round(gather_us / 1000 / args.steps, 3), "paths": paths}
    summary.update(card())
    print(json.dumps(summary), flush=True)


if __name__ == "__main__":
    main()
