"""Step time of DECIMAL SUM(bigint) against SUM(double), each with COUNT, GROUP BY int64, on one GPU.

    python tools/bench_agg_decimal.py [--rows 100000000] [--groups 1000000 62500] [--steps 10] [--rounds 3]

A step is one whole aggregation of device-resident columns (table init + update + finalize), as in bench.py --workload
agg.  The two plans alternate within each round, in one process over the same keys, so both see the same clocks and the
same neighbours on a shared machine.  Values are below 2^31 (bigint) and their DOUBLE copies.  The DECIMAL table holds one
more 8-byte word per slot (the high word of the 128-bit sum), and each row adds the low-word atomic plus a high-word atomic
only on a carry or a negative value.  Prints the card's name and power limit with the numbers, one JSON line per
measurement and a summary line.
"""
from __future__ import annotations

import argparse
import json
import os
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
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--groups", type=int, nargs="+", default=[1_000_000, 62_500])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import torch
    from tidb_b200 import abi
    from tidb_b200.device import DeviceAgg
    from tidb_b200.plan import AggFunc, AggPlan, FieldType

    if not torch.cuda.is_available():
        raise SystemExit("bench_agg_decimal needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    info = card()
    print(json.dumps(info), flush=True)
    stream = torch.cuda.Stream(device=dev)
    INT = FieldType(abi.TYPE_LONGLONG, abi.FLAG_NOT_NULL)
    DBL = FieldType(abi.TYPE_DOUBLE, abi.FLAG_NOT_NULL)
    n = args.rows
    summary = []
    for G in args.groups:
        with torch.cuda.stream(stream):
            g = torch.Generator(device=dev); g.manual_seed(45)
            keys = torch.randint(0, G, (n,), device=dev, generator=g, dtype=torch.int64)
            xi = torch.randint(0, 1 << 31, (n,), device=dev, generator=g, dtype=torch.int64)
            xd = xi.to(torch.float64)
        stream.synchronize()
        plans = {
            "sum_double": (AggPlan([INT, DBL], [0], [AggFunc(abi.AGG_FIRSTROW, 0), AggFunc(abi.AGG_SUM, 1, abi.TYPE_DOUBLE),
                                                      AggFunc(abi.AGG_COUNT, 1, abi.TYPE_DOUBLE)], stream=stream.cuda_stream,
                                   expected_groups=G), xd),
            "sum_decimal": (AggPlan([INT, INT], [0], [AggFunc(abi.AGG_FIRSTROW, 0),
                                                       AggFunc(abi.AGG_SUM, 1, abi.TYPE_LONGLONG, ret_type=abi.TYPE_NEWDECIMAL),
                                                       AggFunc(abi.AGG_COUNT, 1, abi.TYPE_LONGLONG)], stream=stream.cuda_stream,
                                    expected_groups=G), xi),
        }

        def one(plan, x):
            agg = DeviceAgg(plan)
            with torch.cuda.stream(stream):
                agg.push([keys, x])
                rows, _, _ = agg.finish()
            assert rows == G
            agg.close()

        def timed(plan, x):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with torch.cuda.stream(stream):
                e0.record(stream)
            for _ in range(args.steps):
                one(plan, x)
            with torch.cuda.stream(stream):
                e1.record(stream)
            stream.synchronize()
            return e0.elapsed_time(e1) / args.steps

        for name, (plan, x) in plans.items():
            for _ in range(args.warmup):
                one(plan, x)
        res = {k: [] for k in plans}
        for r in range(args.rounds):
            order = list(plans) if r % 2 == 0 else list(plans)[::-1]
            for name in order:
                ms = timed(*plans[name])
                res[name].append(ms)
                print(json.dumps({"rows": n, "groups": G, "plan": name, "round": r, "step_ms": round(ms, 3), **info}), flush=True)
        summary.append({"rows": n, "groups": G, **{f"{k}_ms": [round(v, 3) for v in vs] for k, vs in res.items()}, **info})
        del keys, xi, xd
        torch.cuda.empty_cache()
    print(json.dumps({"summary": summary}), flush=True)


if __name__ == "__main__":
    main()
