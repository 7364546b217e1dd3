"""Step time of DECIMAL SUM(bigint) and SUM(DECIMAL(15,2)) against SUM(double), each with COUNT, GROUP BY int64, on one GPU.

    python tools/bench_agg_decimal.py [--rows 100000000] [--groups 1000000 62500] [--steps 10] [--rounds 3]
    python tools/bench_agg_decimal.py --profile [--out DIR]    # kernel times of the DECIMAL(15,2) plan (torch.profiler)

A step is one whole aggregation of device-resident columns (table init + update + finalize), as in bench.py --workload
agg.  The two plans alternate within each round, in one process over the same keys, so both see the same clocks and the
same neighbours on a shared machine.  Values are below 2^31 (bigint) and their DOUBLE copies.  The DECIMAL table holds one
more 8-byte word per slot (the high word of the 128-bit sum), and each row adds the low-word atomic plus a high-word atomic
only on a carry or a negative value.  The DECIMAL(15,2) plan reads 40-byte MyDecimal cells in FromBin's form (two
integer words, one fraction word), built on the device from the same values / 100; k_dec_to_scaled turns them into
int64 cents once per push (40 B read + 8 B written per row), then the update is the DECIMAL SUM(bigint) one.  Prints the
card's name and power limit with the numbers, one JSON line per measurement and a summary line.  --profile runs the
DECIMAL(15,2) plan under torch.profiler instead (a separate run: tracing slows the host) and prints the device time of
every kernel per step.
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
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None, help="--profile: also write the kernel table here")
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
            xc = dec_cells(torch, xi)
        stream.synchronize()
        plans = {
            "sum_double": (AggPlan([INT, DBL], [0], [AggFunc(abi.AGG_FIRSTROW, 0), AggFunc(abi.AGG_SUM, 1, abi.TYPE_DOUBLE),
                                                      AggFunc(abi.AGG_COUNT, 1, abi.TYPE_DOUBLE)], stream=stream.cuda_stream,
                                   expected_groups=G), xd),
            "sum_decimal": (AggPlan([INT, INT], [0], [AggFunc(abi.AGG_FIRSTROW, 0),
                                                       AggFunc(abi.AGG_SUM, 1, abi.TYPE_LONGLONG, ret_type=abi.TYPE_NEWDECIMAL),
                                                       AggFunc(abi.AGG_COUNT, 1, abi.TYPE_LONGLONG)], stream=stream.cuda_stream,
                                    expected_groups=G), xi),
            "sum_decimal_15_2": (AggPlan([INT, FieldType(abi.TYPE_NEWDECIMAL, abi.FLAG_NOT_NULL, 15, 2)], [0],
                                         [AggFunc(abi.AGG_FIRSTROW, 0),
                                          AggFunc(abi.AGG_SUM, 1, abi.TYPE_NEWDECIMAL, ret_type=abi.TYPE_NEWDECIMAL, ret_frac=2),
                                          AggFunc(abi.AGG_COUNT, 1, abi.TYPE_NEWDECIMAL)], stream=stream.cuda_stream,
                                         expected_groups=G), xc),
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

        if args.profile:
            profile(torch, args, G, lambda: one(*plans["sum_decimal_15_2"]), stream, info)
            del keys, xi, xd, xc
            torch.cuda.empty_cache()
            continue
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
        del keys, xi, xd, xc
        torch.cuda.empty_cache()
    if not args.profile:
        print(json.dumps({"summary": summary}), flush=True)


def dec_cells(torch, x):
    """(n, 40) uint8 MyDecimal cells of DECIMAL(15,2) for the non-negative int64 cents x, as FromBin stores them:
    digitsInt 13 (two integer words), digitsFrac 2, one left-aligned fraction word"""
    n = x.numel()
    w = torch.zeros((n, 10), dtype=torch.int32, device=x.device)
    w[:, 0] = 13 | (2 << 8) | (2 << 16)
    ip = x // 100
    w[:, 1] = (ip // 10 ** 9).to(torch.int32)
    w[:, 2] = (ip % 10 ** 9).to(torch.int32)
    w[:, 3] = ((x % 100) * 10 ** 7).to(torch.int32)
    return w.view(torch.uint8).view(n, 40)


def profile(torch, args, G, step, stream, info) -> None:
    """device time per kernel and step of the DECIMAL(15,2) plan, from torch.profiler's CUDA activities"""
    from torch.profiler import ProfilerActivity, profile as tprofile
    for _ in range(args.warmup):
        step()
    stream.synchronize()
    with tprofile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            step()
        stream.synchronize()
    per = {}
    for ev in prof.key_averages():
        dt = getattr(ev, "device_time_total", None)
        if dt is None:
            dt = getattr(ev, "cuda_time_total", 0)
        if dt and ev.key.startswith(("_ZN2tg", "void tg::", "tg::")):
            per[ev.key] = (round(dt / 1e3 / args.steps, 4), ev.count // args.steps)
    for k, (ms, cnt) in sorted(per.items(), key=lambda kv: -kv[1][0]):
        print(json.dumps({"rows": args.rows, "groups": G, "plan": "sum_decimal_15_2", "kernel": k, "ms_per_step": ms,
                          "launches_per_step": cnt, **info}), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, f"kernels_{G}.txt"), "w") as fh:
            fh.write(prof.key_averages().table(sort_by="self_cuda_time_total", row_limit=30))


if __name__ == "__main__":
    main()
