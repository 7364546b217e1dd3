"""Step time of SUM(price * (1 - disc)) over DECIMAL(15,2) against the same over DOUBLE, and of the Q3-shaped plans, on one GPU.

    python tools/bench_agg_decimal_expr.py [--rows 100000000] [--groups 1000000 62500] [--steps 10] [--rounds 3]
    python tools/bench_agg_decimal_expr.py --profile [--out DIR]   # kernel times per plan (torch.profiler)

A step is one whole aggregation of device-resident columns (table init + update + finalize), as in bench.py --workload
agg.  Plans, each over the same keys, prices (900.00 .. 105000.00) and discounts (0.00 .. 0.10):
  double      GROUP BY k: FIRSTROW(k), SUM(price * (1 - disc)) over DOUBLE columns (agg_arg_real), COUNT(*)
  decimal     the same over DECIMAL(15,2) cells: k_dec_to_scaled on both columns, then the exact 192-bit product sum
  q3_double   GROUP BY (k, date, prio), FIRSTROW x 3, SUM(price * (1 - disc)) over DOUBLE: the multi-key table
  q3_decimal  the same over DECIMAL(15,2)
The plans alternate within each round, in one process, so all see the same clocks and neighbours on a shared machine.
The DECIMAL cells are in FromBin's form (two integer words, one fraction word), built on the device.  Prints the card's
name and power limit with the numbers, one JSON line per measurement and a summary line.  --profile runs every plan under
torch.profiler instead (a separate run: tracing slows the host) and prints the device time of every kernel per step.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_agg_decimal import card, dec_cells   # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--groups", type=int, nargs="+", default=[1_000_000, 62_500])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None, help="--profile: also write the kernel tables here")
    args = ap.parse_args()
    import torch
    from tidb_b200 import abi
    from tidb_b200.device import DeviceAgg
    from tidb_b200.plan import AggFunc, AggPlan, FieldType

    if not torch.cuda.is_available():
        raise SystemExit("bench_agg_decimal_expr needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    info = card()
    print(json.dumps(info), flush=True)
    stream = torch.cuda.Stream(device=dev)
    INT = FieldType(abi.TYPE_LONGLONG, abi.FLAG_NOT_NULL)
    DBL = FieldType(abi.TYPE_DOUBLE, abi.FLAG_NOT_NULL)
    DEC = FieldType(abi.TYPE_NEWDECIMAL, abi.FLAG_NOT_NULL, 15, 2)
    n = args.rows
    summary = []

    def revenue(a, b, dec):
        if dec:
            return AggFunc(abi.AGG_SUM, a, abi.TYPE_NEWDECIMAL, ret_type=abi.TYPE_NEWDECIMAL, ret_frac=4, arg_col2=b,
                           arg_expr=abi.ARGEXPR_MUL_CSUB, arg_const=1.0)
        return AggFunc(abi.AGG_SUM, a, abi.TYPE_DOUBLE, arg_col2=b, arg_expr=abi.ARGEXPR_MUL_CSUB, arg_const=1.0)

    for G in args.groups:
        with torch.cuda.stream(stream):
            g = torch.Generator(device=dev); g.manual_seed(46)
            keys = torch.randint(0, G, (n,), device=dev, generator=g, dtype=torch.int64)
            date = keys * 7919 % 2400 + 8000
            prio = torch.zeros_like(keys)
            price = torch.randint(90_000, 10_500_000, (n,), device=dev, generator=g, dtype=torch.int64)
            disc = torch.randint(0, 11, (n,), device=dev, generator=g, dtype=torch.int64)
            pd, dd = price.to(torch.float64) / 100, disc.to(torch.float64) / 100
            pc, dc = dec_cells(torch, price), dec_cells(torch, disc)
            del price, disc
        stream.synchronize()
        s = stream.cuda_stream
        plans = {}
        for name, dec, (p, d), ty in (("double", False, (pd, dd), DBL), ("decimal", True, (pc, dc), DEC)):
            plans[name] = (AggPlan([INT, ty, ty], [0], [AggFunc(abi.AGG_FIRSTROW, 0), revenue(1, 2, dec), AggFunc(abi.AGG_COUNT, -1)],
                                   stream=s, expected_groups=G), [keys, p, d])
            plans["q3_" + name] = (AggPlan([INT, INT, INT, ty, ty], [0, 1, 2], [AggFunc(abi.AGG_FIRSTROW, c) for c in (0, 1, 2)] +
                                           [revenue(3, 4, dec)], stream=s, expected_groups=G), [keys, date, prio, p, d])
        plans = {k: plans[k] for k in ("double", "decimal", "q3_double", "q3_decimal")}

        def one(plan, cols):
            agg = DeviceAgg(plan)
            with torch.cuda.stream(stream):
                agg.push(cols)
                rows, _, _ = agg.finish()
            assert rows == G, (rows, G)
            agg.close()

        def timed(plan, cols):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with torch.cuda.stream(stream):
                e0.record(stream)
            for _ in range(args.steps):
                one(plan, cols)
            with torch.cuda.stream(stream):
                e1.record(stream)
            stream.synchronize()
            return e0.elapsed_time(e1) / args.steps

        if args.profile:
            for name, (plan, cols) in plans.items():
                profile(torch, args, G, name, lambda: one(plan, cols), stream, info)
        else:
            for plan, cols in plans.values():
                for _ in range(args.warmup):
                    one(plan, cols)
            res = {k: [] for k in plans}
            for r in range(args.rounds):
                for name in (list(plans) if r % 2 == 0 else list(plans)[::-1]):
                    ms = timed(*plans[name])
                    res[name].append(ms)
                    print(json.dumps({"rows": n, "groups": G, "plan": name, "round": r, "step_ms": round(ms, 3), **info}), flush=True)
            summary.append({"rows": n, "groups": G, **{f"{k}_ms": [round(v, 3) for v in vs] for k, vs in res.items()}, **info})
        del keys, date, prio, pd, dd, pc, dc, plans
        torch.cuda.empty_cache()
    if not args.profile:
        print(json.dumps({"summary": summary}), flush=True)


def profile(torch, args, G, name, step, stream, info) -> None:
    """device time per kernel and step of one plan, from torch.profiler's CUDA activities"""
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
        print(json.dumps({"rows": args.rows, "groups": G, "plan": name, "kernel": k, "ms_per_step": ms, "launches_per_step": cnt,
                          **info}), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, f"kernels_{name}_{G}.txt"), "w") as fh:
            fh.write(prof.key_averages().table(sort_by="self_cuda_time_total", row_limit=30))


if __name__ == "__main__":
    main()
