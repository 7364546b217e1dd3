"""Step time of COUNT(DISTINCT v) against COUNT(v), device-resident, on one GPU.

    python tools/bench_agg_distinct.py [--rows 100000000] [--steps 5] [--rounds 3]
    python tools/bench_agg_distinct.py --profile [--out DIR]    # kernel times of every DISTINCT shape (torch.profiler)

Shapes (all BIGINT NOT NULL columns):
    grouped_1m     COUNT(DISTINCT v) GROUP BY g, 1 M groups x about 8 values each (v uniform in 0..7)
    grouped_62k    COUNT(DISTINCT v) GROUP BY g, 62.5 K groups (v uniform in 0..127: about 128 values each)
    nogroup_10m    COUNT(DISTINCT v) without GROUP BY, 10 M distinct values
    nogroup_100m   COUNT(DISTINCT v) without GROUP BY, 100 M distinct values (v a permutation)
A step is one whole aggregation of the device-resident columns (open, one push, finish, close), as in bench.py --workload
agg.  Each shape alternates with the same plan without DISTINCT within every round, in one process over the same columns,
so both see the same clocks and neighbours on a shared machine.  Prints the card's name and power limit with the numbers,
one JSON line per measurement (step time, mark_ms = device time of the dedup pass, set bytes, rows/s) and a summary line.
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
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--shapes", nargs="+", default=["grouped_1m", "grouped_62k", "nogroup_10m", "nogroup_100m"])
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None, help="--profile: also write the kernel tables here")
    args = ap.parse_args()
    import torch
    from tidb_b200 import abi
    from tidb_b200.device import DeviceAgg
    from tidb_b200.plan import AggFunc, AggPlan, FieldType

    if not torch.cuda.is_available():
        raise SystemExit("bench_agg_distinct needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    info = card()
    print(json.dumps(info), flush=True)
    stream = torch.cuda.Stream(device=dev)
    INT = FieldType(abi.TYPE_LONGLONG, abi.FLAG_NOT_NULL)
    n = args.rows
    summary = []
    for shape in args.shapes:
        with torch.cuda.stream(stream):
            g = torch.Generator(device=dev); g.manual_seed(46)
            if shape.startswith("grouped"):
                G, V = (1_000_000, 8) if shape == "grouped_1m" else (62_500, 128)
                keys = torch.randint(0, G, (n,), device=dev, generator=g, dtype=torch.int64)
                vals = torch.randint(0, V, (n,), device=dev, generator=g, dtype=torch.int64)
                cols, group_by, fr = [keys, vals], [0], [AggFunc(abi.AGG_FIRSTROW, 0)]
            else:
                G = 1
                vals = (torch.randperm(n, device=dev, generator=g) if shape == "nogroup_100m"
                        else torch.randint(0, 10_000_000, (n,), device=dev, generator=g, dtype=torch.int64))
                cols, group_by, fr = [vals, vals], [], []
        stream.synchronize()
        plans = {d: AggPlan([INT, INT], group_by, fr + [AggFunc(abi.AGG_COUNT, 1, distinct=d)], stream=stream.cuda_stream,
                            expected_groups=G if group_by else 0) for d in (True, False)}
        last = {}

        def one(distinct):
            agg = DeviceAgg(plans[distinct])
            with torch.cuda.stream(stream):
                agg.push(cols)
                rows, _, _ = agg.finish()
            assert rows == G
            if distinct:
                last["ds"] = agg.distinct_stats()
            agg.close()

        def timed(distinct):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            mark = 0.0
            with torch.cuda.stream(stream):
                e0.record(stream)
            for _ in range(args.steps):
                one(distinct)
                if distinct:
                    mark += last["ds"].mark_ms
            with torch.cuda.stream(stream):
                e1.record(stream)
            stream.synchronize()
            return e0.elapsed_time(e1) / args.steps, mark / args.steps

        if args.profile:
            profile(torch, args, shape, lambda: one(True), stream, info)
        else:
            for d in (True, False):
                for _ in range(args.warmup):
                    one(d)
            res = {"distinct": [], "plain": [], "mark": []}
            for r in range(args.rounds):
                for d in ((True, False) if r % 2 == 0 else (False, True)):
                    ms, mark = timed(d)
                    res["distinct" if d else "plain"].append(ms)
                    rec = {"rows": n, "shape": shape, "plan": "count_distinct" if d else "count", "round": r, "step_ms": round(ms, 3),
                           "rows_per_s": round(n / (ms * 1e-3)), **info}
                    if d:
                        ds = last["ds"]
                        res["mark"].append(mark)
                        rec.update({"mark_ms": round(mark, 3), "pairs": ds.pairs, "set_slots": ds.set_slots, "set_grows": ds.set_grows,
                                    "set_bytes": ds.set_slots * (16 if not group_by else 32)})
                    print(json.dumps(rec), flush=True)
            summary.append({"rows": n, "shape": shape, **{f"{k}_ms": [round(v, 3) for v in vs] for k, vs in res.items()}, **info})
        del cols, vals
        if shape.startswith("grouped"):
            del keys
        torch.cuda.empty_cache()
    if not args.profile:
        print(json.dumps({"summary": summary}), flush=True)


def profile(torch, args, shape, step, stream, info) -> None:
    """device time per kernel and step of the COUNT(DISTINCT v) plan, from torch.profiler's CUDA activities"""
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
            per[ev.key] = (round(dt / 1e3 / args.steps, 4), ev.count / args.steps)
    for k, (ms, cnt) in sorted(per.items(), key=lambda kv: -kv[1][0]):
        print(json.dumps({"rows": args.rows, "shape": shape, "kernel": k, "ms_per_step": ms, "launches_per_step": cnt, **info}), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, f"kernels_{shape}.txt"), "w") as fh:
            fh.write(prof.key_averages().table(sort_by="self_cuda_time_total", row_limit=30))


if __name__ == "__main__":
    main()
