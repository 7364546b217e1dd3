"""Step time of GROUP BY over string columns against the same plan over pre-encoded BIGINT keys, device-resident, on
one GPU.

    python tools/bench_agg_string.py [--rows 100000000] [--steps 5] [--rounds 3] [--shapes q1 q16 highcard]
    python tools/bench_agg_string.py --profile          # kernel times (torch.profiler), k_str_dict_encode's share

Shapes:
    q1        two CHAR(1) keys (l_returnflag, l_linestatus: 4 groups), SUM and AVG of two DECIMAL(15, 2) columns, COUNT(*)
    q16       Brand#NN x 25-byte p_type x an int size (about 20 K groups), COUNT(DISTINCT ps_suppkey)
    highcard  10 M distinct 18-byte Customer#NNNNNNNNN keys, COUNT(*)
String keys are utf8mb4_bin (46), TiDB's default for CHAR and VARCHAR: with several GROUP BY columns their FIRSTROW
also runs the per-group tail MIN.  A step is one whole aggregation (open, one push, finish, close).  Each
string plan alternates with its BIGINT-key twin within every round, in one process over the same rows.  Prints the
card's name and power limit with the numbers, one JSON line per measurement (step time, encode_ms = device time of the
encode pass, dictionary entries and bytes) and a summary line.  --profile adds the encode kernel's time, the key bytes
per row, and the time of a device copy of the key columns' offsets and bytes for scale.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_agg_distinct import card  # noqa: E402


def dec_cells(torch, scaled, dev):
    """DECIMAL(15, 2) cells of non-negative values scaled < 10^11, in the stored form: one integer word, one fraction word"""
    n = scaled.shape[0]
    w = torch.zeros((n, 10), dtype=torch.int32, device=dev)
    w[:, 0] = 9 | (2 << 8) | (2 << 16)
    w[:, 1] = (scaled // 100).to(torch.int32)
    w[:, 2] = ((scaled % 100) * 10_000_000).to(torch.int32)
    return w.view(torch.uint8).reshape(n, 40)


def strings_of(torch, table, idx, dev):
    """(offsets, bytes) of rows table[idx] (table: a list of bytes of one length), built on the device"""
    w = len(table[0])
    assert all(len(b) == w for b in table)
    mat = torch.tensor([list(b) for b in table], dtype=torch.uint8, device=dev)
    return torch.arange(0, w * (idx.shape[0] + 1), w, dtype=torch.int64, device=dev), mat[idx].reshape(-1)


def customer_keys(torch, ids, dev):
    """18-byte Customer#NNNNNNNNN keys of ids, fixed width"""
    n = ids.shape[0]
    out = torch.empty((n, 18), dtype=torch.uint8, device=dev)
    out[:, :9] = torch.tensor(list(b"Customer#"), dtype=torch.uint8, device=dev)
    v = ids.clone()
    for j in range(17, 8, -1):
        out[:, j] = (v % 10 + 48).to(torch.uint8)
        v //= 10
    return torch.arange(0, 18 * (n + 1), 18, dtype=torch.int64, device=dev), out.reshape(-1)


def build_shape(torch, shape, n, dev, g):
    from tidb_b200 import abi
    from tidb_b200.plan import AggFunc, FieldType
    S = FieldType(abi.TYPE_STRING, abi.FLAG_NOT_NULL, collation=46)
    INT = FieldType(abi.TYPE_LONGLONG, abi.FLAG_NOT_NULL)
    DEC = FieldType(abi.TYPE_NEWDECIMAL, abi.FLAG_NOT_NULL, 15, 2)
    fr = lambda c: AggFunc(abi.AGG_FIRSTROW, c)  # noqa: E731
    if shape == "q1":
        combo = torch.randint(0, 4, (n,), device=dev, generator=g)
        flag_id = torch.tensor([0, 1, 1, 2], device=dev)[combo]
        stat_id = torch.tensor([0, 0, 1, 0], device=dev)[combo]
        keys = [strings_of(torch, [b"A", b"N", b"R"], flag_id, dev), strings_of(torch, [b"F", b"O"], stat_id, dev)]
        ints = [flag_id.to(torch.int64), stat_id.to(torch.int64)]
        qty = dec_cells(torch, torch.randint(100, 5001, (n,), device=dev, generator=g), dev)
        price = dec_cells(torch, torch.randint(90000, 10_500_000, (n,), device=dev, generator=g), dev)
        funcs = [fr(0), fr(1)] + [AggFunc(name, c, ret_type=abi.TYPE_NEWDECIMAL, ret_frac=2 if name == abi.AGG_SUM else 6)
                                  for c in (2, 3) for name in (abi.AGG_SUM, abi.AGG_AVG)] + [AggFunc(abi.AGG_COUNT, -1)]
        return ([S, S, DEC, DEC], [INT, INT, DEC, DEC], [0, 1], funcs, keys, ints, [qty, price], 4)
    if shape == "q16":
        brands = [b"Brand#%d%d" % (a, b) for a in range(1, 6) for b in range(1, 6)]
        types = [(a + b" " + b + b" " + c).ljust(25) for a in (b"STANDARD", b"SMALL", b"MEDIUM", b"LARGE", b"ECONOMY")
                 for b in (b"ANODIZED", b"BURNISHED", b"PLATED", b"POLISHED", b"BRUSHED") for c in (b"TIN", b"NICKEL", b"BRASS", b"STEEL")]
        bid = torch.randint(0, len(brands), (n,), device=dev, generator=g)
        tid = torch.randint(0, len(types), (n,), device=dev, generator=g)
        size = torch.randint(0, 8, (n,), device=dev, generator=g).to(torch.int64)
        supp = torch.randint(0, 10_000, (n,), device=dev, generator=g).to(torch.int64)
        keys = [strings_of(torch, brands, bid, dev), strings_of(torch, types, tid, dev)]
        funcs = [fr(0), fr(1), fr(2), AggFunc(abi.AGG_COUNT, 3, distinct=True)]
        return ([S, S, INT, INT], [INT, INT, INT, INT], [0, 1, 2], funcs, keys, [bid.to(torch.int64), tid.to(torch.int64)], [size, supp],
                len(brands) * len(types) * 8)
    ids = torch.randint(0, 10_000_000, (n,), device=dev, generator=g).to(torch.int64)
    return ([S, INT], [INT, INT], [0], [fr(0), AggFunc(abi.AGG_COUNT, -1)], [customer_keys(torch, ids, dev)], [ids],
            [torch.zeros(n, dtype=torch.int64, device=dev)], 10_000_000)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--shapes", nargs="+", default=["q1", "q16", "highcard"])
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    import torch
    from tidb_b200.device import DeviceAgg
    from tidb_b200.plan import AggPlan

    if not torch.cuda.is_available():
        raise SystemExit("bench_agg_string needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    info = card()
    print(json.dumps(info), flush=True)
    stream = torch.cuda.Stream(device=dev)
    n = args.rows
    summary = []
    for shape in args.shapes:
        g = torch.Generator(device=dev); g.manual_seed(16)
        with torch.cuda.stream(stream):
            stypes, itypes, gb, funcs, keys, ints, rest, groups = build_shape(torch, shape, n, dev, g)
        stream.synchronize()
        plans = {"string": AggPlan(stypes, gb, funcs, stream=stream.cuda_stream),
                 "bigint": AggPlan(itypes, gb, funcs, stream=stream.cuda_stream)}
        cols = {"string": list(keys) + list(rest), "bigint": list(ints) + list(rest)}
        last = {}

        def one(kind):
            agg = DeviceAgg(plans[kind])
            with torch.cuda.stream(stream):
                agg.push(cols[kind])
                rows, _, _ = agg.finish()
            last["rows"] = rows
            if kind == "string":
                last["ss"] = agg.string_stats()
            agg.close()

        def timed(kind):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            enc = 0.0
            with torch.cuda.stream(stream):
                e0.record(stream)
            for _ in range(args.steps):
                one(kind)
                if kind == "string":
                    enc += last["ss"].encode_ms
            with torch.cuda.stream(stream):
                e1.record(stream)
            stream.synchronize()
            return e0.elapsed_time(e1) / args.steps, enc / args.steps

        key_bytes = sum(int(o.numel()) * 8 + int(b.numel()) for o, b in keys)
        if args.profile:
            profile(torch, args, shape, lambda: one("string"), stream, info, keys, key_bytes)
        else:
            for k in ("string", "bigint"):
                for _ in range(args.warmup):
                    one(k)
            res = {"string": [], "bigint": [], "encode": []}
            for r in range(args.rounds):
                for k in (("string", "bigint") if r % 2 == 0 else ("bigint", "string")):
                    ms, enc = timed(k)
                    res[k].append(ms)
                    rec = {"rows": n, "shape": shape, "plan": k, "round": r, "step_ms": round(ms, 3), "groups": last["rows"],
                           "rows_per_s": round(n / (ms * 1e-3)), **info}
                    if k == "string":
                        ss = last["ss"]
                        res["encode"].append(enc)
                        rec.update({"encode_ms": round(enc, 3), "dict_entries": ss.dict_entries, "dict_bytes": ss.dict_bytes,
                                    "dict_slots": ss.dict_slots, "dict_grows": ss.dict_grows})
                    print(json.dumps(rec), flush=True)
            summary.append({"rows": n, "shape": shape, "key_bytes_per_row": round(key_bytes / n, 2),
                            **{f"{k}_ms": [round(v, 3) for v in vs] for k, vs in res.items()}, **info})
        del cols, keys, ints, rest, plans
        torch.cuda.empty_cache()
    if not args.profile:
        print(json.dumps({"summary": summary}), flush=True)


def profile(torch, args, shape, step, stream, info, keys, key_bytes) -> None:
    """device time per kernel of the string plan, and a device copy of its key columns' offsets and bytes for scale"""
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
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(stream):
        e0.record(stream)
        for _ in range(args.steps):
            for o, b in keys:
                o.clone(); b.clone()
        e1.record(stream)
    stream.synchronize()
    copy_ms = e0.elapsed_time(e1) / args.steps
    enc = sum(ms for k, (ms, _) in per.items() if "k_str_dict_encode" in k)
    print(json.dumps({"rows": args.rows, "shape": shape, "encode_kernel_ms": round(enc, 4), "key_bytes_per_row": round(key_bytes / args.rows, 2),
                      "key_copy_ms": round(copy_ms, 4), "encode_over_copy": round(enc / copy_ms, 2) if copy_ms else None, **info}), flush=True)
    for k, (ms, cnt) in sorted(per.items(), key=lambda kv: -kv[1][0]):
        print(json.dumps({"rows": args.rows, "shape": shape, "kernel": k, "ms_per_step": ms, "launches_per_step": cnt, **info}), flush=True)


if __name__ == "__main__":
    main()
