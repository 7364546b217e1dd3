#!/usr/bin/env python
"""Q3-shape (BASELINE configs[3]) at SF-like sizes on 1..N GPUs: end-to-end device time and GB/s over the scanned column bytes
(SURVEY 8d: 24.24 GB at SF = 100).  N = 1: python tools/bench_q3.py --sf 100;  N > 1: python -m torch.distributed.run
--nproc-per-node N ... tools/bench_q3.py --sf 100 (every rank generates its shard of the tables; the plan exchanges).
SF <= 10 on one GPU is verified against the torch rendering of the query; tests/ verify against the oracle operators.
--decimal (one GPU): the exact plan on DECIMAL(15,2) prices (q3.gen(decimal=True)): J2 carries the cells, the revenue is
an exact DECIMAL at scale 4 (verified cell by cell against the integer reference) and TopN orders by it; the record also
names the card and its power limit.  Two 40-byte lineitem columns take 48 GB at SF 100."""
import argparse, json, os, sys, tempfile
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from bench import peaks
from tidb_b200 import q3
ap = argparse.ArgumentParser(); ap.add_argument("--sf", type=float, default=10); ap.add_argument("--steps", type=int, default=3)
ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "bench_q3.jsonl")); ap.add_argument("--verify", type=int, default=1)
ap.add_argument("--decimal", action="store_true", help="DECIMAL(15,2) prices and the exact plan (one GPU)")
a = ap.parse_args()
world, rank, local = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0"))
torch.cuda.set_device(local)
dev = torch.device("cuda", local); stream = torch.cuda.Stream(device=dev)
nc, no, nl = int(150_000 * a.sf), int(1_500_000 * a.sf), int(6_000_000 * a.sf)
peak, src = peaks()
if world > 1 and a.decimal:
    raise SystemExit("--decimal runs on one GPU: the exchange moves 8-byte columns only")
if world > 1:
    import torch.distributed as dist
    dist.init_process_group("nccl", device_id=dev)
    with torch.cuda.stream(stream):
        d = q3.gen(dev, nc, no, nl, rank=rank, world=world)
    stream.synchronize()
    qd = q3.Q3Distributed(rank, world, dev, stream, d.o_orderkey.numel(), d.l_orderkey.numel())
    res = qd.run(d)
    dist.barrier(); torch.cuda.synchronize(dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(a.steps):
        qd.run(d)
    e1.record(stream)
    stream.synchronize(); dist.barrier()
    t = {}
    qd.run(d, timings=t)
    ms = torch.tensor([e0.elapsed_time(e1) / a.steps], dtype=torch.float64, device=dev)
    dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    ms = float(ms.item())
    scanned = d.scanned_bytes() * world
    if rank == 0:
        rec = dict(op="Q3-shape", sf=a.sf, n_gpus=world, rows=dict(customer=nc, orders=no, lineitem=nl), groups=res["groups"], ms=ms,
                   phases_ms={k: (round(v, 3) if not isinstance(v, dict) else {kk: (round(vv, 3) if not isinstance(vv, dict) else vv) for kk, vv in v.items()}) for k, v in t.items()},
                   scanned_gb=scanned / 1e9, gbs=scanned / ms / 1e6, frac=scanned / ms / 1e6 / (peak * world),
                   top=[[float(x) for x in c[:3]] for c in res["top"]], timing="wall per query incl. host-side exchange bookkeeping, max over ranks")
        print(json.dumps(rec)); os.makedirs(os.path.dirname(a.out), exist_ok=True); open(a.out, "a").write(json.dumps(rec) + "\n")
    qd.close(); dist.barrier(); dist.destroy_process_group()
    sys.exit(0)
with torch.cuda.stream(stream):
    d = q3.gen(dev, nc, no, nl, decimal=a.decimal)
    got = q3.run(d, dev, stream)
    if a.verify:
        exp = q3.reference(d)
        order = torch.argsort(got["orderkey"])
        assert torch.equal(got["orderkey"][order], exp["orderkey"]) and torch.equal(got["o_date"][order], exp["o_date"])
        if a.decimal:   # canonical cells of the exact sum at scale 4: one or two integer words, one fraction word
            w = got["revenue"][order].view(torch.int32).view(-1, 10).to(torch.int64)
            one = (w[:, 0] & 0xFF) == 9
            s4 = torch.where(one, w[:, 1] * 10**4 + w[:, 2] // 10**5, (w[:, 1] * 10**9 + w[:, 2]) * 10**4 + w[:, 3] // 10**5)
            assert bool(((w[:, 0] & 0xFF) <= 18).all()) and torch.equal(s4, exp["revenue_s4"])
        else:
            assert torch.allclose(got["revenue"][order], exp["revenue"], rtol=1e-6, atol=0)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    import time
    walls = []
    e0.record(stream)
    for _ in range(a.steps):
        w0 = time.perf_counter()
        q3.run(d, dev, stream, keep_groups=False)      # ends with the TopN rows on the host: the stream is idle when it returns
        walls.append((time.perf_counter() - w0) * 1e3)
    e1.record(stream)
    stream.synchronize()
    t = {}
    q3.run(d, dev, stream, keep_groups=False, timings=t)
stream.synchronize()
ms = e0.elapsed_time(e1) / a.steps
rec = dict(op="Q3-shape", sf=a.sf, n_gpus=1, rows=dict(customer=nc, orders=no, lineitem=nl), groups=int(got["orderkey"].numel()), ms=ms, wall_ms_per_run=[round(w, 2) for w in walls],
           phases_ms={k: (round(v, 3) if not isinstance(v, dict) else v) for k, v in t.items() if k != "rows"}, operator_rows=t.get("rows"),
           scanned_gb=d.scanned_bytes() / 1e9, gbs=d.scanned_bytes() / ms / 1e6, frac=d.scanned_bytes() / ms / 1e6 / peak, verified=bool(a.verify))
if a.decimal:
    from bench_join_decimal import card   # tools/ is the script's directory
    rec.update(decimal=True, top=[int(x) for x in got["top"][0]], **card())
print(json.dumps(rec)); os.makedirs(os.path.dirname(a.out), exist_ok=True); open(a.out, "a").write(json.dumps(rec) + "\n")
