#!/usr/bin/env python
"""Where does the L2 partition pass of the join probe stop paying?  Times the bench.py join shape (unique build keys, one
8-byte payload, 100 M probe rows) for tables of several sizes and densities and several slice counts, so that the slice
size at which the segment probe stops getting faster (the knee) and the cost of longer linear-probe runs at higher load
factors can be read off one run.

  python tools/probe_slices.py --sweep slice --out DIR     2.5 M build rows at load factor 0.35, P = 4, 8, 16
  python tools/probe_slices.py --sweep shape --out DIR     10 M build rows at load factors 0.35 .. 0.8, P = 16 and no pass
  python tools/probe_slices.py --lf 0.7 --parts 16 ...     one point (any axis takes a comma-separated list)
  python tools/probe_slices.py --sweep match --profile DIR  the bench shape at 100 .. 50 % match, in-place segment probe
                                                           forced on and off (TG_PROBE_INPLACE): where the automatic
                                                           choice should switch (join.cu: kInplaceMinMatch)
  --profile DIR                                            one more pass per point under torch.profiler: time per kernel

Every point prints one JSON line: step time at 100 % match and at 50 % match (the keys of bench.py's side line), table
slots, P and slice size, plus the card name and power limit read in the same run.  Not a bench: bench.py gives the
reported numbers."""
import argparse, json, os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from bench import ODD, gen_local, make_plan
from tidb_b200 import abi
from tidb_b200.device import DeviceJoin

SLOT_BYTES = 16
MAX_PARTS = 16   # TG_MAX_PARTS

SWEEPS = {   # (build rows, load factors, parts; 0 = the library's own choice, -1 = no partition pass)
    "slice": (2_500_000, "0.35", "4,8,16"),
    "shape": (10_000_000, "0.35,0.5,0.7,0.8", "16,-1"),
}
MATCHES = (1.0, 0.999, 0.99, 0.98, 0.95, 0.5)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return dict(card=name, power_limit_w=float(q[0]), sm_max_mhz=float(q[1]))
    except Exception as e:   # the numbers are reported without a power limit rather than not at all
        return dict(card=name, power_limit_w=None, note=f"nvidia-smi: {e}")


def timed(j, stream, cols, steps):
    with torch.cuda.stream(stream):
        for _ in range(3):
            j.probe(cols, sync=False)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(steps):
            j.probe(cols, sync=False)
        e1.record(stream)
    stream.synchronize()
    return e0.elapsed_time(e1) / steps


def profile(j, stream, cols, steps):
    """ms per step of each kernel, from a torch.profiler capture of `steps` probes"""
    from torch.profiler import ProfilerActivity, profile as tprof
    with tprof(activities=[ProfilerActivity.CUDA]) as prof:
        with torch.cuda.stream(stream):
            for _ in range(steps):
                j.probe(cols, sync=False)
        stream.synchronize()
    out = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if t > 0:
            out[ev.key] = out.get(ev.key, 0.0) + t / 1e3 / steps
    return dict(sorted(out.items(), key=lambda kv: -kv[1]))


def sweep_match(a, info, sinks):
    """bench.py's join at several match fractions, in-place segment probe forced on (1) and off (0): step time and, with
    --profile, ms per kernel"""
    nb = a.build_rows or 10_000_000
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    with torch.cuda.stream(stream):
        bk, bv, _, pv = gen_local(torch, dev, 0, 1, nb, a.probe_rows)
    j = DeviceJoin(make_plan(0, stream.cuda_stream))
    with torch.cuda.stream(stream):
        j.build([bk, bv])
    for m in MATCHES:
        with torch.cuda.stream(stream):
            g = torch.Generator(device=dev); g.manual_seed(4343)
            ids = torch.randint(0, nb, (a.probe_rows,), device=dev, generator=g, dtype=torch.int64)
            ids = torch.where(torch.rand(a.probe_rows, device=dev, generator=g) < m, ids, ids + nb)   # id >= nb: a miss
            want = int((ids < nb).sum().item())
            pk = ids * ODD
            del ids
        for mode in ("1", "0"):
            os.environ["TG_PROBE_INPLACE"] = mode
            with torch.cuda.stream(stream):
                rows, _, _ = j.probe([pk, pv], sync=True)
            assert rows == want, (m, mode, rows, want)
            rec = dict(match=m, inplace=mode == "1", probe_rows=a.probe_rows, build_rows=nb, ms=round(timed(j, stream, [pk, pv], a.steps), 3), **info)
            print(json.dumps(rec), flush=True)
            if sinks[0]:
                sinks[0].write(json.dumps(rec) + "\n"); sinks[0].flush()
            if a.profile:
                sinks[1].write(json.dumps(dict(match=m, inplace=mode == "1", kernels_ms=profile(j, stream, [pk, pv], a.steps))) + "\n"); sinks[1].flush()
        del pk
    j.close()
    os.environ.pop("TG_PROBE_INPLACE", None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sweep", choices=sorted(SWEEPS) + ["match"], default=None)
    ap.add_argument("--build-rows", type=int, default=None)
    ap.add_argument("--probe-rows", type=int, default=100_000_000)
    ap.add_argument("--lf", default=None, help="load factors; 0 = the library default")
    ap.add_argument("--parts", default=None, help="TG_PROBE_PARTS; 0 = the library's choice, -1 = TG_PROBE_PARTITION=0")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--profile", default=None, metavar="DIR", help="also write DIR/profile.jsonl: ms per step of every kernel")
    ap.add_argument("--out", default=None, metavar="DIR", help="also append the JSON lines to DIR/probe_slices.jsonl")
    a = ap.parse_args()
    info = card()
    sinks = []
    for d, name in ((a.out, "probe_slices.jsonl"), (a.profile, "profile.jsonl")):
        if d:
            os.makedirs(d, exist_ok=True)
        sinks.append(open(os.path.join(d, name), "a") if d else None)
    if a.sweep == "match":
        return sweep_match(a, info, sinks)
    nb, lfs, parts = SWEEPS[a.sweep] if a.sweep else (10_000_000, "0", "0")
    nb = a.build_rows or nb
    lfs, parts = a.lf or lfs, a.parts or parts
    L = lambda s, f: [f(x) for x in s.split(",")]
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    l2 = torch.cuda.get_device_properties(dev).L2_cache_size
    with torch.cuda.stream(stream):
        bk, bv, pk, pv = gen_local(torch, dev, 0, 1, nb, a.probe_rows)
        g2 = torch.Generator(device=dev); g2.manual_seed(4343)
        ids2 = torch.randint(0, 2 * nb, (a.probe_rows,), device=dev, generator=g2, dtype=torch.int64)
        pk2 = ids2 * ODD
        rows50 = int((ids2 < nb).sum().item())
        del ids2
    stream.synchronize()
    for lf in L(lfs, float):
        plan = make_plan(0, stream.cuda_stream)
        if lf:
            plan.load_factor = lf
        j = DeviceJoin(plan)
        with torch.cuda.stream(stream):
            j.build([bk, bv])
        bs = j.stats()
        table_mb = bs.table_slots * SLOT_BYTES / 2**20
        for p in L(parts, int):
            os.environ["TG_PROBE_PARTITION"] = "0" if p < 0 else "1"
            os.environ["TG_PROBE_PARTS"] = str(max(p, 0))
            with torch.cuda.stream(stream):
                rows, _, _ = j.probe([pk, pv], sync=True)
                rows2, _, _ = j.probe([pk2, pv], sync=True)
            assert rows == a.probe_rows and rows2 == rows50, (rows, rows2, rows50)
            paths = j.stats().paths   # accumulated over the handle's probes
            assert p < 0 or paths & abi.JOIN_PATH_PROBE_SEG, paths
            nparts = max(p, 0) or min(MAX_PARTS, -(-int(bs.table_slots * SLOT_BYTES) // (l2 // 4)))   # join.cu: probe_slices
            rec = dict(build_rows=nb, probe_rows=a.probe_rows, lf=lf or None, table_slots=bs.table_slots,
                       table_mb=round(table_mb, 1), parts=nparts if p >= 0 else 1, slice_mb=round(table_mb / nparts, 2) if p >= 0 else None,
                       partition=p >= 0, paths=paths, build_ms=round(bs.build_ms, 2),
                       ms=round(timed(j, stream, [pk, pv], a.steps), 3), ms_match50=round(timed(j, stream, [pk2, pv], a.steps), 3), **info)
            print(json.dumps(rec), flush=True)
            if sinks[0]:
                sinks[0].write(json.dumps(rec) + "\n"); sinks[0].flush()
            if a.profile:
                prof = dict(lf=rec["lf"], parts=rec["parts"], partition=rec["partition"],
                            kernels_ms=profile(j, stream, [pk, pv], a.steps), kernels_ms_match50=profile(j, stream, [pk2, pv], a.steps))
                sinks[1].write(json.dumps(prof) + "\n"); sinks[1].flush()
        j.close()
    os.environ.pop("TG_PROBE_PARTITION", None); os.environ.pop("TG_PROBE_PARTS", None)


if __name__ == "__main__":
    main()
