#!/usr/bin/env python
"""Where the time of the join probe step goes, kernel by kernel, next to what a plain copy of the same bytes costs.

  python tools/bench_probe_pass.py [--steps 20] [--out DIR]

Runs bench.py's N = 1 join (100 M probe rows against 10 M unique build keys, one 8-byte payload, 100 % match): a
verifying call whose row count the host reads, a few warm-up steps, `--steps` steps timed with CUDA events, then `--steps`
more under torch.profiler for the time per kernel (the partition scatter, the segment probe, the hole fill and the rest).
The ceiling row copies two 100 M-row int64 columns device to device with torch (1.6 GB read + 1.6 GB written, the
scatter's traffic), timed with CUDA events in the same run.  The card name and power limit are read in the same run.
TIDBGPU_LIB selects another build of the library.  Prints one JSON line; --out also writes it to DIR/probe_pass.json."""
import argparse, json, os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from bench import gen_local, make_plan
from tidb_b200 import abi
from tidb_b200.device import DeviceJoin


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return dict(card=name, power_limit_w=float(q[0]), sm_max_mhz=float(q[1]))
    except Exception as e:   # the numbers are reported without a power limit rather than not at all
        return dict(card=name, power_limit_w=None, note=f"nvidia-smi: {e}")


def event_ms(stream, fn, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(stream):
        e0.record(stream)
        for _ in range(steps):
            fn()
        e1.record(stream)
    stream.synchronize()
    return e0.elapsed_time(e1) / steps


def kernel_ms(stream, fn, steps):
    """ms per step of each kernel, from a torch.profiler capture of `steps` calls"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        with torch.cuda.stream(stream):
            for _ in range(steps):
                fn()
        stream.synchronize()
    out = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if t > 0:
            out[ev.key] = out.get(ev.key, 0.0) + t / 1e3 / steps
    return {k: round(v, 4) for k, v in sorted(out.items(), key=lambda kv: -kv[1])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--build-rows", type=int, default=10_000_000)
    ap.add_argument("--probe-rows", type=int, default=100_000_000)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None, metavar="DIR")
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    with torch.cuda.stream(stream):
        bk, bv, pk, pv = gen_local(torch, dev, 0, 1, a.build_rows, a.probe_rows)
    j = DeviceJoin(make_plan(0, stream.cuda_stream))
    with torch.cuda.stream(stream):
        j.build([bk, bv])
        rows, _, _ = j.probe([pk, pv], sync=True)
    assert rows == a.probe_rows, (rows, a.probe_rows)
    step = lambda: j.probe([pk, pv], sync=False)
    event_ms(stream, step, 3)
    step_ms = event_ms(stream, step, a.steps)
    kernels = kernel_ms(stream, step, a.steps)
    j.close()

    # ceiling: the scatter's bytes as a plain device copy of two int64 columns
    with torch.cuda.stream(stream):
        dst = [torch.empty_like(pk), torch.empty_like(pv)]
    copy = lambda: (dst[0].copy_(pk), dst[1].copy_(pv))
    event_ms(stream, copy, 3)
    copy_ms = event_ms(stream, copy, a.steps)
    copy_bytes = 2 * 2 * 8 * a.probe_rows

    def pick(sub):
        return round(sum(v for k, v in kernels.items() if sub in k), 4)
    scatter_ms = pick("k_partition_scatter_bulk")
    rec = dict(build_rows=a.build_rows, probe_rows=a.probe_rows, steps=a.steps, lib=os.path.abspath(abi.LIB_PATH),
               step_ms=round(step_ms, 4),
               split_ms=dict(scatter=scatter_ms, probe_inplace=pick("k_probe_inner_u1_seg_inplace"), probe_lean=pick("k_probe_inner_u1_seg_lean"),
                             holes=pick("k_inplace_holes"), scan=pick("k_scan"), fill=pick("k_inplace_fill")),
               scatter_tbs=round(copy_bytes / (scatter_ms * 1e-3) / 1e12, 3) if scatter_ms else None,
               ceiling=dict(what="torch copy_ of two int64 columns, device to device", bytes=copy_bytes, ms=round(copy_ms, 4),
                            tbs=round(copy_bytes / (copy_ms * 1e-3) / 1e12, 3)),
               kernels_ms=kernels, **card())
    line = json.dumps(rec)
    print(line, flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "probe_pass.json"), "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
