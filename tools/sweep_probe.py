#!/usr/bin/env python
"""A/B sweep of the fused probe kernel's launch parameters on one H100 (config 2 shape).
Each line of --out (default: sweep_probe.jsonl in the temporary directory) is one (table layout, kernel variant) point, timed with CUDA events
over `--steps` launches after 2 warm-ups.  Not a bench: use bench.py for reported numbers."""
import argparse, itertools, json, os, sys, tempfile
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from bench import gen_local, make_plan, peaks
from tidb_b200.device import DeviceJoin

ap = argparse.ArgumentParser()
ap.add_argument("--build-rows", type=int, default=10_000_000)
ap.add_argument("--probe-rows", type=int, default=100_000_000)
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--lf", default="0.4")
ap.add_argument("--pair", default="1")
ap.add_argument("--l2", default="0")
ap.add_argument("--variant", default="1")
ap.add_argument("--R", default="4")
ap.add_argument("--evict", default="0")
ap.add_argument("--ctas", default="0")
ap.add_argument("--part", default="1")
ap.add_argument("--parts", default="0")
ap.add_argument("--tma", default="0")
ap.add_argument("--stages", default="4")
ap.add_argument("--tma-ctas", default="3")
ap.add_argument("--agg", default="1")
ap.add_argument("--lean", default="0", help="TG_PROBE_SEG_LEAN: 0 production segment probe, 1 lean, 2 lean + register prefetch")
ap.add_argument("--carve", default="-1", help="TG_PROBE_CARVEOUT: preferred shared-memory carve-out (%%) of the segment probe, -1 = default")
ap.add_argument("--segvec", default="1", help="TG_PROBE_SEG_VEC")
ap.add_argument("--subseg", default="1", help="TG_PROBE_SUBSEG: CTA-private sub-segments in the L2 partition pass")
ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "sweep_probe.jsonl"))
a = ap.parse_args()
L = lambda s, f: [f(x) for x in s.split(",")]
dev = torch.device("cuda", 0)
stream = torch.cuda.Stream(device=dev)
with torch.cuda.stream(stream):
    bk, bv, pk, pv = gen_local(torch, dev, 0, 1, a.build_rows, a.probe_rows)
stream.synchronize()
os.makedirs(os.path.dirname(a.out), exist_ok=True)
fout = open(a.out, "a")
for lf, pair, l2 in itertools.product(L(a.lf, float), L(a.pair, int), L(a.l2, int)):
    os.environ["TG_PAIR_HOME"] = str(pair); os.environ["TG_L2_FETCH"] = str(l2)
    plan = make_plan(0, stream.cuda_stream); plan.load_factor = lf
    j = DeviceJoin(plan)
    with torch.cuda.stream(stream):
        j.build([bk, bv])
    bs = j.stats()
    for subseg, variant, R, ev, ctas, part, parts, tma, stages, tctas, agg, lean, carve, segvec in itertools.product(L(a.subseg, int), L(a.variant, int), L(a.R, int), L(a.evict, int), L(a.ctas, int), L(a.part, int), L(a.parts, int), L(a.tma, int), L(a.stages, int), L(a.tma_ctas, int), L(a.agg, int), L(a.lean, int), L(a.carve, int), L(a.segvec, int)):
        if variant == 0 and (R != L(a.R, int)[0] or ev != L(a.evict, int)[0] or part != L(a.part, int)[0] or parts != L(a.parts, int)[0]):
            continue
        if part == 0 and parts != L(a.parts, int)[0]:
            continue
        if tma == 0 and (stages != L(a.stages, int)[0] or tctas != L(a.tma_ctas, int)[0] or agg != L(a.agg, int)[0]):
            continue
        if part != 1 and (lean != L(a.lean, int)[0] or carve != L(a.carve, int)[0] or segvec != L(a.segvec, int)[0]):
            continue
        os.environ.update(TG_PROBE_SUBSEG=str(subseg)); os.environ.update(TG_PROBE_SEG_LEAN=str(lean), TG_PROBE_CARVEOUT=str(carve), TG_PROBE_SEG_VEC=str(segvec))
        os.environ.update(TG_PROBE_VARIANT=str(variant), TG_PROBE_R=str(R), TG_PROBE_EVICT_LAST=str(ev), TG_PROBE_CTAS_PER_SM=str(ctas), TG_PROBE_PARTITION=str(part), TG_PROBE_PARTS=str(parts), TG_PROBE_TMA=str(tma), TG_PROBE_STAGES=str(stages), TG_PROBE_TMA_CTAS=str(tctas), TG_PROBE_CTA_AGG=str(agg))
        with torch.cuda.stream(stream):
            rows, _, _ = j.probe([pk, pv], sync=True)
            assert rows == a.probe_rows, rows
            j.probe([pk, pv], sync=False)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(a.steps):
                j.probe([pk, pv], sync=False)
            e1.record(stream)
        stream.synchronize()
        ms = e0.elapsed_time(e1) / a.steps
        rec = dict(subseg=subseg, lean=lean, carve=carve, segvec=segvec, lf=lf, pair=pair, l2=l2, part=part, parts=parts, tma=tma, stages=stages, tma_ctas=tctas, agg=agg, variant=variant, R=R, evict_last=ev, ctas=ctas, ms=ms, grows=a.probe_rows / ms / 1e6,
                   frac=64 * a.probe_rows / (ms * 1e-3) / 1e9 / peaks()[0], slots=bs.table_slots, build_ms=bs.build_ms)
        print(json.dumps(rec)); fout.write(json.dumps(rec) + "\n"); fout.flush()
    j.close()
