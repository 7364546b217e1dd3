#!/usr/bin/env python
"""Secondary measurements (not the bench.py headline): HashAgg config 3 (100M rows / 1M groups, SUM+COUNT) and the VecEval
kernels, device resident, CUDA events, with roofline fractions against MEASURED_PEAKS.json.  Results are verified
against torch reference reductions (COUNT bit-exact, SUM within 1e-6 relative)."""
import argparse, ctypes as C, json, os, sys, tempfile
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from bench import peaks
from tidb_b200 import abi
from tidb_b200.device import DeviceAgg, dev_chunk
from tidb_b200.plan import AggFunc, AggPlan, FieldType

ap = argparse.ArgumentParser()
ap.add_argument("--rows", type=int, default=100_000_000)
ap.add_argument("--groups", type=int, default=1_000_000)
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "bench_ops.jsonl"))
a = ap.parse_args()
dev = torch.device("cuda", 0)
peak, src = peaks()
lib = abi.load_lib()
stream = torch.cuda.Stream(device=dev)
os.makedirs(os.path.dirname(a.out), exist_ok=True)
fout = open(a.out, "a")
def emit(rec):
    print(json.dumps(rec)); fout.write(json.dumps(rec) + "\n"); fout.flush()

INT = FieldType(abi.TYPE_LONGLONG, abi.FLAG_NOT_NULL); DBL = FieldType(abi.TYPE_DOUBLE, abi.FLAG_NOT_NULL)
with torch.cuda.stream(stream):
    g = torch.Generator(device=dev); g.manual_seed(44)
    keys = torch.randint(0, a.groups, (a.rows,), device=dev, generator=g, dtype=torch.int64)
    x = torch.floor(torch.rand(a.rows, device=dev, generator=g, dtype=torch.float64) * 1e7)
stream.synchronize()
for G in sorted({a.groups, 1000}):
    k = keys if G == a.groups else keys % G
    plan = AggPlan([INT, DBL], [0], [AggFunc(abi.AGG_FIRSTROW, 0), AggFunc(abi.AGG_SUM, 1, abi.TYPE_DOUBLE), AggFunc(abi.AGG_COUNT, 1, abi.TYPE_DOUBLE)],
                   stream=stream.cuda_stream, expected_groups=G)
    times = []
    for it in range(a.steps + 1):
        agg = DeviceAgg(plan)
        with torch.cuda.stream(stream):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            agg.push([k, x])
            rows, cols, nulls = agg.finish()
            e1.record(stream)
        stream.synchronize()
        if it > 0:
            times.append(e0.elapsed_time(e1))
        if it == a.steps:
            st = agg.stats()
            from tidb_b200.parallel import KeyExchange
            def view(p, n, dt):
                class _A: pass
                o = _A(); o.__cuda_array_interface__ = {"shape": (n,), "typestr": dt, "data": (p, False), "version": 3}
                return torch.as_tensor(o, device=dev)
            gk = view(cols[0], rows, "<i8"); s = view(cols[1], rows, "<f8"); c = view(cols[2], rows, "<i8")
            assert rows == G and torch.equal(torch.sort(gk).values, torch.arange(G, device=dev))
            exp_c = torch.bincount(k, minlength=G); exp_s = torch.zeros(G, dtype=torch.float64, device=dev).scatter_add_(0, k, x)
            assert torch.equal(c, exp_c[gk]), "COUNT must be bit-exact"
            assert torch.allclose(s, exp_s[gk], rtol=1e-6, atol=0), "SUM within 1e-6 relative"
        agg.close()
    ms = sum(times) / len(times)
    bytes_alg = 16 * a.rows + 24 * G
    emit(dict(op="hashagg SUM+COUNT", rows=a.rows, groups=G, ms=ms, grows=a.rows / ms / 1e6, achieved_gbs=bytes_alg / ms / 1e6,
              frac=bytes_alg / ms / 1e6 / peak, update_ms=st.update_ms, finalize_ms=st.finalize_ms, launches=st.kernel_launches, peak=src))

# VecEval, device resident
n = a.rows
res = torch.empty(n, dtype=torch.int64, device=dev); resf = torch.empty(n, dtype=torch.float64, device=dev)
rn = torch.empty((n + 7) // 8, dtype=torch.uint8, device=dev)
def col(t):
    c = abi.TgColumn(); c.length = t.numel(); c.data = t.data_ptr(); c.elem_len = 8; c.null_bitmap = None; return c
ck, cx = col(keys), col(x)
def timeit(fn, nbytes, name):
    with torch.cuda.stream(stream):
        fn(); e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(a.steps): fn()
        e1.record(stream)
    stream.synchronize()
    ms = e0.elapsed_time(e1) / a.steps
    emit(dict(op=name, rows=n, ms=ms, grows=n / ms / 1e6, achieved_gbs=nbytes / ms / 1e6, frac=nbytes / ms / 1e6 / peak))
sp = C.c_void_p(stream.cuda_stream)
timeit(lambda: abi.check(lib.tg_vec_compare_int(0, 1, abi.CMP_LT, 0, 0, C.byref(ck), None, C.c_int64(a.groups // 2), C.c_void_p(res.data_ptr()), C.c_void_p(rn.data_ptr()), sp)), n * 16 + n // 8, "vec LT(int col, const) -> int64 0/1")
timeit(lambda: abi.check(lib.tg_vec_arith_real(0, 1, abi.ARITH_MUL, C.byref(cx), C.byref(cx), C.c_double(0), C.c_void_p(resf.data_ptr()), C.c_void_p(rn.data_ptr()), sp)), n * 24 + n // 8, "vec MUL(real col, real col)")
assert torch.equal(res, (keys < a.groups // 2).to(torch.int64)) and torch.equal(resf, x * x)
