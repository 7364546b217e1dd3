"""Parity at BASELINE.json's full sizes, against the oracle (not only size-independent properties):
  configs[1]  hash join 100M x 10M int64 keys, 8-byte payload, 100 % and 50 % match  -> every output row, bit-exact
  configs[2]  HashAgg SUM/COUNT GROUP BY int64, 100M rows / 1M groups (+ 1 % NULL x)  -> COUNT bit-exact, SUM within 1e-6
The oracle (oracle/join.cpp, oracle/agg.cpp) runs on the host cores of the GPU machine; these tests take about two minutes and
~25 GB of host memory.  TG_SKIP_FULL_SCALE=1 skips them (e.g. on a small host)."""
import os

import numpy as np
import pytest

import oracle_lib as O
from tidb_b200 import abi
from tidb_b200.chunk import Chunk, Column
from tidb_b200.plan import AggFunc, AggPlan, FieldType, JoinPlan

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(os.environ.get("TG_SKIP_FULL_SCALE") == "1", reason="TG_SKIP_FULL_SCALE=1")]
ODD = np.int64(0x9E3779B97F4A7C15 - (1 << 64))
INT = FieldType(abi.TYPE_LONGLONG, abi.FLAG_NOT_NULL)


def _threads():
    try:
        return max(1, min(64, len(os.sched_getaffinity(0))))
    except Exception:
        return 8


@pytest.mark.parametrize("match", [1.0, 0.5])
def test_config2_join_100m_x_10m_vs_oracle(match):
    import torch
    from tidb_b200.device import DeviceJoin
    nb, npb = 10_000_000, 100_000_000
    rng = np.random.default_rng(42)
    ids = rng.permutation(nb).astype(np.int64)
    bk, bv = ids * ODD, ids * 7
    rng = np.random.default_rng(43)
    pid = rng.integers(0, int(nb / match), npb).astype(np.int64)       # 50 %: uniform over twice the key range (SURVEY 8d input 2)
    pk, pv = pid * ODD, np.arange(npb, dtype=np.int64)
    plan = JoinPlan(abi.JOIN_INNER, [INT, INT], [INT, INT], [0], [0], build_is_right=True, device=0)
    dev = torch.device("cuda", 0)
    j = DeviceJoin(plan)
    j.build([torch.from_numpy(bk).to(dev), torch.from_numpy(bv).to(dev)])
    dpk, dpv = torch.from_numpy(pk).to(dev), torch.from_numpy(pv).to(dev)
    rows, cols, _ = j.probe([dpk, dpv])

    def view(p):
        class _A:
            pass
        a = _A()
        a.__cuda_array_interface__ = {"shape": (rows,), "typestr": "<i8", "data": (p, False), "version": 3}
        return torch.as_tensor(a, device=dev)
    got = [view(p).cpu().numpy() for p in cols]
    j.close()
    del dpk, dpv
    torch.cuda.empty_cache()
    oj = O.OracleJoin(plan, _threads())
    n, ocols = oj.run(Chunk([Column(bk), Column(bv)]).split(1 << 16), Chunk([Column(pk), Column(pv)]).split(1 << 16))
    oj.close()
    assert rows == n == int((pid < nb).sum())                                      # output row count bit-exact
    exp = [v for v, _ in ocols]
    go, eo = np.argsort(got[1], kind="stable"), np.argsort(exp[1], kind="stable")   # the probe payload is a unique row id
    for g, e in zip(got, exp):
        assert np.array_equal(g[go], e[eo])                                         # every output row, all four columns


@pytest.mark.parametrize("null_x", [False, True])
def test_config3_hashagg_100m_rows_1m_groups_vs_oracle(null_x):
    import torch
    from tidb_b200.device import DeviceAgg
    n, G = 100_000_000, 1_000_000
    rng = np.random.default_rng(44)
    g = rng.integers(0, G, n).astype(np.int64)
    x = np.floor(rng.random(n) * 1e7)
    xn = (rng.random(n) < 0.01) if null_x else None
    DBL = FieldType(abi.TYPE_DOUBLE, 0 if null_x else abi.FLAG_NOT_NULL)
    plan = AggPlan([INT, DBL], [0], [AggFunc(abi.AGG_FIRSTROW, 0), AggFunc(abi.AGG_SUM, 1, abi.TYPE_DOUBLE), AggFunc(abi.AGG_COUNT, 1, abi.TYPE_DOUBLE)],
                   expected_groups=G)
    dev = torch.device("cuda", 0)
    agg = DeviceAgg(plan)
    dn = None
    if null_x:
        dn = [None, torch.from_numpy(np.packbits(~xn, bitorder="little")).to(dev)]
    agg.push([torch.from_numpy(g).to(dev), torch.from_numpy(x).to(dev)], dn)
    rows, cols, nulls = agg.finish()

    def view(p, dt):
        class _A:
            pass
        a = _A()
        a.__cuda_array_interface__ = {"shape": (rows,), "typestr": dt, "data": (p, False), "version": 3}
        return torch.as_tensor(a, device=dev).cpu().numpy()
    gk, s, c = view(cols[0], "<i8"), view(cols[1], "<f8"), view(cols[2], "<i8")
    agg.close()
    oa = O.OracleAgg(plan, _threads(), min(16, _threads()))
    on, ocols = oa.run(Chunk([Column(g), Column(x, xn)]).split(1 << 16))
    oa.close()
    assert rows == on == G
    (ok, _), (os_, osn), (oc, _) = ocols
    go, eo = np.argsort(gk), np.argsort(ok)
    assert np.array_equal(gk[go], ok[eo])
    assert np.array_equal(c[go], oc[eo])                               # COUNT bit-exact
    assert not osn.any() and np.allclose(s[go], os_[eo], rtol=1e-6, atol=0)   # SUM(double) within 1e-6 relative
