"""The N > 1 product path on real GPUs (needs >= 2 devices; `python -m pytest tests/test_gpu_multigpu.py -m gpu`):
MailboxExchange (bulk stores into the peers over NVLink + device mailboxes) feeding tg_join_probe_dev_seg, several
pipelined steps, both transports; the union of the ranks' outputs must equal the oracle's join of the global inputs as
sorted row multisets (checkChunksEqual, inner_join_probe_test.go:137).  Overflow of a receive region and a silent sender
must surface as errors on every rank."""
import os
import socket
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import oracle_lib as O
from nested_loop import columns_sorted
from tidb_b200 import abi
from tidb_b200.chunk import Chunk, Column
from tidb_b200.plan import FieldType, JoinPlan

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close()
    return p


@pytest.mark.parametrize("dma", [0, 1, 2, 3])
def test_mailbox_exchange_two_ranks_vs_oracle(dma):
    lib = abi.load_lib()
    if lib.tg_device_count() < 2:
        pytest.skip("needs 2 GPUs")
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import mgpu_worker as W
    world, nb, npr, steps = 2, 60_000, 300_000, 4
    with tempfile.TemporaryDirectory() as td:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
               "--master-port", str(_free_port()), os.path.join(ROOT, "tests", "mgpu_worker.py"), "--out", td,
               "--build-rows", str(nb), "--probe-rows", str(npr), "--steps", str(steps), "--dma", str(dma)]
        r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-6000:]
        res = [np.load(os.path.join(td, f"rank{k}.npz")) for k in range(world)]
    INT = FieldType(abi.TYPE_LONGLONG, abi.FLAG_NOT_NULL)
    plan = JoinPlan(abi.JOIN_INNER, [INT, INT], [INT, INT], [0], [0], build_is_right=True)
    shards = [W.gen(k, world, nb, npr, 0) for k in range(world)]
    build = Chunk([Column(np.concatenate([s[0] for s in shards])), Column(np.concatenate([s[1] for s in shards]))])
    for s_ in range(steps):
        ps = [W.gen(k, world, nb, npr, s_) for k in range(world)]
        probe = Chunk([Column(np.concatenate([p[2] for p in ps])), Column(np.concatenate([p[3] for p in ps]))])
        n, ocols = O.OracleJoin(plan, 4).run(build.split(4096), probe.split(4096))
        got = [np.concatenate([res[k][f"s{s_}c{c}"] for k in range(world)]) for c in range(4)]
        assert len(got[0]) == n, (s_, len(got[0]), n)
        assert np.array_equal(columns_sorted(ocols), columns_sorted([(g, np.zeros(len(g), dtype=bool)) for g in got])), f"step {s_}"
    # skewed steps: spill area + counted exchange of the spilled rows; the union over ranks must still be the whole join
    ps = [W.gen_skew(k, world, nb, npr, s_) for k in range(world) for s_ in range(2)]
    probe = Chunk([Column(np.concatenate([p[0] for p in ps])), Column(np.concatenate([p[1] for p in ps]))])
    n, ocols = O.OracleJoin(plan, 4).run(build.split(4096), probe.split(4096))
    got = [np.concatenate([res[k][f"skew_c{c}"] for k in range(world)]) for c in range(4)]
    assert sum(int(res[k]["spilled_rows"][0]) for k in range(world)) > 0.2 * 2 * world * npr, "the skewed steps must actually spill"
    assert len(got[0]) == n, (len(got[0]), n)
    assert np.array_equal(columns_sorted(ocols), columns_sorted([(g, np.zeros(len(g), dtype=bool)) for g in got])), "skewed steps"
    for k in range(world):
        assert int(res[k]["overflow_detected"][0]) == 1, "a receive-region overflow must be reported on every rank"
        assert int(res[k]["timeout_detected"][0]) == 1, "a silent sender must end the wait with an error, not a hang"


def test_q3_two_ranks_vs_oracle():
    # the distributed Q3-shape plan (broadcast customer, repartition filtered orders and lineitem by order key over NVLink,
    # shard-local J2 + HashAgg + TopN, global TopN) on 2 ranks against the oracle operators on the concatenated shards
    lib = abi.load_lib()
    if lib.tg_device_count() < 2:
        pytest.skip("needs 2 GPUs")
    sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import topn as OT
    from test_gpu_q3 import oracle_q3
    world = 2
    with tempfile.TemporaryDirectory() as td:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
               "--master-port", str(_free_port()), os.path.join(ROOT, "tests", "mgpu_q3_worker.py"), "--out", td]
        r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-6000:]
        res = [dict(np.load(os.path.join(td, f"q3_rank{k}.npz"))) for k in range(world)]
    cols = ["c_custkey", "c_seg", "o_orderkey", "o_custkey", "o_date", "o_prio", "l_orderkey", "l_price", "l_disc", "l_ship"]
    h = {c: np.concatenate([res[k][c] for k in range(world)]) for c in cols}
    n1, n2, ng, (ok, rev, od, op) = oracle_q3(h)
    assert int(res[0]["groups"][0]) == ng
    exp_top = OT.topn_rows(list(zip(ok.tolist(), rev.tolist(), od.tolist(), op.tolist())), ["int", "real", "int", "int"], [(1, True), (2, False)], 0, 10)
    top = [res[0][f"top{c}"] for c in range(4)]
    assert len(top[0]) == len(exp_top) == 10
    for i, e in enumerate(exp_top):
        assert (int(top[0][i]), int(top[2][i]), int(top[3][i])) == (e[0], e[2], e[3])
        assert top[1][i] == pytest.approx(e[1], rel=1e-6)
