"""The Q3-shape pipeline on TiDB's exact types (tidb_b200/q3.py with gen(decimal=True)) at SF = 0.1: l_extendedprice and
l_discount are DECIMAL(15,2) cells, J2 carries them, the aggregation sums SUM(l_extendedprice * (1 - l_discount)) as an
exact DECIMAL at scale 4 and TopN orders by that DECIMAL column DESC, then o_orderdate.  Against the exact integer
reference of q3.reference: the group count, every revenue cell bit for bit (the canonical cell of the exact sum,
tests/mydecimal_expr.py), and the TopN rows' (revenue, o_orderdate) keys, tie groups as sets."""
import numpy as np
import pytest
import torch

import mydecimal_expr as X
from tidb_b200 import q3

pytestmark = pytest.mark.gpu


def test_q3_decimal_exact_revenue_and_topn():
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    with torch.cuda.stream(stream):
        d = q3.gen(dev, 15_000, 150_000, 600_000, decimal=True)
        got = q3.run(d, dev, stream, topn=10)
        ref = q3.reference(d)
        stream.synchronize()
    assert d.l_price.shape == (600_000, 40) and d.l_disc.shape == (600_000, 40)
    # the same rows as the DOUBLE plan's data: only the price columns change type
    with torch.cuda.stream(stream):
        dd = q3.gen(dev, 15_000, 150_000, 600_000)
        stream.synchronize()
    assert torch.equal(q3.cents_of(d.l_price), torch.round(dd.l_price * 100).to(torch.int64))
    assert torch.equal(q3.cents_of(d.l_disc), torch.round(dd.l_disc * 100).to(torch.int64))

    ok = ref["orderkey"].cpu().numpy()
    s4 = ref["revenue_s4"].cpu().numpy()
    od = ref["o_date"].cpu().numpy()
    assert got["groups"] == len(ok)
    g_ok = got["orderkey"].cpu().numpy()
    order = np.argsort(g_ok)
    assert np.array_equal(g_ok[order], ok)
    assert np.array_equal(got["o_date"].cpu().numpy()[order], od)
    assert np.array_equal(got["o_prio"].cpu().numpy()[order], ref["o_prio"].cpu().numpy())
    cells = got["revenue"].cpu().numpy()[order]
    assert cells.shape == (len(ok), 40)
    bad = [i for i in range(len(ok)) if bytes(cells[i]) != X.sum_result(int(s4[i]), q3.REVENUE_FRAC)]
    assert not bad, f"{len(bad)} revenue cells differ, first for order key {ok[bad[0]]}"

    # TopN 10: ORDER BY revenue DESC, o_orderdate
    top_ok, top_rev, top_date, top_prio = got["top"]
    assert len(top_ok) == 10 and top_rev.shape == (10, 40)
    exp = np.lexsort((od, -s4))[:10]
    row = {int(k): i for i, k in enumerate(ok)}
    got_rows = [row[int(k)] for k in top_ok]
    assert len(set(got_rows)) == 10
    for i, r in enumerate(got_rows):
        assert bytes(top_rev[i]) == bytes(cells[r]) and top_date[i] == od[r] and top_prio[i] == ref["o_prio"].cpu().numpy()[r]
    assert [(s4[r], od[r]) for r in got_rows] == [(s4[r], od[r]) for r in exp]
    # a key group wholly inside the first 10 rows holds the reference's rows (the last group may be cut)
    last = (s4[exp[-1]], od[exp[-1]])
    assert {r for r in got_rows if (s4[r], od[r]) != last} == {int(r) for r in exp if (s4[r], od[r]) != last}
