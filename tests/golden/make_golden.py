#!/usr/bin/env python
"""Generate tests/golden/*.json — small seeded join / aggregation cases with the result the CPU oracle (oracle/, the
restatement of the reference's algorithm) produces.  Re-run after an intentional semantic change of the oracle:

    python tests/golden/make_golden.py

The reference itself (Go) is not run by this project, so the expected outputs come from the oracle, which is pinned to the
reference by the known-answer tests in tests/test_oracle_kat.py / test_oracle_join.py / test_oracle_agg_vec.py.  The
fixtures freeze today's oracle behaviour: tests/test_golden.py fails if either the oracle (CPU) or the CUDA path (GPU)
drifts from them.  Rows are stored as sorted lists; NULL = null; doubles as repr strings (bit exact)."""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE)); sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from nested_loop import columns_to_rows  # noqa: E402
from test_oracle_agg_vec import run_agg  # noqa: E402
from test_oracle_join import JOIN_TYPES, make_case, run_oracle  # noqa: E402
from tidb_b200 import abi  # noqa: E402
from tidb_b200.chunk import Chunk, Column  # noqa: E402
from tidb_b200.plan import AggFunc, AggPlan, FieldType, JoinPlan  # noqa: E402


def enc(v):
    if v is None:
        return None
    if isinstance(v, (float, np.floating)):
        return {"f": repr(float(v))}
    return int(v)


def rows_json(rows):
    key = lambda r: tuple((0, 0) if v is None else (1, float(v)) for v in r)
    return [[enc(v) for v in r] for r in sorted(rows, key=key)]


def chunk_json(chunks):
    out = []
    for c in chunks:
        cols = []
        for col in c.columns:
            nulls = col.nulls()
            cols.append({"dtype": str(col.data.dtype), "data": [enc(v) for v in col.data.tolist()],
                         "nulls": [bool(x) for x in nulls.tolist()]})
        out.append({"cols": cols, "sel": None if c.sel is None else [int(x) for x in c.sel.tolist()]})
    return out


def types_json(ts):
    return [[t.tp, t.flag] for t in ts]


def main():
    cases = []
    for jt in JOIN_TYPES:
        for build_is_right in (True, False):
            if jt in (abi.JOIN_LEFT_OUTER_SEMI, abi.JOIN_ANTI_LEFT_OUTER_SEMI) and not build_is_right:
                continue   # NewJoinProbe panics (base_join_probe.go:913)
            rng = np.random.default_rng(9000 + jt * 2 + int(build_is_right))
            ltypes, rtypes, l, r = make_case(rng, 120, 160, 0.12, True, jt % 2 == 0)
            semi = jt >= abi.JOIN_SEMI
            lused, rused = [0, 1, 2], ([] if semi else [2, 0])
            plan = JoinPlan(jt, ltypes, rtypes, [1], [0], build_is_right=build_is_right, lused=lused, rused=rused)
            cases.append({"join_type": jt, "build_is_right": build_is_right, "left_types": types_json(ltypes),
                          "right_types": types_json(rtypes), "left_keys": [1], "right_keys": [0], "lused": lused, "rused": rused,
                          "left": chunk_json(l), "right": chunk_json(r), "expected": rows_json(run_oracle(plan, l, r))})
    json.dump({"source": "oracle/join.cpp via tests/golden/make_golden.py", "cases": cases}, open(os.path.join(HERE, "join_cases.json"), "w"))

    # same plan shape as tests/test_gpu_agg_vec.py::test_agg_random_vs_oracle: nullable group key (NULL keys form a group),
    # nullable double argument, NOT NULL int argument
    INT, INT_NN, DBL = FieldType(abi.TYPE_LONGLONG, 0), FieldType(abi.TYPE_LONGLONG, abi.FLAG_NOT_NULL), FieldType(abi.TYPE_DOUBLE, 0)
    rng = np.random.default_rng(77)
    n = 600
    g = rng.integers(0, 23, n).astype(np.int64); gn = rng.random(n) < 0.05
    x = np.floor(rng.random(n) * 1000) / 8; xn = rng.random(n) < 0.1       # multiples of 1/8: every partial sum is exact
    y = rng.integers(-50, 50, n).astype(np.int64)
    chunks = Chunk([Column(g, gn), Column(x, xn), Column(y)]).split(64)
    funcs = [(abi.AGG_FIRSTROW, 0, abi.TYPE_LONGLONG), (abi.AGG_SUM, 1, abi.TYPE_DOUBLE), (abi.AGG_COUNT, 1, abi.TYPE_DOUBLE),
             (abi.AGG_AVG, 1, abi.TYPE_DOUBLE), (abi.AGG_COUNT, -1, abi.TYPE_LONGLONG), (abi.AGG_MIN, 2, abi.TYPE_LONGLONG),
             (abi.AGG_MAX, 2, abi.TYPE_LONGLONG)]
    plan = AggPlan([INT, DBL, INT_NN], [0], [AggFunc(a, c, t) for a, c, t in funcs])
    agg = {"col_types": types_json([INT, DBL, INT_NN]), "group_by": [0], "funcs": [list(f) for f in funcs], "input": chunk_json(chunks),
           "expected": rows_json(run_agg(plan, chunks)), "float_cols": [1, 3]}
    json.dump({"source": "oracle/agg.cpp via tests/golden/make_golden.py", "cases": [agg]}, open(os.path.join(HERE, "agg_cases.json"), "w"))
    print("wrote", len(cases), "join cases and 1 aggregation case")


if __name__ == "__main__":
    main()
