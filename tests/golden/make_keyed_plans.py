#!/usr/bin/env python
"""Writes tests/golden/keyed_plans.npz: for every case of tests/keyed_plan_cases.py, three keyed budgets and, under each, the key
bounds the call recorded, whether it streamed, and its outputs.  Needs a CUDA device.

    python tests/golden/make_keyed_plans.py [PROJECT_ROOT] [OUT]

PROJECT_ROOT: the checkout whose built package computes the plans (default: this one).  The budgets of each case's plans are found
here, on the package that writes the fixture, on a grid of factor 1.2 down from 4 GiB: 0 (resident, one chunk); the middle of the
caps under which the call stays resident but runs in several chunks (chunked), or streams in exactly one key range (one_range); and
the first cap that streams it through at least 4 key ranges (streamed).  The
fixture was written with the package of the commit before the keyed calls' resident and streamed drivers became one pipeline, so
that the test pins the plans and outputs of both to what they were."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = os.path.dirname(HERE)
root = os.path.abspath(sys.argv[1]) if len(sys.argv) > 1 else os.path.dirname(TESTS)
out = sys.argv[2] if len(sys.argv) > 2 else os.path.join(HERE, "keyed_plans.npz")
sys.path[:0] = [TESTS, os.path.join(root, "ml-ease_b200")]

import mlease_b200 as mb  # noqa: E402
import keyed_plan_cases as kc  # noqa: E402

res = {}
for name, case in kc.CASES.items():
    data = case["make"]()
    b0, s0, _ = kc.run(mb, name, 0, data)
    assert not s0 and len(b0) == 2, (name, b0, s0)
    found = {"resident": [0], "chunked": [], "one_range": [], "streamed": []}
    cap = 4 << 30
    while cap > 4096 and not found["streamed"]:
        b, s, _ = kc.run(mb, name, cap, data)
        kind = "chunked" if not s and len(b) > 2 else "one_range" if s and len(b) == 2 else "streamed" if s and len(b) > 4 else None
        if kind:
            found[kind].append(cap)
        cap = int(cap / 1.2)
    plans = case.get("plans", ("resident", "chunked", "streamed"))
    if not all(found[p] for p in plans):
        print("%-26s NO PLAN: %s" % (name, {p: found[p] for p in plans}), flush=True)
        continue
    for i, plan in enumerate(plans):
        budget = found[plan][(len(found[plan]) - 1) // 2] if plan != "streamed" else found[plan][0]
        b, s, o = kc.run(mb, name, budget, data)
        res["%s__%d__budget" % (name, i)] = np.int64(budget)
        res["%s__%d__bounds" % (name, i)] = b
        res["%s__%d__streamed" % (name, i)] = np.bool_(s)
        for k, a in o.items():
            res["%s__%d__%s" % (name, i, k)] = a
        print("%-26s %-9s budget %11d: %s, %d chunks %s" % (name, plan, budget, "streamed" if s else "resident", len(b) - 1,
                                                           np.diff(b).tolist() if len(b) < 12 else ""), flush=True)
os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
np.savez_compressed(out, **res)
print("wrote", out, os.path.getsize(out), "bytes", "package", mb.__file__)
