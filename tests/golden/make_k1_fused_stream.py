#!/usr/bin/env python
"""Writes tests/golden/k1_fused_stream.npz: the outputs of the fused multi-lambda CSR K1 (k1_csr_fused_kernel) on the seeded cases
of tests/k1_fused_stream_cases.py, for L = 1 .. 4 -- the gradient pass (g, f, sqrt(d)), the Hv pass and the Hessian-diagonal pass
of each case -- plus a digest of each case's inputs.  Needs a CUDA device.

    python tests/golden/make_k1_fused_stream.py [PROJECT_ROOT] [OUT]

PROJECT_ROOT: the checkout whose built package computes the outputs (default: this one).  The fixture was written once with the
package of the commit before phase A read 16-bit column ids, so that the test pins that change, and any later rework of the
kernel's loads, to the outputs they have to keep bit for bit."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = os.path.dirname(HERE)
root = os.path.abspath(sys.argv[1]) if len(sys.argv) > 1 else os.path.dirname(TESTS)
out = sys.argv[2] if len(sys.argv) > 2 else os.path.join(HERE, "k1_fused_stream.npz")
sys.path[:0] = [TESTS, os.path.join(root, "ml-ease_b200")]

import mlease_b200 as mb  # noqa: E402
import k1_fused_stream_cases as kc  # noqa: E402

res = {}
for L in (1, 2, 3, 4):
    r = kc.run_case(mb, L)
    assert r["info"]["kind"] == "fused" and r["info"]["RT"] == kc.SEG_ROWS, (r["info"]["kind"], r["info"]["RT"])
    for k in ("g", "f", "sd", "hv", "diag"):
        res["%s%d" % (k, L)] = r[k]
    res["digest%d" % L] = np.array(r["digest"])
    print("L=%d: LP=%d, %d segments x %d rows, digest %s" % (L, r["info"]["G"], r["info"]["chunks"][0], r["info"]["RT"], r["digest"][:16]))
os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
np.savez_compressed(out, **res)
print("wrote", out, os.path.getsize(out), "bytes", "package", mb.__file__)
