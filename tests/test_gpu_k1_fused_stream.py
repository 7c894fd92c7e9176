"""The fused multi-lambda CSR K1 (-m gpu) against a golden fixture, bit for bit: gradient (g, f, sqrt(d)), Hv and Hessian-diagonal
passes for L = 1 .. 4 on the cases of tests/k1_fused_stream_cases.py (long rows, an empty segment, segment starts at every 16-byte
residue, column ids >= 32768), written by tests/golden/make_k1_fused_stream.py.  Each output is also held to the per-column bounds
of tests/k1_reference.py, so the fixture itself is checked against fp64."""
import os

import numpy as np
import pytest

import k1_fused_stream_cases as kc
import k1_reference as kr

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "k1_fused_stream.npz")


@pytest.fixture(scope="module")
def mb():
    import mlease_b200
    return mlease_b200


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


@pytest.mark.gpu
@pytest.mark.parametrize("L", [1, 2, 3, 4])
def test_fused_k1_matches_golden(mb, golden, L):
    r = kc.run_case(mb, L)
    assert str(golden["digest%d" % L]) == r["digest"], "the seeded inputs changed: regenerate the fixture on a trusted build"
    info = r["info"]
    assert info["kind"] == "fused" and info["G"] == {1: 1, 2: 2, 3: 4, 4: 4}[L]
    assert info["RT"] == kc.SEG_ROWS and np.all(info["chunks"] == kc.SEGS)
    for k in ("g", "f", "sd", "hv", "diag"):
        np.testing.assert_array_equal(r[k], golden["%s%d" % (k, L)], err_msg="%s L=%d" % (k, L))
    _, parts, W, V, _ = kc.make_case(L)
    for b in range(len(W)):
        part = parts[b // L]
        ref = kr.reference(part, W[b])
        plan = kr.plan_from_info(info, b, part.n)
        err = kr.row_errors(part, ref, plan)
        bnd, _ = kr.grad_bound(part, ref, plan, err)
        assert np.all(kr.ratio(r["g"][b] - ref.g, bnd) <= 1.0), ("g", L, b)
        assert abs(r["f"][b] - ref.f) <= kr.loss_bound(part, ref, plan, err), ("f", L, b)
        assert np.all(kr.ratio(r["sd"][b].astype(np.float64) - ref.sd, kr.sd_bound(ref, err)) <= 1.0), ("sd", L, b)
        for mode, name in ((1, "hv"), (2, "diag")):
            hv_ref, hv_bnd = kr.hv_reference_and_bound(part, W[b], V[b], mode, plan)
            assert np.all(kr.ratio(r[name][b] - hv_ref, hv_bnd) <= 1.0), (name, L, b)


def test_cases_cover_the_streaming_edges():
    """The inputs hold what the fixture is meant to exercise (CPU-side, no device needed to see it)."""
    for L in (1, 2, 3, 4):
        arrs, _, _, _, _ = kc.make_case(L)
        for a in arrs:
            rp = a["rowptr"]
            starts = rp[np.arange(kc.SEGS) * kc.SEG_ROWS]
            assert set((starts % 8).tolist()) == set(range(8))
            assert rp[(kc.EMPTY_SEG + 1) * kc.SEG_ROWS] == rp[kc.EMPTY_SEG * kc.SEG_ROWS]
            assert np.diff(rp).max() > 112
            assert kc.N_ROWS - (kc.SEGS - 1) * kc.SEG_ROWS < kc.SEG_ROWS
        if L == 1:
            assert arrs[0]["colidx"].max() >= 32768
