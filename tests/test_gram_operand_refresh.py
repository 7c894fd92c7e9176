"""The CSR Gram's e4m3 operand is written by a separate pass from sqrt(d) of the current point before every build.  A pass that
is skipped, or that runs before K1 has rewritten sqrt(d), leaves the bytes of an earlier point: the Hessian is then stale, which
only slows the solver's convergence and so escapes the parity tests.  These tests build two Hessians at different points in one
session and check the second against an emulation at the second point."""
import os
import sys

import numpy as np
import pytest

from oracle import oracle as orc

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gram_reference import e4m3_round  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def mb():
    import mlease_b200
    return mlease_b200


def _problem(n, d, seed):
    rng = np.random.default_rng(seed)
    X = (rng.normal(size=(n, d)) * (rng.random((n, d)) < 0.05)).astype(np.float32)
    y = (rng.random(n) < 0.4).astype(np.int32)
    w = rng.uniform(0.5, 2.0, n).astype(np.float32)
    o = rng.normal(0, 0.1, n).astype(np.float32)
    rp = np.concatenate([[0], np.cumsum((X != 0).sum(1))]).astype(np.int64)
    rows, cols = np.nonzero(X)
    return X, y, w, o, rp, cols.astype(np.int32), X[rows, cols].astype(np.float32)


def _expected(X, w, o, v, wv):
    """The library's Hessian at wv: the e4m3-rounded scaled rows' Gram plus the oracle's prior term."""
    n = X.shape[0]
    Xb = np.hstack([X.astype(np.float64), np.ones((n, 1))])
    p = 1.0 / (1.0 + np.exp(-(Xb @ wv + o)))
    dd = w * p * (1 - p)
    sd = np.sqrt(dd).astype(np.float32)
    amax = 0.5 * np.sqrt(np.float32(w.max())) * max(float(np.abs(v).max()), 1.0)
    g = 2.0 ** (np.frexp(np.float32(224.0) / np.float32(amax))[1] - 1)   # the library's power-of-two operand scale
    Xt = e4m3_round((Xb.astype(np.float32) * (sd * np.float32(g))[:, None]).astype(np.float32)) / g
    return Xt.T @ Xt


def test_csr_hessian_follows_the_point(mb):
    n, d = 3000, 300
    X, y, w, o, rp, ci, v = _problem(n, d, seed=11)
    rng = np.random.default_rng(4)
    pm = np.zeros(d + 1); pv = np.full(d + 1, 0.5)
    w1 = np.zeros(d + 1)
    w2 = rng.normal(0, 0.8, d + 1)
    with mb.AdmmSession(1, d, [1.0]) as s:
        s.add_partition_csr(0, rp, ci, v, y, w, o)
        _, _, H1 = s.objective(0, w1, pm, 1.0 / pv, want_hessian=True, tensor=True)
        _, _, H2 = s.objective(0, w2, pm, 1.0 / pv, want_hessian=True, tensor=True)
        _, _, H2_again = s.objective(0, w2, pm, 1.0 / pv, want_hessian=True, tensor=True)
    data = orc.Csr(rp, ci, v, y, w, o, d)
    H_ref = orc.objective("hessian", data, w2, pm, pv)
    scale = np.abs(H_ref).max()
    Xb = np.hstack([X.astype(np.float64), np.ones((n, 1))])
    p = 1.0 / (1.0 + np.exp(-(Xb @ w2 + o)))
    prior = H_ref - (Xb * (w * p * (1 - p))[:, None]).T @ Xb
    G1 = _expected(X, w, o, v, w1)
    G2 = _expected(X, w, o, v, w2)
    assert np.abs(G1 - G2).max() / scale > 1e-2   # the two points are far apart: a stale operand cannot pass the checks below
    e_emu = np.abs(H2 - (G2 + prior)).max() / scale
    e_ref = np.abs(H2 - H_ref).max() / scale
    assert e_emu < 1e-3, ("wgmma vs e4m3 emulation at the second point", e_emu)
    assert e_ref < 2e-2, ("wgmma vs oracle", e_ref)
    assert np.array_equal(H2, H2_again)
    assert not np.array_equal(H1, H2)
