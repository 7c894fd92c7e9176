"""CPU self-tests of chol_reference: the exact systems cover every tiling of the explicit-inverse Cholesky and have the outputs the
reference claims, a one-ulp change at a tile edge breaks the bitwise comparison, and the real-Hessian bounds hold for a correct
fp64 factorisation but not for one with a seeded fault."""
import os
import sys

import numpy as np
import pytest
import scipy.linalg as sla

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import chol_reference as cr  # noqa: E402
from factored_reference import ldh_of  # noqa: E402

WIDTHS = [1, 30, 31, 32, 63, 64, 200, 991, 992, 1023, 1024, 1300, 2047]


@pytest.mark.parametrize("D", WIDTHS)
def test_coverage_and_exact_outputs(D):
    Dt = D + 1
    pairs = cr.chol_pairs(Dt)
    cr.assert_coverage(Dt, pairs)
    E, H = cr.exact_system(Dt, pairs)
    assert not (E @ E).any()
    ex = cr.exact_outputs(E)
    ldh = ldh_of(Dt)
    assert np.array_equal(ex["L"] @ ex["L"].T, H)
    Hp = np.eye(ldh)
    Hp[:Dt, :Dt] = H
    assert np.array_equal(ex["Y"] @ Hp @ ex["Y"].T, np.eye(ldh))
    assert np.array_equal(ex["Hinv"] @ Hp, np.eye(ldh))
    if D >= 200:
        # off-diagonal E^T E (rows with two entries) and E E^T (columns with two entries) really reach Hinv and H
        EtE, EEt = E.T @ E, E @ E.T
        assert (EtE - np.diag(np.diag(EtE))).any() and (EEt - np.diag(np.diag(EEt))).any()


@pytest.mark.parametrize("D", [200, 1024])
def test_one_ulp_at_a_tile_edge_breaks_the_exact_comparison(D):
    Dt = D + 1
    E, _ = cr.exact_system(Dt, cr.chol_pairs(Dt))
    ex = cr.exact_outputs(E)
    for key, (i, j) in (("L", (64, 63)), ("Y", (128, 127)), ("Hinv", (63, 64)), ("Ldinv", (Dt - 1, 0))):
        bad = ex[key].copy()
        bad[i, j] = np.nextafter(bad[i, j], np.inf)
        assert not cr.same_bits(bad, ex[key]), key
    assert cr.same_bits(-0.0 * ex["Y"], 0.0 * ex["Y"])   # the sign of a zero is not a difference


def _spd(n, seed):
    r = np.random.default_rng(seed)
    X = r.normal(size=(n, 3 * n)) * r.uniform(0.5, 2.0, (n, 1))
    return X @ X.T / (3 * n) + np.diag(r.uniform(0.1, 2.0, n))


def _ldinv(L, ldh):
    Lp = np.eye(ldh)
    Lp[:L.shape[0], :L.shape[0]] = L
    out = np.zeros((ldh, 32))
    for k0 in range(0, ldh, 32):
        out[k0:k0 + 32] = sla.solve_triangular(Lp[k0:k0 + 32, k0:k0 + 32], np.eye(32), lower=True)
    return out


@pytest.mark.parametrize("Dt", [201, 1025])
def test_bounds_hold_for_fp64_and_catch_faults(Dt):
    H = _spd(Dt, Dt)
    ldh = ldh_of(Dt)
    L = np.linalg.cholesky(H)
    Yd = sla.solve_triangular(L, np.eye(Dt), lower=True)
    Y = np.eye(ldh)
    Y[:Dt, :Dt] = Yd
    Hi = Y.T @ Y
    assert cr.factor_excess(H, L) <= 1
    assert cr.inverse_excess(L, Y, _ldinv(L, ldh)) <= 1
    assert cr.hinv_excess(Y, Hi) <= 1
    # seeded faults: one factor entry off by 1e-9 relative, a dropped row-block product in Y, a Hinv tile from the wrong column
    Lb = L.copy()
    Lb[Dt - 1, 64] *= 1 + 1e-9
    assert cr.factor_excess(H, Lb) > 1
    Yb = Y.copy()
    Yb[64:96, :32] = 0.0
    assert cr.inverse_excess(L, Yb, _ldinv(L, ldh)) > 1
    Hb = Hi.copy()
    Hb[64:128, 0:64] = Hi[64:128, 64:128]
    assert cr.hinv_excess(Y, Hb) > 1


def _ring(Dt, H, seed):
    """(g, S, Y, rho): a gradient and a full ring of secant pairs with y = H s + noise (s . y > 0)."""
    r = np.random.default_rng(seed)
    S = r.normal(size=(cr.BFGS_M, Dt)) * 0.1
    Y = S @ H + 1e-3 * r.normal(size=(cr.BFGS_M, Dt))
    rho = 1.0 / np.einsum("jk,jk->j", S, Y)
    assert (rho > 0).all()
    return r.normal(size=Dt), S, Y, rho


@pytest.mark.parametrize("count,h0", [(0, 1.0), (1, 2.5), (6, 1.0), (7, 2.5), (13, 2.5)])
def test_two_loop_bound_holds_and_catches_faults(count, h0):
    Dt = 201
    H = _spd(Dt, 3)
    Hinv = np.linalg.inv(H)
    g, S, Y, rho = _ring(Dt, H, count)
    ref, bound = cr.two_loop(Hinv, g, S, Y, rho, count, h0)
    emu, _ = cr.two_loop(Hinv, g, S, Y, rho, count, h0, dtype=np.float64)   # the kernels' order in fp64
    assert cr._excess(emu - ref, bound) <= 1
    assert ref @ g < 0   # a descent direction
    ed, ep, en = cr.direction_excess(emu, emu @ g, np.abs(emu).max(), g, ref, bound)
    assert max(ed, ep, en) <= 1
    for fault in ("slot", "reverse", "h0_first"):
        bad, _ = cr.two_loop(Hinv, g, S, Y, rho, count, h0, dtype=np.float64, fault=fault)
        caught = cr._excess(bad - ref, bound) > 1
        # each fault changes the direction only where it has something to act on
        if fault == "slot" and count >= 1 or fault == "reverse" and min(count, cr.BFGS_M) >= 2 or fault == "h0_first" and count >= 1 and h0 != 1.0:
            assert caught, fault
