"""CPU tests of the consensus-step replica (consensus_reference.py): hand-computed float/double cases of the z-weights, the L1
threshold and its band edges, the rho schedule and the diff's NaN rule, and the replica against the oracle's ADMM driver
(oracle.admm_run)."""
import math
import os
import struct
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import consensus_reference as cr  # noqa: E402


def fl(x):
    """Round a Python double to float32 through struct (independent of numpy): a float32 +, -, *, / of two floats equals the rounded
    double result, since a double holds the exact result to more than 2 * 24 + 2 bits."""
    return struct.unpack("f", struct.pack("f", x))[0]


def test_z_weights_float_arithmetic():
    # P = 3, rho = 0.1, lambda = 0.7: weight = float(pr / (lambda + pr)) with pr = float(3 * rho)
    P, lam, rho = 3, 0.7, 0.1
    pr = fl(fl(3.0) * fl(rho))
    w_float = fl(pr / fl(fl(lam) + pr))
    w_double = P * fl(rho) / (fl(lam) + P * fl(rho))
    assert w_float != w_double                      # the case separates the two arithmetics
    wz = cr.z_weights(P, [lam], [rho], Dg=4, ldx=8)
    assert wz[0, 0] == w_float and wz[0, 3] == w_float
    assert wz[0, 4] == 1.0 and not wz[0, 5:].any()   # unpenalised intercept, zero padding
    assert cr.z_weights(P, [lam], [rho], Dg=4, ldx=8, penalize_intercept=True)[0, 4] == w_float
    # lambda.map: float sum, double division; entries <= 0 keep the lambda's weight
    lm = [1.3, 0.0, -2.0, 5.5]
    wz = cr.z_weights(P, [lam], [rho], Dg=4, ldx=8, lambda_map=lm)
    w0 = pr / (fl(fl(1.3) + pr) + 0.0)
    assert wz[0, 0] == w0 and w0 != pr / (fl(1.3) + pr) and w0 != fl(pr / fl(fl(1.3) + pr))
    assert wz[0, 1] == w_float and wz[0, 2] == w_float
    assert wz[0, 3] == pr / (fl(fl(5.5) + pr) + 0.0)


def test_l1_threshold_float_product():
    P, lam, rho = 7, 0.3, 0.1
    t = cr.l1_thresholds(P, [lam], [rho])[0]
    assert t == fl(lam) / (fl(fl(rho) * 7.0) + 0.0)
    assert t != fl(lam) / (fl(rho) * 7.0)


def _state(L, Dt, ldx, nlocal, rng):
    nprob = nlocal * L
    return dict(vec=rng.normal(size=(nprob, 5, ldx)), fvec=rng.normal(size=(nprob, 3, ldx)).astype(np.float32), z=rng.normal(size=(L, ldx)),
                exch=rng.normal(size=L * Dt + 1), diff=np.full(L, -1.0), ctrl=np.full((nprob, 3), 5, np.int32))


def test_l1_band_edges_and_intercept():
    P, Dt, ldx = 4, 6, 8
    t = cr.l1_thresholds(P, [0.9], [1.0])[0]
    st = _state(1, Dt, ldx, 1, np.random.default_rng(0))
    up = np.nextafter(t, np.inf)
    # S / P with P = 4 is exact: the means are t, -t, one ulp outside each, 0, and a large intercept
    means = np.array([t, -t, up, -up, 0.0, 1e3])
    st["exch"][:Dt] = means * P
    out = cr.consensus(st, 1, Dt, P, 1, None, [1.0], l1thr=[t])
    z = out["z"][0, :Dt]
    assert z[0] == t and z[1] == -t                        # strict > / <: the band edge stays
    assert z[2] == up - t and z[3] == -up + t and z[2] > 0  # one ulp outside is thresholded
    assert z[4] == 0.0 and z[5] == 1e3                     # the intercept is never thresholded
    assert (out["z"][0, Dt:] == st["z"][0, Dt:]).all() and out["exch"][-1] == st["exch"][-1]


def test_rho_schedule():
    assert cr.rho_eff(1.0, 1) == 1.0 and cr.rho_eff(2.5, 3) == float(np.float32(2.5))
    assert cr.rho_eff(0.1, 1, boost_rate=3.0) == fl(0.1) * 3.0 and cr.rho_eff(0.1, 2, boost_rate=3.0) == fl(0.1)
    for i in (2, 3, 7):
        assert cr.rho_eff(0.1, i, coef=0.25) == fl(0.1) * fl(math.exp(fl(-(i - 1) * fl(0.25))))
    # the exponential is double (Math.exp) of the float product: at coefficient 0.289, iteration 2, float's expf would round the
    # other way (0.74901223f)
    assert cr.rho_rate(2, coef=0.289) == np.float32(0.7490122) != np.float32(0.74901223)
    assert cr.rho_eff(1.0, 2, coef=0.289) == float(np.float32(0.7490122))


def test_diff_nan_rule():
    assert cr.max_abs_diff([1.0, np.nan, -3.0, 2.0]) == 3.0          # a NaN coefficient is skipped
    assert np.isnan(cr.max_abs_diff([1.0, 5.0, np.nan]))             # a NaN intercept is the diff
    assert cr.max_abs_diff([np.nan, np.nan, 0.5]) == 0.5
    assert cr.max_abs_diff([np.inf, 1.0]) == np.inf
    # a NaN diff moves neither maxdiff nor mindiff
    assert cr.finish([np.nan, 2e-5], 1e-6, 1e-4) == (2e-5, 2e-5, 1)
    assert cr.finish([np.nan], 1e-6, 1e-4) == (0.0, 99999999.0, 1)
    assert cr.finish([3e-4, 1e-5], 1e-6, 1e-4)[2] == 0 and cr.finish([1e-5], 1e-4, 1e-4)[2] == 0
    assert cr.finish([1e-5], 1e-5, -1.0)[2] == 1                     # epsilon < 0: the default 1e-4


def test_pack_and_consensus_by_hand():
    """One lambda, two local partitions of P = 3, Dt = 2: every output by hand."""
    L, Dt, ldx, P = 1, 2, 4, 3
    st = _state(L, Dt, ldx, 2, np.random.default_rng(1))
    st["vec"][0, cr.BETA, :Dt] = [0.1, 1.0 / 3.0]
    st["vec"][1, cr.BETA, :Dt] = [0.2, -0.5]
    st["fvec"][0, cr.UF, :Dt] = [0.25, 0.0]
    st["fvec"][1, cr.UF, :Dt] = [-0.125, 1.0]
    out = cr.pack(st, L, Dt, 2)
    for b, (x, u) in enumerate([([0.1, 1 / 3], [0.25, 0.0]), ([0.2, -0.5], [-0.125, 1.0])]):
        assert out["fvec"][b, cr.XF, :Dt].tolist() == [fl(v) for v in x]
        assert out["fvec"][b, cr.UPX, :Dt].tolist() == [fl(a + b_) for a, b_ in zip(u, x)]
        assert out["vec"][b, cr.XD, :Dt].tolist() == x
    S = [0.0 + (fl(0.1) + 0.25) + (fl(0.2) - 0.125), 0.0 + (fl(1 / 3) + 0.0) + (-0.5 + 1.0)]
    assert out["exch"][:Dt].tolist() == S and out["exch"][Dt] == st["exch"][Dt]
    assert (out["fvec"][:, :, Dt:] == st["fvec"][:, :, Dt:]).all() and (out["vec"][:, :, Dt:] == st["vec"][:, :, Dt:]).all()
    wz = cr.z_weights(P, [1.0], [1.0], Dt - 1, ldx)
    c = cr.consensus(out, L, Dt, P, 2, wz, [0.75], fused=True)
    zn = [wz[0, 0] * (S[0] * (1 / 3)), 1.0 * (S[1] * (1 / 3))]
    assert c["z"][0, :Dt].tolist() == zn
    assert c["diff"][0] == max(abs(out["z"][0, k] - zn[k]) for k in range(Dt))
    for b in range(2):
        upx = out["fvec"][b, cr.UPX, :Dt].astype(np.float64)
        un = [fl(upx[k] - zn[k]) for k in range(Dt)]
        assert c["fvec"][b, cr.UF, :Dt].tolist() == un
        assert c["vec"][b, cr.M, :Dt].tolist() == [fl(zn[k]) - un[k] for k in range(Dt)]
        q, x, m = out["vec"][b, cr.Q, :Dt], out["vec"][b, cr.XD, :Dt], out["vec"][b, cr.M, :Dt]
        assert c["vec"][b, cr.GT, :Dt].tolist() == [-q[k] * (x[k] - m[k]) for k in range(Dt)]
        assert c["vec"][b, cr.BETA, :Dt].tolist() == x.tolist() and (c["vec"][b, cr.Q, :Dt] == 0.75).all()
        assert c["ctrl"][b].tolist() == [5, 1, 0]
    # not fused: g_t and the flags are not written
    c2 = cr.consensus(out, L, Dt, P, 2, wz, [0.75], fused=False)
    assert (c2["vec"][:, cr.GT] == out["vec"][:, cr.GT]).all() and (c2["ctrl"] == out["ctrl"]).all()


def _csr_data(rng, P, n, D, nnz):
    from oracle import oracle as orc
    ci = np.stack([np.sort(rng.choice(D, nnz, replace=False)) for _ in range(P * n)]).astype(np.int32)
    v = rng.normal(size=(P * n, nnz)).astype(np.float32)
    bs = rng.normal(size=D) / np.sqrt(nnz)
    y = (rng.random(P * n) < 1 / (1 + np.exp(-((v * bs[ci]).sum(1) - 0.5)))).astype(np.int32)
    return orc.Csr(np.arange(P * n + 1, dtype=np.int64) * nnz, ci.reshape(-1), v.reshape(-1), y, n_features=D)


@pytest.mark.parametrize("case", ["l2", "l2_map_penalized", "l1"])
@pytest.mark.parametrize("N", [1, 3])
def test_replica_against_oracle_driver(case, N):
    """From the oracle's x, u and u + x of iteration N, the replica's pack and consensus give the oracle's z of iteration N and its
    diff.  Not bit for bit: the oracle forms xbar and ubar separately, (1/P) * term per partition, the device sums x + u first and
    multiplies the sum by 1/P.  Per entry both are within (2P + 6) roundings of relative 2^-53 of w * sum_p (|x_p| + |u_p|) / P of
    the exact value; the test allows twice that."""
    from oracle import oracle as orc
    rng = np.random.default_rng(11 + N)
    P, n, D = 3, 400, 24
    lambdas, rhos = [0.3, 2.0], [1.0, 0.7]
    data = _csr_data(rng, P, n, D, 5)
    kw = dict(regularizer=1 if case == "l1" else 2, penalize_intercept=case == "l2_map_penalized")
    lmap = None
    if case == "l2_map_penalized":
        lmap = np.abs(rng.normal(size=D)).astype(np.float32) * 3
        lmap[::5] = 0.0
        lmap[1] = -1.0
    r = orc.admm_run(data, [0, n, 2 * n, 3 * n], lambdas, rhos=rhos, niters=N, mode="exact", epsilon=0.0, lambda_map=lmap, **kw)
    assert r["iters_done"] == N
    L, Dt = len(lambdas), D + 1
    ldx = (Dt + 3) // 4 * 4
    nprob = P * L
    st = dict(vec=np.zeros((nprob, 5, ldx)), fvec=np.zeros((nprob, 3, ldx), np.float32), z=np.zeros((L, ldx)), exch=np.zeros(L * Dt + 1),
              diff=np.zeros(L), ctrl=np.zeros((nprob, 3), np.int32))
    for p in range(P):
        for l in range(L):
            st["vec"][p * L + l, cr.BETA, :Dt] = r["x_last"][p, l]
            st["fvec"][p * L + l, cr.UF, :Dt] = r["u_last"][p, l]
    if N > 1:
        st["z"][:, :Dt] = r["z_hist"][N - 2]
    st = cr.pack(st, L, Dt, P)
    for p in range(P):
        for l in range(L):
            assert (st["fvec"][p * L + l, cr.UPX, :Dt] == r["uplusx_last"][p, l]).all()   # uplusx is bitwise the oracle's
    wz = cr.z_weights(P, lambdas, rhos, D, ldx, lambda_map=lmap, penalize_intercept=kw["penalize_intercept"])
    thr = cr.l1_thresholds(P, lambdas, rhos) if case == "l1" else None
    out = cr.consensus(st, L, Dt, P, P, wz, [1.0] * L, l1thr=thr)
    for l in range(L):
        mag = sum(np.abs(r["x_last"][p, l].astype(np.float32).astype(np.float64)) + np.abs(r["u_last"][p, l].astype(np.float64))
                  for p in range(P)) / P
        w = np.ones(Dt) if case == "l1" else wz[l, :Dt]
        bound = 2 * (2 * P + 6) * 2.0 ** -53 * w * mag
        err = np.abs(out["z"][l, :Dt] - r["z_hist"][N - 1, l])
        assert (err <= bound).all(), (case, l, float((err / np.where(bound > 0, bound, 1)).max()))
        assert abs(out["diff"][l] - r["diff_hist"][N - 1, l]) <= bound.max(), (case, l)
        assert np.abs(r["z_hist"][N - 1, l]).max() > 1e-3   # (a nontrivial z)
