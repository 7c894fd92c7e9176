"""numpy replica of the ADMM consensus step (csrc/k4_consensus.cu) and of the host values it reads (session.cu), in the device's
exact operation order: every output is meant to equal the device's bit for bit (up to the sign of a zero and the payload of a NaN).

K4 is elementwise IEEE arithmetic.  Its only sum runs over the local partitions in the fixed order p = 0 .. nlocal - 1, the diff is
a max (exact in any order), and no product in it is followed by an add (so FMA contraction cannot change a bit).  The float32 steps
of the reference (jobs/RegressionAdmmTrain.java) are numpy float32 scalar operations here, which round like the device's.

State layout (that of the test hook mlease_internal_consensus): per problem b = local partition * L + lambda, vec [nprob, 5, ldx]
(beta, m, q, g_t, x_d), fvec [nprob, 3, ldx] float32 (u_f, uplusx_f, x_f), ctrl [nprob, 3] (hess_valid, skip_eval, k1_chunks); per
lambda z [L, ldx], the exchange exch [L Dt + 1] (the last slot is the failed-fit count, which K4 never touches) and diff [L]."""
import math

import numpy as np

f32 = np.float32
BETA, M, Q, GT, XD = range(5)
UF, UPX, XF = range(3)
HESS_VALID, SKIP_EVAL, K1_CHUNKS = range(3)


def z_weights(P, lambdas, rhos, Dg, ldx, lambda_map=None, penalize_intercept=False):
    """wz [L, ldx] as finalize() builds it (:381-386, :392-403): pr = float(P) * rho in float, weight = double(float(pr / (lambda + pr)));
    a lambda.map entry > 0 gives double(pr) / (double(float(lambda_k + pr)) + 0.0) (entries <= 0 are ignored); the intercept weight is
    1, or `weight` under penalize_intercept; the padding is 0."""
    L = len(lambdas)
    wz = np.zeros((L, ldx))
    for l in range(L):
        lf, rf = f32(lambdas[l]), f32(rhos[l])
        pr = f32(f32(P) * rf)
        weight = float(f32(pr / f32(lf + pr)))
        for k in range(Dg):
            w = weight
            if lambda_map is not None and f32(lambda_map[k]) > 0:
                w = float(pr) / (float(f32(f32(lambda_map[k]) + pr)) + 0.0)
            wz[l, k] = w
        wz[l, Dg] = weight if penalize_intercept else 1.0
    return wz


def l1_thresholds(P, lambdas, rhos):
    """The L1 soft threshold per lambda (:409): double(lambda) / (double(float(rho * float(P))) + 0.0)."""
    return np.array([float(f32(lam)) / (float(f32(f32(r) * f32(P))) + 0.0) for lam, r in zip(lambdas, rhos)])


def rho_rate(i, boost_rate=0.0, coef=0.0):
    """rho.adapt.rate the reducers of iteration i see (float): the boost at iteration 1 (begin_initialized), then
    float(Math.exp(float(-(i - 1) * coef))) for i > 1 when the coefficient is > 0 (:313-316, :323-327).  The exponential is double
    (math.exp), of the float product."""
    rate = f32(boost_rate) if (i == 1 and f32(boost_rate) > 0) else f32(1.0)
    if i > 1 and f32(coef) > 0:
        rate = f32(math.exp(float(f32(f32(-(i - 1)) * f32(coef)))))
    return rate


def rho_eff(rho, i, boost_rate=0.0, coef=0.0):
    """The prior precision of iteration i: double(float rho), times the rate when it is not 1 (:652-658)."""
    r = float(f32(rho))
    rate = rho_rate(i, boost_rate, coef)
    if rate != f32(1.0):
        r = r * float(rate)
    return r


def _copy(st):
    return {k: np.array(v, copy=True) for k, v in st.items()}


def reset(st, L, Dt, rho1):
    """admm_reset: every vector of every problem 0 over the whole ldx (q: rho of iteration 1 on [0, Dt), 1 on the padding), z of
    every lambda 0 over the whole ldx (written by the problems of local partition 0), hess_valid = skip_eval = 0."""
    st = _copy(st)
    nprob, _, ldx = st["vec"].shape
    for b in range(nprob):
        l = b % L
        st["vec"][b, [BETA, M, XD]] = 0.0   # (g_t is not reset)
        st["fvec"][b] = 0.0
        st["vec"][b, Q, :Dt] = rho1[l]
        st["vec"][b, Q, Dt:] = 1.0
        st["ctrl"][b, HESS_VALID] = 0
        st["ctrl"][b, SKIP_EVAL] = 0
    st["z"][:] = 0.0
    return st


def init(st, L, Dt):
    """admm_init: m = beta = double(float(z)) on [0, Dt) (the reducers read z as float, u is the empty map)."""
    st = _copy(st)
    for b in range(st["vec"].shape[0]):
        zf = st["z"][b % L, :Dt].astype(f32).astype(np.float64)
        st["vec"][b, M, :Dt] = zf
        st["vec"][b, BETA, :Dt] = zf
    return st


def pack(st, L, Dt, nlocal):
    """admm_pack: per problem x_f = float(beta), x_d = beta, uplusx_f = float(double(u_f) + beta); per lambda the exchange
    S[l][k] = 0.0 + (double(x_f) + double(u_f)) summed over the local partitions in order."""
    st = _copy(st)
    vec, fvec = st["vec"], st["fvec"]
    for l in range(L):
        s = np.zeros(Dt)
        for p in range(nlocal):
            b = p * L + l
            x = vec[b, BETA, :Dt].copy()
            xf = x.astype(f32)
            uf = fvec[b, UF, :Dt].copy()
            fvec[b, XF, :Dt] = xf
            vec[b, XD, :Dt] = x
            fvec[b, UPX, :Dt] = (uf.astype(np.float64) + x).astype(f32)
            s = s + (xf.astype(np.float64) + uf.astype(np.float64))
        st["exch"][l * Dt:(l + 1) * Dt] = s
    return st


def max_abs_diff(d):
    """LinearModel.maxAbsValue of z_prev - z (models/LinearModel.java:728-740): starts from |intercept| (the last entry) and takes a
    coefficient only when `maxabs < v` -- a NaN coefficient is skipped, a NaN intercept is the answer."""
    d = np.abs(np.asarray(d, np.float64))
    m = d[-1]
    for v in d[:-1]:
        if m < v:
            m = v
    return m


def consensus(st, L, Dt, P, nlocal, wz, rho_next, l1thr=None, fused=False):
    """admm_consensus_kernel on the summed exchange (the launcher zeroes diff first).  Per lambda and k < Dt: zn = wz * (S * (1/P))
    (L2), or S * (1/P) soft-thresholded by strict comparisons except at the intercept column Dt - 1 (L1); diff = |z - zn| reduced as
    maxAbsValue; z = zn.  Per local problem: u_f = float(double(uplusx_f) - zn); on fused batches g_t = -q_old (x_d - m_old), the
    data-term gradient at x_d estimated from the OLD prior; m = double(float(zn)) - double(u_f); beta = x_d; q = rho_next.  Fused
    batches also get skip_eval = 1, k1_chunks = 0.  Returns the new state (diff filled in)."""
    st = _copy(st)
    vec, fvec, z = st["vec"], st["fvec"], st["z"]
    invP = 1.0 / float(P)
    for l in range(L):
        S = st["exch"][l * Dt:(l + 1) * Dt]
        if l1thr is not None:
            zn = S * invP
            t = float(l1thr[l])
            c = zn[:Dt - 1].copy()
            c = np.where(c > t, c - t, np.where(c < -t, c + t, c))
            zn = np.concatenate([c, zn[Dt - 1:]])
        else:
            zn = wz[l, :Dt] * (S * invP)
        with np.errstate(invalid="ignore"):
            st["diff"][l] = max_abs_diff(z[l, :Dt] - zn)
        z[l, :Dt] = zn
        zf = zn.astype(f32).astype(np.float64)
        for p in range(nlocal):
            b = p * L + l
            with np.errstate(invalid="ignore", over="ignore"):
                un = (fvec[b, UPX, :Dt].astype(np.float64) - zn).astype(f32)
                fvec[b, UF, :Dt] = un
                if fused:
                    vec[b, GT, :Dt] = -vec[b, Q, :Dt] * (vec[b, XD, :Dt] - vec[b, M, :Dt])
                vec[b, M, :Dt] = -1.0 * un.astype(np.float64) + 1.0 * zf
            vec[b, BETA, :Dt] = vec[b, XD, :Dt]
            vec[b, Q, :Dt] = rho_next[l]
            if fused:
                st["ctrl"][b, SKIP_EVAL] = 1
                st["ctrl"][b, K1_CHUNKS] = 0
    return st


def finish(diff, liblinear_eps, epsilon):
    """consensus_finish: maxdiff / mindiff over the lambdas with the reference's `maxdiff < diff` / `mindiff > diff` (a NaN diff
    changes neither), stop = maxdiff < epsilon (default 1e-4 when epsilon < 0) and liblinear_eps <= 1e-5 (:456-472, :493-496)."""
    mx, mn = 0.0, 99999999.0
    for d in diff:
        if mx < d:
            mx = float(d)
        if mn > d:
            mn = float(d)
    eps = epsilon if epsilon >= 0 else 0.0001
    return mx, mn, int(mx < eps and float(f32(liblinear_eps)) <= 0.00001)
