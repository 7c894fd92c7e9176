"""fp64 numpy reference of mlease_test_auc: the weighted Mann-Whitney statistic, tied pairs counting 1/2, computed exactly as the
header defines it -- runs r of equal pred in ascending order, P_r / N_r their positive / negative weight, Nb_r the negative weight
of the runs below, U = sum_r P_r (Nb_r + N_r / 2), auc = U / (P N), NaN when P or N is 0."""
import numpy as np


def segment_upn(response, pred, weight=None):
    """(U, P, N) of one segment: rows with response 1 are positive, 0 and -1 negative; weight None means 1."""
    r = np.asarray(response)
    p = np.asarray(pred, np.float32).astype(np.float64) + 0.0   # -0.0 + 0.0 = +0.0: the two zeros tie
    w = np.ones(len(r)) if weight is None else np.asarray(weight, np.float32).astype(np.float64)
    if len(r) == 0:
        return 0.0, 0.0, 0.0
    order = np.argsort(p, kind="stable")
    ps, pos, ws = p[order], r[order] == 1, w[order]
    head = np.r_[True, ps[1:] != ps[:-1]]
    run = np.cumsum(head) - 1
    P_r = np.bincount(run, weights=np.where(pos, ws, 0.0))
    N_r = np.bincount(run, weights=np.where(pos, 0.0, ws))
    Nb_r = np.r_[0.0, np.cumsum(N_r)[:-1]]
    return float(np.sum(P_r * (Nb_r + 0.5 * N_r))), float(P_r.sum()), float(N_r.sum())


def auc_of(U, P, N):
    return U / (P * N) if P > 0 and N > 0 else float("nan")


def test_auc_ref(response, pred, weight=None, key_rowstart=None):
    """mlease_test_auc's outputs: (auc [S], weight [2], key_auc [S, K] or None, key_weight [K, 2] or None)."""
    pred = np.atleast_2d(np.asarray(pred, np.float32))
    response = np.asarray(response)
    S = pred.shape[0]
    auc = np.array([auc_of(*segment_upn(response, pred[s], weight)) for s in range(S)])
    _, P, N = segment_upn(response, pred[0], weight)
    wt = np.array([P, N])
    if key_rowstart is None:
        return auc, wt, None, None
    krs = np.asarray(key_rowstart, np.int64)
    K = len(krs) - 1
    kauc = np.full((S, K), np.nan)
    kw = np.zeros((K, 2))
    for k in range(K):
        a, b = krs[k], krs[k + 1]
        wk = None if weight is None else np.asarray(weight)[a:b]
        for s in range(S):
            kauc[s, k] = auc_of(*segment_upn(response[a:b], pred[s, a:b], wk))
        _, kw[k, 0], kw[k, 1] = segment_upn(response[a:b], pred[0, a:b], wk)
    return auc, wt, kauc, kw


test_auc_ref.__test__ = False


def brute_force_auc(response, pred, weight=None):
    """auc by enumerating every (positive, negative) pair: 1 when the positive scores higher, 1/2 on a tie."""
    r = np.asarray(response)
    p = np.asarray(pred, np.float32).astype(np.float64)
    w = np.ones(len(r)) if weight is None else np.asarray(weight, np.float64)
    U = P = N = 0.0
    for i in range(len(r)):
        if r[i] == 1:
            P += w[i]
        else:
            N += w[i]
    for i in range(len(r)):
        if r[i] != 1:
            continue
        for j in range(len(r)):
            if r[j] == 1:
                continue
            U += w[i] * w[j] * (1.0 if p[i] > p[j] else 0.5 if p[i] == p[j] else 0.0)
    return auc_of(U, P, N)
