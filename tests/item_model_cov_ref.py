"""fp64 numpy references for the full posterior of ItemModelTrain's per-key fits (LibLinear.train with computeFullPostVar,
llf/LibLinear.java:315-326): the exact Hessian of a key's fit over its list, its inverse by Cholesky, the bound the GPU's inverse
is held to, and the packed lower-triangle layout of mlease_item_model_train_cov."""
import numpy as np

EPS64 = 2.0 ** -53


def key_rows(pb, k):
    """the rows of key k: (rowptr from 0, colidx, vals, response, weight, offset)"""
    a, b = pb["krs"][k], pb["krs"][k + 1]
    rp = pb["rp"][a:b + 1]
    return rp - rp[0], pb["ci"][rp[0]:rp[-1]], pb["v"][rp[0]:rp[-1]], pb["y"][a:b], pb["w"][a:b], pb["o"][a:b]


def prior_precision(cols, D, lambda_map, il, dl):
    """q over a list (global columns, D = the intercept) as the fit builds it: 1/(1/lambda) of lambda_map's entry > 0, else of the
    default lambda; the intercept's of the intercept lambda (all lambdas float32)"""
    lm = np.zeros(D, np.float32) if lambda_map is None else np.asarray(lambda_map, np.float32)
    q = np.empty(len(cols))
    for i, c in enumerate(cols):
        lam = np.float32(il) if c == D else (lm[c] if lm[c] > 0 else np.float32(dl))
        q[i] = 1.0 / (1.0 / np.float64(lam))
    return q


def hessian(pb, k, cols, beta, q, binary=False):
    """H = diag(q) + sum_i w_i p_i (1-p_i) x_i x_i^T over the list cols (ascending, the intercept D last, x = 1 there) at beta (the
    list's coefficients, float64), p_i = 1 / (1 + exp(-y_i (x_i . beta + o_i))), y = +-1"""
    rp, ci, v, y, w, o = key_rows(pb, k)
    n, m = len(y), len(cols)
    X = np.zeros((n, m))
    for i in range(n):
        pos = np.searchsorted(cols, ci[rp[i]:rp[i + 1]])
        X[i, pos] = 1.0 if binary else v[rp[i]:rp[i + 1]].astype(np.float64)
    X[:, m - 1] = 1.0
    s = X @ beta + o.astype(np.float64)
    yy = np.where(y == 1, 1.0, -1.0)
    p = 1.0 / (1.0 + np.exp(-yy * s))
    d = w.astype(np.float64) * p * (1.0 - p)
    return np.diag(q) + (X * d[:, None]).T @ X


def inverse(H):
    """Sigma = H^-1 by Cholesky, and the 2-norm condition number of H"""
    L = np.linalg.cholesky(H)
    Li = np.linalg.solve(L, np.eye(len(H)))
    ev = np.linalg.eigvalsh(H)
    return Li.T @ Li, ev[-1] / ev[0]


def sigma_bound(H, sigma, c=8.0):
    """entrywise bound on the GPU's Sigma from fp64 Cholesky and an explicit inverse: c * Dt * kappa_2(H) * 2^-53 * max |Sigma|"""
    _, kappa = inverse(H)
    return c * len(H) * kappa * EPS64 * np.abs(sigma).max()


def unpack(block, n):
    """the packed lower triangle (row-major, entry (a, b) at a(a+1)/2 + b) as a symmetric n x n matrix"""
    assert len(block) == n * (n + 1) // 2
    S = np.zeros((n, n))
    S[np.tril_indices(n)] = block
    return S + np.tril(S, -1).T
