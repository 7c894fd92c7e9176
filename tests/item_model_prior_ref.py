"""fp64 replica of ItemModelTrain under per-key priors (mlease_item_model_train_prior) for the tests: each key's fits by the oracle's
LibLinear with the per-column prior mean and variance vectors that initSetup (llf/LibLinear.java:476-497) builds from the key's prior
list, and the union lists the library returns."""
import numpy as np

from oracle import oracle as orc


def usual_var(lam):
    """the variance the library reports for a column under lambda: 1 / q with q = 1 / (1 / lambda), in fp64"""
    return 1.0 / (1.0 / (1.0 / np.float64(np.float32(lam))))


def key_fits(pb, il, dl, lambda_map, prior, means=None, binary=False):
    """prior = (prior_ptr, prior_col, prior_mean, prior_var).  -> per key None (no rows) or a dict: cols (the union list, then D),
    listed [n] (the rows list the column; the intercept counts as listed), model [IL, DL, n] (the replica's fit at listed columns, the
    prior mean at prior-only ones), povar [IL, DL, n] (the variance of prior-only columns, NaN at listed ones), and per grid point the
    oracle's data, pm and pv to evaluate the Hessian diagonal at another fit."""
    D, K = pb["D"], pb["K"]
    pp, pc, pmn, pvr = (np.asarray(a) for a in prior)
    lm = np.zeros(D, np.float32) if lambda_map is None else np.asarray(lambda_map, np.float32)
    means = np.zeros(K) if means is None else np.asarray(means, np.float64)
    out = []
    for k in range(K):
        a, b = pb["krs"][k], pb["krs"][k + 1]
        if b == a:
            out.append(None)
            continue
        rp = pb["rp"][a:b + 1]
        v = np.ones(rp[-1] - rp[0], np.float32) if binary else pb["v"][rp[0]:rp[-1]]
        data = orc.Csr(rp - rp[0], pb["ci"][rp[0]:rp[-1]], v, pb["y"][a:b], pb["w"][a:b], pb["o"][a:b], D)
        lmask = np.zeros(D + 1, bool)
        lmask[np.unique(data.colidx)] = True
        lmask[D] = True
        e = np.arange(pp[k], pp[k + 1])
        po = e[~lmask[pc[e]]]                                   # prior-only entries
        cols = np.concatenate([np.union1d(np.nonzero(lmask[:D])[0], pc[po]), [D]]).astype(np.int64)
        n = len(cols)
        listed = lmask[cols]
        rec = dict(cols=cols, listed=listed, model=np.zeros((len(il), len(dl), n)), povar=np.full((len(il), len(dl), n), np.nan),
                   data=data, pm={}, pv={})
        at = {c: i for i, c in enumerate(cols)}
        for ia, lam_i in enumerate(il):
            for ib, lam_d in enumerate(dl):
                pv = np.where(lm > 0, 1.0 / np.where(lm > 0, lm, 1).astype(np.float64), 1.0 / np.float64(np.float32(lam_d)))
                pv = np.append(pv, 1.0 / np.float64(np.float32(lam_i)))
                pm = np.zeros(D + 1)
                pm[D] = means[k]
                for i in e:                                     # initSetup: an entry of a column the data lists
                    if lmask[pc[i]]:
                        pm[pc[i]] = pmn[i]
                        if pvr[i] > 0:
                            pv[pc[i]] = pvr[i]
                beta, _ = orc.liblinear_train(data, np.zeros(D + 1), pm, pv, 1e-14, 100000)
                rec["model"][ia, ib] = beta[cols]
                for i in po:
                    c = pc[i]
                    rec["model"][ia, ib, at[c]] = pmn[i]
                    rec["povar"][ia, ib, at[c]] = pvr[i] if pvr[i] > 0 else (usual_var(lm[c]) if lm[c] > 0 else usual_var(lam_d))
                rec["pm"][ia, ib], rec["pv"][ia, ib] = pm, pv
        out.append(rec)
    return out
