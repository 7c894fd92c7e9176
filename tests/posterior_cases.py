"""Seeded inputs of the ADMM posterior and of predictive-variance scoring whose structure reaches the branches the kernels take only
above a size, with their fp64 references.

postvar_hess_col_kernel (csrc/k6_postvar.cu) walks a column's rows HC_STAGE positions at a time and its cells HC_CELLS at a time:
  - the stage case lists designated columns of one partition in exactly 1, 255, 256, 257, 511, 512 and 513 rows and one column in
    every row, beside a partition with no stored entry (its rows hold the intercept alone) and one with empty rows;
  - the window cases (D' = 12 288, 12 289, 12 290, 24 601) list only an active set S clustered at the window edges, so H is block
    diagonal: one block on S and the intercept, diag(q) on every empty column, and Sigma is known in closed form from the block's
    inverse.  Rows list pairs at distances 12 287, 12 288 and >= 24 576 where the width allows them.
score_var_kernel and score_keyed_cov_kernel (csrc/k5_score.cu) walk a record's entry pairs in COV_TILE-entry tiles; the long records
hold 1, 255, 256, 257, 512, 513 and 1 100 entries.

Shared conventions: float32 values, y in {0, 1}, weights in [0.5, 2] with some rows at exactly 0, offsets ~ N(0, 0.1), sorted unique
columns per row.  A partition is (rowptr, cols, vals, y, w, o) as test_gpu_admm_posterior builds them."""
import math

import numpy as np
import scipy.sparse as sp

EPS = 2.0 ** -53
HC_STAGE = 256       # postvar_hess_col_kernel: column positions staged per step
HC_CELLS = 12288     # postvar_hess_col_kernel: fp64 cells of a column window
COV_TILE = 256       # score_var_kernel, score_keyed_cov_kernel: entries of a pair tile
STAGE_COUNTS = (1, 255, 256, 257, 511, 512, 513)
WINDOW_WIDTHS = (12288, 12289, 12290, 24601)
RECORD_LENS = (1, 255, 256, 257, 512, 513, 1100)


def _labels(rng, n, zero_w=()):
    y = np.where(rng.random(n) < 0.4, 1, 0).astype(np.int32)
    w = rng.uniform(0.5, 2.0, n).astype(np.float32)
    w[list(zero_w)] = 0.0
    o = rng.normal(0, 0.1, n).astype(np.float32)
    return y, w, o


def _csr(rng, rows):
    rowptr = np.zeros(len(rows) + 1, np.int64)
    rowptr[1:] = np.cumsum([len(r) for r in rows])
    cols = np.concatenate([np.asarray(r, np.int64) for r in rows] + [np.zeros(0, np.int64)]).astype(np.int32)
    vals = rng.normal(0, 1, len(cols)).astype(np.float32)
    return rowptr, cols, vals


def _lambda_map(rng, Dg, k):
    lm = np.zeros(Dg, np.float32)
    lm[rng.choice(Dg, k, replace=False)] = rng.uniform(0.2, 5.0, k).astype(np.float32)
    return lm


def stage_case(seed=0):
    """D' = 700 over three partitions.  Partition 0 (1 100 rows): column stage_cols[k] listed by exactly STAGE_COUNTS[k] rows, column
    all_col by every row, three filler columns per row on average; its rows of weight 0 hold no stage-two position.  Partition 1:
    60 rows and no stored entry.  Partition 2: 400 rows, every third one empty."""
    rng = np.random.default_rng(7000 + seed)
    Dg, n0 = 699, 1100
    stage_cols = (31, 32, 95, 96, 350, 351, 697)
    all_col = 698
    designated = set(stage_cols) | {all_col}
    filler = np.array([c for c in range(Dg) if c not in designated])
    rows = [set() for _ in range(n0)]
    stage_two = set()
    for c, k in zip(stage_cols, STAGE_COUNTS):
        rs = np.sort(rng.choice(n0, k, replace=False))
        for r in rs:
            rows[r].add(c)
        stage_two.update(rs[HC_STAGE:].tolist())
    for r in range(n0):
        rows[r].add(all_col)
        rows[r].update(rng.choice(filler, rng.poisson(3), replace=False).tolist())
    stage_two.update(range(HC_STAGE, n0))   # all_col's stage-two rows
    zero_w = [r for r in rng.choice(n0, 60, replace=False) if r not in stage_two]
    p0 = _csr(rng, [sorted(r) for r in rows]) + _labels(rng, n0, zero_w)
    n1 = 60
    p1 = (np.zeros(n1 + 1, np.int64), np.zeros(0, np.int32), np.zeros(0, np.float32)) + _labels(rng, n1, range(0, n1, 13))
    n2 = 400
    rows2 = [[] if i % 3 == 0 else sorted(rng.choice(Dg, int(rng.integers(1, 12)), replace=False).tolist()) for i in range(n2)]
    p2 = _csr(rng, rows2) + _labels(rng, n2, range(1, n2, 17))
    return dict(name="stage", Dg=Dg, parts=[p0, p1, p2], z=rng.normal(0, 0.2, Dg + 1), lam=1.0,
                lambda_map=_lambda_map(rng, Dg, 40), stage_cols=stage_cols, all_col=all_col)


def window_edges(Dt):
    """the columns of S that sit at the window edges of column 0 and next to the intercept (listed together in the edge rows)"""
    Dg = Dt - 1
    e = {0, 1, 2, HC_CELLS - 2, HC_CELLS - 1, HC_CELLS, HC_CELLS + 1, 2 * HC_CELLS - 1, 2 * HC_CELLS, 2 * HC_CELLS + 1, Dg - 2, Dg - 1}
    return sorted(c for c in e if 0 <= c < Dg)


def window_distances(Dt):
    """the pair distances c2 - c1 (c2 the intercept included) the edge rows must list: the last cell of the first window, the first of
    the second, and the third window where the width has one"""
    d = [HC_CELLS - 1] + ([HC_CELLS] if Dt - 1 >= HC_CELLS else [])
    return d + ([2 * HC_CELLS] if Dt - 1 >= 2 * HC_CELLS else [])


def window_case(Dt, seed=0):
    """D' = Dt over two partitions of 1 200 rows listing only S: clusters at columns 0, HC_CELLS, 2 HC_CELLS and the intercept, and
    300 columns at random; the first 16 rows of each partition list every edge column; lambda_map on 300 columns, most of them empty"""
    rng = np.random.default_rng(7100 + Dt + seed)
    Dg = Dt - 1
    S = set(range(24)) | set(range(Dg - 24, Dg))
    for e in (HC_CELLS, 2 * HC_CELLS):
        S |= set(range(e - 12, e + 13))
    S |= set(rng.choice(Dg, 300, replace=False).tolist())
    S = np.array(sorted(c for c in S if 0 <= c < Dg))
    edges = window_edges(Dt)
    parts = []
    for p in range(2):
        n = 1200
        rows = []
        for i in range(n):
            r = set(S[rng.random(len(S)) < 12.0 / len(S)].tolist())
            if i < 16:
                r |= set(edges)
            rows.append(sorted(r))
        parts.append(_csr(rng, rows) + _labels(rng, n, range(20, n, 19)))
    z = np.zeros(Dt)
    z[S] = rng.normal(0, 0.2, len(S))
    z[Dg] = -0.3
    return dict(name="window%d" % Dt, Dg=Dg, parts=parts, z=z, lam=1.0, lambda_map=_lambda_map(rng, Dg, 300), S=S)


def q_of(case):
    """the prior precision of the z-update (test_gpu_admm_posterior._q): lambda, lambda_map's own where > 0, 0 at the intercept"""
    Dg = case["Dg"]
    lamf = float(np.float32(case["lam"]))
    lm = case["lambda_map"]
    q = np.full(Dg + 1, lamf)
    q[:Dg] = np.where(lm > 0, lm.astype(np.float64), lamf)
    q[Dg] = 0.0
    return q


def _design(part, Dg):
    """the partition's rows with the intercept column, fp64 CSR [n, Dg + 1]"""
    rowptr, cols, vals = part[:3]
    n = len(rowptr) - 1
    return sp.hstack([sp.csr_matrix((vals.astype(np.float64), cols, rowptr), shape=(n, Dg)), np.ones((n, 1))]).tocsr()


def row_weights(part, Dg, z):
    """d_i = w_i p_i (1 - p_i) at z, the row's offset included"""
    y, w, o = part[3:]
    s = _design(part, Dg) @ z + o.astype(np.float64)
    p = 1.0 / (1.0 + np.exp(-np.where(y > 0, 1.0, -1.0) * s))
    return w.astype(np.float64) * p * (1 - p)


def active(case):
    """A: every listed column and the intercept, ascending"""
    Dg = case["Dg"]
    return np.union1d(np.concatenate([p[1] for p in case["parts"]]).astype(np.int64), [Dg])


def reference(case):
    """fp64: A, H on A without the prior (hA), the full H's diagonal with the prior (hdiag: q plus each column's terms d_r x_rc^2,
    summed exactly and rounded once), Sigma on A (sA), the prior q"""
    Dg = case["Dg"]
    A = active(case)
    q = q_of(case)
    hA = np.zeros((len(A), len(A)))
    terms = [[] for _ in A]
    for part in case["parts"]:
        X = _design(part, Dg)
        d = row_weights(part, Dg, case["z"])
        XA = X.tocsc()[:, A]
        hA += (XA.T @ sp.diags(d) @ XA).toarray()
        for k in range(len(A)):
            r, x = XA.indices[XA.indptr[k]:XA.indptr[k + 1]], XA.data[XA.indptr[k]:XA.indptr[k + 1]]
            terms[k].append(d[r] * x * x)
    hdiag = q.copy()
    hdiag[A] = [math.fsum(np.concatenate(t).tolist() + [q[c]]) for t, c in zip(terms, A)]
    sA = np.linalg.inv(hA + np.diag(q[A]))
    return dict(A=A, hA=hA, hdiag=hdiag, sA=sA, q=q)


def diag_ulps(case, dense=()):
    """the ulps of 1/hdiag the diagonal mode may differ by, per column: 4, plus the fp64 additions of its sum in the device's order --
    per CSR partition ceil(m / 32) of a lane (m the rows listing the column there) and 5 of the warp sum, per dense partition one
    per row (partitions in `dense`), and one per partition; a column no CSR row lists adds nothing.  A sum of positive terms through k
    additions is within k 2^-53 of exact."""
    Dg = case["Dg"]
    k = np.full(Dg + 1, 4.0)
    for p, part in enumerate(case["parts"]):
        n = len(part[0]) - 1
        if p in dense:
            k += n + 1
        else:
            m = np.bincount(part[1], minlength=Dg + 1)
            m[Dg] = n
            k += np.where(m > 0, np.ceil(m / 32) + 6, 0)
    return k


def sigma_bound(case, ref):
    """the bound of test_gpu_admm_posterior._check_inverse, 8 D' kappa 2^-53 max|Sigma|, with kappa that of the active block (the
    empty columns' diagonal is decoupled from it)"""
    A, q = ref["A"], ref["q"]
    hq = ref["hA"] + np.diag(q[A])
    ev = np.linalg.eigvalsh(hq)
    empty = np.setdiff1d(np.arange(case["Dg"] + 1), A)
    smax = max(np.abs(ref["sA"]).max(), (1.0 / q[empty]).max() if len(empty) else 0.0)
    return 8 * (case["Dg"] + 1) * ev[-1] / ev[0] * EPS * smax


def sigma_rows(ref, Dt, r0, r1):
    """rows [r0, r1) of the full Sigma in closed form: inv(block) on A x A, 1/q on the diagonal of every other column, 0 elsewhere"""
    A, q, sA = ref["A"], ref["q"], ref["sA"]
    out = np.zeros((r1 - r0, Dt))
    inA = np.zeros(Dt, bool)
    inA[A] = True
    rr = np.arange(r0, r1)
    e = rr[~inA[rr]]
    out[e - r0, e] = 1.0 / q[e]
    ia = np.searchsorted(A, rr[inA[rr]])
    out[np.ix_(A[ia] - r0, A)] = sA[ia]
    return out


def products(case, part_idx, a, b):
    """every row of the partition listing columns a and b (b may be the intercept): (row, d_r x_ra x_rb)"""
    Dg = case["Dg"]
    part = case["parts"][part_idx]
    X = _design(part, Dg).tocsc()
    d = row_weights(part, Dg, case["z"])
    xa, xb = X[:, a].toarray().ravel(), X[:, b].toarray().ravel()
    r = np.nonzero((xa != 0) & (xb != 0))[0]
    return r, d[r] * xa[r] * xb[r]


def stage_two_products(case):
    """per designated column of more than HC_STAGE rows (the all-rows column included): the largest product d_r x_rc^2 of a row at
    position >= HC_STAGE of the column's row-ordered list in partition 0 -> [(c, c, product)]"""
    out = []
    for c in [cc for cc, k in zip(case["stage_cols"], STAGE_COUNTS) if k > HC_STAGE] + [case["all_col"]]:
        r, pr = products(case, 0, c, c)
        late = pr[HC_STAGE:]
        out.append((c, c, late[np.argmax(np.abs(late))]))
    return out


def cross_window_products(case):
    """per distance of window_distances: the largest product of an edge-row pair (c1, c1 + distance) -> [(c1, c2, product)]"""
    Dt = case["Dg"] + 1
    edges = window_edges(Dt) + [Dt - 1]
    out = []
    for dist in window_distances(Dt):
        best = None
        for c1 in edges:
            if c1 + dist in edges:
                pr = np.concatenate([products(case, p, c1, c1 + dist)[1] for p in range(len(case["parts"]))])
                if len(pr) and (best is None or abs(pr).max() > abs(best[2])):
                    best = (c1, c1 + dist, pr[np.argmax(np.abs(pr))])
        out.append(best)
    return out


def sigma_without(case, ref, c1, c2, prod):
    """Sigma on A with one product d_r x_r,c1 x_r,c2 missing from H (both triangles)"""
    A = ref["A"]
    i, j = np.searchsorted(A, [c1, c2])
    h = ref["hA"].copy()
    h[i, j] -= prod
    if i != j:
        h[j, i] -= prod
    return np.linalg.inv(h + np.diag(ref["q"][A]))


# ---- long records for score_var ----
def long_records(seed=0, D=3000, lens=RECORD_LENS):
    """two records of every length over D features, a model, a random SPD Sigma [D + 1, D + 1] and its diagonal"""
    rng = np.random.default_rng(7200 + seed)
    rows = [np.sort(rng.choice(D, L, replace=False)) for L in lens for _ in range(2)]
    rowptr, cols, vals = _csr(rng, rows)
    o = rng.normal(0, 0.1, len(rows)).astype(np.float32)
    model = rng.normal(0, 0.05, D + 1)
    A = rng.normal(0, 1, (D + 1, D + 1))
    cov = A @ A.T / D + np.eye(D + 1)
    return dict(D=D, rowptr=rowptr, cols=cols, vals=vals, o=o, model=model, cov=cov, var=np.diag(cov).copy())


def intercept_g(model, D, n_rep):
    b = model[D]
    return n_rep * np.exp(-b) / (n_rep - 1 + n_rep * np.exp(-b))


def record_terms(rec, i, n_rep, binary):
    """record i's g (its entries, then gI at the intercept) and columns"""
    D = rec["D"]
    j0, j1 = rec["rowptr"][i], rec["rowptr"][i + 1]
    x = np.ones(j1 - j0) if binary else rec["vals"][j0:j1].astype(np.float64)
    return np.append(x, intercept_g(rec["model"], D, n_rep)), np.append(rec["cols"][j0:j1], D)


def score_var_ref(rec, S, n_rep, binary, diag):
    """fp64 g^T Sigma g (diag: sum of S[c] g_c^2) of every record"""
    out = []
    for i in range(len(rec["rowptr"]) - 1):
        g, idx = record_terms(rec, i, n_rep, binary)
        out.append(np.sum(S[idx] * g * g) if diag else g @ S[np.ix_(idx, idx)] @ g)
    return np.array(out)


def cross_tile_terms(g, S):
    """the terms 2 g_a g_b S[a, b] of every pair of entries a, b in different COV_TILE tiles of a record (g, S over its entries, the
    intercept excluded); empty below COV_TILE + 1 entries"""
    n = len(g)
    t = np.arange(n) // COV_TILE
    a, b = np.nonzero(t[:, None] > t[None, :])
    return 2.0 * g[a] * g[b] * S[a, b]


def float_tol(ref, ulps=2):
    """ulps float ulps of float32(ref), the tolerance of the pred_var tests"""
    return ulps * np.spacing(np.abs(np.float32(ref))).astype(np.float64)
