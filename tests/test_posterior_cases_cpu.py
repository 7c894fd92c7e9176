"""The cases of tests/posterior_cases.py hold what they claim (exact per-partition column counts, row lengths, the window-crossing pairs,
far inside the kernels' limits), and every tolerance the GPU tests hold them to sees the failure it exists for: one product of a
stage-two row, one cross-window cell or one cross-tile pair missing from the reference moves it by more than the tolerance."""
import numpy as np
import pytest

import posterior_cases as pc


def _within_limits(case):
    for rowptr, cols, vals, y, w, o in case["parts"]:
        n, nnz = len(rowptr) - 1, int(rowptr[-1])
        assert n < 2 ** 27 and nnz + n < 2 ** 32 - 64
        assert len(cols) == nnz == len(vals) and vals.dtype == np.float32 and len(y) == len(w) == len(o) == n
        assert set(np.unique(y)) <= {0, 1}
        assert np.all((w == 0) | ((w >= 0.5) & (w <= 2.0))) and np.any(w == 0)
        for i in range(n):
            c = cols[rowptr[i]:rowptr[i + 1]]
            assert np.all(np.diff(c) > 0) and (len(c) == 0 or (c[0] >= 0 and c[-1] < case["Dg"]))


def _col_counts(part, Dg):
    return np.bincount(part[1], minlength=Dg)


def test_stage_case_structure():
    case = pc.stage_case()
    Dg = case["Dg"]
    assert Dg + 1 == 700
    _within_limits(case)
    p0, p1, p2 = case["parts"]
    cnt = _col_counts(p0, Dg)
    assert [int(cnt[c]) for c in case["stage_cols"]] == list(pc.STAGE_COUNTS)
    assert cnt[case["all_col"]] == len(p0[0]) - 1 > 2 * pc.HC_STAGE
    assert cnt.max() == cnt[case["all_col"]]
    # the partition with no stored entry, and rows that hold the intercept alone
    assert p1[0][-1] == 0 and len(p1[1]) == 0 and len(p1[0]) > 1
    assert np.sum(np.diff(p2[0]) == 0) > 100
    # every stage-two row of every designated column carries weight
    for c in [c for c, k in zip(case["stage_cols"], pc.STAGE_COUNTS) if k > pc.HC_STAGE] + [case["all_col"]]:
        r = np.nonzero(np.diff(p0[0]) > 0)[0]
        rows = [i for i in r if c in p0[1][p0[0][i]:p0[0][i + 1]]]
        assert np.all(p0[4][rows[pc.HC_STAGE:]] > 0), c


@pytest.mark.parametrize("Dt", pc.WINDOW_WIDTHS)
def test_window_case_structure(Dt):
    case = pc.window_case(Dt)
    Dg = case["Dg"]
    assert Dg + 1 == Dt
    _within_limits(case)
    S = case["S"]
    assert 300 <= len(S) <= 450 and Dg - 1 in S and 0 in S
    listed = np.unique(np.concatenate([p[1] for p in case["parts"]]))
    assert np.array_equal(listed, S)            # every other column is empty
    # the window-crossing pairs, in one row, the intercept counted as a column of every row
    want = [pc.HC_CELLS - 1, pc.HC_CELLS] + ([2 * pc.HC_CELLS] if Dt > 2 * pc.HC_CELLS else [])
    want = [d for d in want if d <= Dg]
    assert pc.window_distances(Dt) == want
    for rowptr, cols, *_ in case["parts"]:   # row 0 of each partition is an edge row
        r = np.append(cols[rowptr[0]:rowptr[1]], Dg)
        dist = set((r[None, :] - r[:, None]).ravel().tolist())
        assert all(d in dist for d in want), (Dt, want)
    assert Dt <= pc.HC_CELLS or any(c < Dt - pc.HC_CELLS for c in S)   # columns with a second window
    if Dt > 2 * pc.HC_CELLS:
        assert sum(c < Dt - 2 * pc.HC_CELLS for c in S) >= 20            # columns that walk three windows
    # a non-constant prior on the empty columns
    q = pc.q_of(case)
    empty = np.setdiff1d(np.arange(Dg), S)
    assert len(np.unique(q[empty])) > 100


def test_long_record_structure():
    rec = pc.long_records()
    lens = np.diff(rec["rowptr"])
    assert sorted(set(lens.tolist())) == sorted(pc.RECORD_LENS) and np.all(np.bincount(lens)[list(pc.RECORD_LENS)] == 2)
    for i in range(len(lens)):
        c = rec["cols"][rec["rowptr"][i]:rec["rowptr"][i + 1]]
        assert np.all(np.diff(c) > 0) and c[0] >= 0 and c[-1] < rec["D"]
    assert np.all(np.linalg.eigvalsh(rec["cov"]) > 0.5)


def test_keyed_long_row_structure():
    from test_gpu_score_keyed_cov import LONG_ROWS, _data
    for G in (1, 3):
        pb, md = _data(np.random.default_rng(3200 + G), 12, G, empty={1, 12 * G - 1}, row_lens=LONG_ROWS)
        lens = np.diff(pb["rp"])
        assert set(lens.tolist()) == set(LONG_ROWS)
        for k in range(12):
            cols = md["mc"][md["mp"][k]:md["mp"][k + 1]]
            assert len(cols) >= 601 and cols[-1] == pb["D"]
            for i in range(pb["krs"][k], pb["krs"][k + 1]):
                c = pb["ci"][pb["rp"][i]:pb["rp"][i + 1]]
                assert np.all(np.diff(c) > 0)
                listed = np.isin(c, cols).sum()
                assert listed == (len(c) + 1) // 2, (k, i)


# ---- every tolerance sees the failure it exists for ----
def test_stage_tolerance_sees_one_stage_two_product():
    case = pc.stage_case()
    ref = pc.reference(case)
    bound = pc.sigma_bound(case, ref)
    for c1, c2, prod in pc.stage_two_products(case):
        s2 = pc.sigma_without(case, ref, c1, c2, prod)
        assert np.abs(s2 - ref["sA"]).max() > bound, (c1, prod, bound)
        # the diagonal mode's tolerance sees it too, with a dense partition 2 as well
        v, v2 = 1.0 / ref["hdiag"][c1], 1.0 / (ref["hdiag"][c1] - prod)
        assert abs(v2 - v) > max(pc.diag_ulps(case)[c1], pc.diag_ulps(case, dense=(2,))[c1]) * np.spacing(v)


@pytest.mark.parametrize("Dt", pc.WINDOW_WIDTHS)
def test_window_tolerance_sees_one_cross_window_cell(Dt):
    case = pc.window_case(Dt)
    ref = pc.reference(case)
    bound = pc.sigma_bound(case, ref)
    got = pc.cross_window_products(case)
    assert len(got) == len(pc.window_distances(Dt)) and all(g is not None for g in got)
    for c1, c2, prod in got:
        s2 = pc.sigma_without(case, ref, c1, c2, prod)
        assert np.abs(s2 - ref["sA"]).max() > bound, (Dt, c1, c2, prod, bound)


def test_closed_form_sigma_is_the_inverse():
    """the block formula is the inverse of the full H (checked where numpy inverts the whole matrix)"""
    case = pc.stage_case()
    ref = pc.reference(case)
    Dt = case["Dg"] + 1
    H = np.diag(ref["q"])
    H[np.ix_(ref["A"], ref["A"])] += ref["hA"]
    full = pc.sigma_rows(ref, Dt, 0, Dt)
    assert np.abs(full - np.linalg.inv(H)).max() <= pc.sigma_bound(case, ref)
    assert np.allclose(np.diag(H), ref["hdiag"], rtol=1e-14, atol=0)


@pytest.mark.parametrize("binary", [False, True])
@pytest.mark.parametrize("n_rep", [1, 5])
def test_score_tolerance_sees_one_cross_tile_pair(n_rep, binary):
    rec = pc.long_records()
    want = pc.score_var_ref(rec, rec["cov"], n_rep, binary, False)
    seen = 0
    for i in range(len(rec["rowptr"]) - 1):
        g, idx = pc.record_terms(rec, i, n_rep, binary)
        terms = pc.cross_tile_terms(g[:-1], rec["cov"][np.ix_(idx[:-1], idx[:-1])])
        if len(g) - 1 <= pc.COV_TILE:
            assert len(terms) == 0
            continue
        tol = pc.float_tol(want[i])
        assert np.abs(terms).max() > tol and abs(terms.sum()) > tol, (i, tol)
        seen += 1
    assert seen == 2 * sum(L > pc.COV_TILE for L in pc.RECORD_LENS)


def test_keyed_tolerance_sees_one_cross_tile_pair():
    from test_gpu_score_keyed_cov import LONG_ROWS, _data, _ref
    for G in (1, 3):
        pb, md = _data(np.random.default_rng(3100 + G + 100), 12, G, empty={1, 12 * G - 1}, row_lens=LONG_ROWS)
        want = _ref(pb, md, G)
        seen = 0
        for g in range(G):
            for k in range(12):
                m = g * 12 + k
                blk = md["cv"][md["cp"][m]:md["cp"][m + 1]]
                if not len(blk):
                    continue
                cols = md["mc"][md["mp"][m]:md["mp"][m + 1]]
                n = len(cols)
                S = np.zeros((n, n)); S[np.tril_indices(n)] = blk; S = S + np.tril(S, -1).T
                for i in range(pb["krs"][k], pb["krs"][k + 1]):
                    c = pb["ci"][pb["rp"][i]:pb["rp"][i + 1]]
                    if len(c) <= pc.COV_TILE:
                        continue
                    x = pb["v"][pb["rp"][i]:pb["rp"][i + 1]].astype(np.float64)
                    p = np.searchsorted(cols, c)
                    ok = (p < n) & (cols[np.minimum(p, n - 1)] == c)
                    xl = np.where(ok, x, 0.0)   # unlisted entries take part in no pair
                    terms = pc.cross_tile_terms(xl, S[np.ix_(np.minimum(p, n - 1), np.minimum(p, n - 1))])
                    tol = pc.float_tol(want[g, i])
                    assert np.abs(terms).max() > tol and abs(terms.sum()) > tol, (g, i)
                    seen += 1
        assert seen >= 2 * G
