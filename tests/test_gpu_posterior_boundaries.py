"""The ADMM posterior and predictive-variance scoring where their kernels split the work, on the cases of tests/posterior_cases.py:
postvar_hess_col_kernel's second and later HC_STAGE stages of a column's rows and its second and third HC_CELLS column windows, and
score_var_kernel's pairs across 256-entry tiles of a long record.  Sigma against the fp64 inverse of the active block (closed form on
the empty columns) under test_gpu_admm_posterior's bound; the diagonal mode within 4 ulps plus its summation-order bound
(posterior_cases.diag_ulps) of the exactly summed diagonal; the session's own column index, the one
built for the call and a permuted upload order bit for bit equal; pred_var within 2 float ulps of fp64."""
import hashlib

import numpy as np
import pytest

import mlease_b200 as mb
import posterior_cases as pc
from test_gpu_admm_posterior import _dense

pytestmark = pytest.mark.gpu

CASES = ["stage"] + ["window%d" % Dt for Dt in pc.WINDOW_WIDTHS]


def _case(name):
    return pc.stage_case() if name == "stage" else pc.window_case(int(name[len("window"):]))


def _session(case, order=None, dense=(), **kw):
    """the case's partitions in upload order `order`, those in `dense` as dense rows; no ADMM batch (the posterior takes z)"""
    parts = case["parts"]
    s = mb.AdmmSession(len(parts), case["Dg"], [case["lam"]], lambda_map=case["lambda_map"], **kw)
    for pid in (order if order is not None else range(len(parts))):
        rowptr, cols, vals, y, w, o = parts[pid]
        if pid in dense:
            s.add_partition_dense(pid, _dense(parts[pid], case["Dg"]).astype(np.float32), y, w, o)
        else:
            s.add_partition_csr(pid, rowptr, cols, vals, y, w, o)
    return s


def _need_memory(Dt):
    """skip unless the device has the full posterior's 4 x 8 x ldh^2 bytes free (computed) and 1 GiB beside them"""
    import torch
    ldh = (Dt + 31) // 32 * 32
    need = 4 * 8 * ldh * ldh + (1 << 30)
    free = torch.cuda.mem_get_info(0)[0]
    if free < need:
        pytest.skip("the full posterior at D' = %d needs %d bytes of device memory, %d are free" % (Dt, need, free))


def _check_sigma(case, ref, cov, tag):
    """Sigma in chunks of rows against the closed form within pc.sigma_bound; the empty columns' diagonal within 4 ulps of 1/q"""
    Dt = case["Dg"] + 1
    bound = pc.sigma_bound(case, ref)
    err = 0.0
    for r0 in range(0, Dt, 2048):
        r1 = min(Dt, r0 + 2048)
        err = max(err, float(np.abs(cov[r0:r1] - pc.sigma_rows(ref, Dt, r0, r1)).max()))
    assert err <= bound, (tag, err, bound)
    empty = np.setdiff1d(np.arange(Dt), ref["A"])
    want = 1.0 / ref["q"][empty]
    assert np.all(np.abs(cov[empty, empty] - want) <= 4 * np.spacing(want)), tag
    print(tag, "D'", Dt, "worst ratio", err / bound)
    return err / bound


def _digest(a):
    return hashlib.sha256(memoryview(np.ascontiguousarray(a))).hexdigest()


def _full(s, case):
    var, cov = s.admm_posterior(0, z=case["z"], full=True, want_cov=True)
    s.close()
    assert np.array_equal(var, np.diag(cov))
    return cov


@pytest.mark.parametrize("name", CASES)
def test_full_and_diagonal(name):
    case = _case(name)
    Dt = case["Dg"] + 1
    _need_memory(Dt)
    ref = pc.reference(case)
    P = len(case["parts"])
    perm = list(range(P))[::-1]
    diag_ref = 1.0 / ref["hdiag"]
    diag_tol = pc.diag_ulps(case) * np.spacing(diag_ref)
    # the column index built at upload (default), the one built for the call (matrix-free session), a permuted upload order
    digests, diags = [], []
    for kw, order in [({}, None), (dict(hessian_policy=2), None), ({}, perm)]:
        s = _session(case, order=order, **kw)
        vd = s.admm_posterior(0, z=case["z"], full=False)
        assert np.all(np.abs(vd - diag_ref) <= diag_tol), (name, kw, order, (np.abs(vd - diag_ref) / np.spacing(diag_ref)).max())
        diags.append(vd)
        cov = _full(s, case)
        if not digests:
            _check_sigma(case, ref, cov, name)
        digests.append(_digest(cov))
        del cov
    assert digests[1] == digests[0] and digests[2] == digests[0], name
    assert np.array_equal(diags[1], diags[0]) and np.array_equal(diags[2], diags[0]), name


def test_stage_case_with_a_dense_partition():
    """the session takes dense and CSR partitions side by side for the posterior (only the ADMM batch asks for one kind): partition
    2 of the stage case uploaded dense goes through postvar_hess_dense_kernel, the others through the column walk"""
    case = pc.stage_case()
    ref = pc.reference(case)
    s = _session(case, dense=(2,))
    vd = s.admm_posterior(0, z=case["z"], full=False)
    want = 1.0 / ref["hdiag"]
    assert np.all(np.abs(vd - want) <= pc.diag_ulps(case, dense=(2,)) * np.spacing(want))
    _check_sigma(case, ref, _full(s, case), "stage, partition 2 dense")


@pytest.mark.parametrize("binary", [False, True])
@pytest.mark.parametrize("n_rep", [1, 5])
def test_score_var_long_records(n_rep, binary):
    rec = pc.long_records()
    rp, ci, v, o, model, D = rec["rowptr"], rec["cols"], rec["vals"], rec["o"], rec["model"], rec["D"]
    pred_ref = mb.score(v, model, rowptr=rp, colidx=ci, offset=o, num_features=D, num_click_replicates=n_rep, binary_feature=binary)
    for kw, S, diag in [(dict(cov=rec["cov"]), rec["cov"], False), (dict(var=rec["var"]), rec["var"], True)]:
        pred, pv = mb.score_var(rp, ci, v, model, offset=o, num_click_replicates=n_rep, binary_feature=binary, **kw)
        assert np.array_equal(pred.view(np.uint32), pred_ref.view(np.uint32))
        want = pc.score_var_ref(rec, S, n_rep, binary, diag)
        assert np.all(np.abs(pv - want) <= pc.float_tol(want)), (diag, np.abs(pv - want).max())


def test_score_var_under_the_three_window_posterior():
    """records over S scored with score_var under the Sigma admm_posterior returned at D' = 24 601: pred_var within 2 float ulps of
    fp64 g^T H^-1 g plus ||g||_1^2 times the Sigma bound"""
    Dt = pc.WINDOW_WIDTHS[-1]
    _need_memory(Dt)
    case = pc.window_case(Dt)
    ref = pc.reference(case)
    cov = _full(_session(case), case)
    Dg, S, A = case["Dg"], case["S"], ref["A"]
    rng = np.random.default_rng(7300)
    lens = [L for L in (1, 200, 256, 257, len(S)) if L <= len(S)]
    rows = [np.sort(rng.choice(S, L, replace=False)) for L in lens]
    rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    ci = np.concatenate(rows).astype(np.int32)
    v = rng.normal(0, 1, len(ci)).astype(np.float32)
    _, pv = mb.score_var(rp, ci, v, case["z"], cov=cov)
    del cov
    bound = pc.sigma_bound(case, ref)
    for i in range(len(lens)):
        g = np.append(v[rp[i]:rp[i + 1]].astype(np.float64), 1.0)
        k = np.searchsorted(A, np.append(ci[rp[i]:rp[i + 1]], Dg))
        want = g @ ref["sA"][np.ix_(k, k)] @ g
        assert abs(pv[i] - want) <= pc.float_tol(want) + np.abs(g).sum() ** 2 * bound, (lens[i], pv[i], want)
