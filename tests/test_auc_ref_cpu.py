"""CPU checks of tests/auc_ref.py, the fp64 reference the GPU AUC tests compare against: brute-force pair enumeration on small cases
(ties, -0.0 / +0.0, +-inf, zero weights, single-class and empty keys), sklearn's weighted roc_auc_score, and the binding's no-GPU
failure."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from auc_ref import brute_force_auc, segment_upn, test_auc_ref  # noqa: E402


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def _same(a, b):
    return (np.isnan(a) and np.isnan(b)) or a == b


CASES = [
    ([1, 0], [0.5, 0.1], None),
    ([1, 0], [0.1, 0.5], None),
    ([1, 0, 1, -1], [0.3, 0.3, 0.3, 0.3], None),                       # one tie group: 1/2
    ([1, 0, 1, 0], [-0.0, 0.0, 0.0, -0.0], None),                       # the zeros tie
    ([1, 0, 1, 0, -1], [np.inf, -np.inf, -np.inf, np.inf, 0.0], [2, 1, 3, 1, 2]),
    ([1, 1, 0, 0, 1], [1.0, 2.0, 2.0, 1.0, 3.0], [0, 2, 0, 1, 3]),     # zero weights
    ([1, 1, 1], [0.1, 0.2, 0.3], None),                                 # positives only: NaN
    ([0, -1], [0.1, 0.2], None),                                        # negatives only: NaN
    ([], [], None),                                                     # empty: NaN
]


@pytest.mark.parametrize("resp,pred,w", CASES)
def test_against_brute_force(resp, pred, w):
    assert _same(brute_force_auc(resp, pred, w), (lambda u, p, n: u / (p * n) if p > 0 and n > 0 else np.nan)(*segment_upn(resp, pred, w)))


def test_random_ties_against_brute_force():
    rng = np.random.default_rng(3)
    vals = np.array([-np.inf, -1.0, -0.0, 0.0, 0.5, np.inf], np.float32)
    for _ in range(50):
        n = int(rng.integers(1, 40))
        r = rng.choice([1, 0, -1], n)
        p = rng.choice(vals, n)
        w = rng.integers(0, 4, n).astype(np.float32)
        u, P, N = segment_upn(r, p, w)
        assert _same(brute_force_auc(r, p, w), u / (P * N) if P > 0 and N > 0 else np.nan)


def test_keys_and_sets_layout():
    rng = np.random.default_rng(4)
    n, S = 60, 3
    krs = [0, 0, 10, 11, 40, 40, 60]   # empty keys, a one-row key
    r = rng.choice([1, 0, -1], n)
    p = rng.choice(np.array([0.0, 0.25, 1.0], np.float32), (S, n))
    w = rng.integers(0, 4, n).astype(np.float32)
    auc, wt, kauc, kw = test_auc_ref(r, p, w, krs)
    assert auc.shape == (S,) and kauc.shape == (S, 6) and kw.shape == (6, 2)
    assert wt[0] == w[r == 1].sum() and wt[1] == w[r != 1].sum()
    for s in range(S):
        assert _same(auc[s], brute_force_auc(r, p[s], w))
        for k in range(6):
            a, b = krs[k], krs[k + 1]
            assert _same(kauc[s, k], brute_force_auc(r[a:b], p[s, a:b], w[a:b]))
    assert np.isnan(kauc[:, 0]).all() and np.isnan(kauc[:, 2]).all() and (kw[0] == 0).all()


def test_against_sklearn():
    metrics = pytest.importorskip("sklearn.metrics")
    rng = np.random.default_rng(5)
    for n in (10, 1000, 20000):
        r = rng.choice([1, 0, -1], n)
        p = np.round(rng.normal(size=n), 2).astype(np.float32)   # plenty of ties
        w = rng.random(n).astype(np.float32)
        u, P, N = segment_upn(r, p, w)
        ref = metrics.roc_auc_score((r == 1).astype(int), p.astype(np.float64), sample_weight=w.astype(np.float64))
        assert abs(u / (P * N) - ref) <= 1e-12


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU failure mode")
def test_no_cpu_fallback():
    import mlease_b200 as mb
    with pytest.raises(mb.MleaseError, match="no CPU fallback"):
        mb.test_auc([1, 0, 1], [0.1, 0.2, 0.3])
    with pytest.raises(mb.MleaseError, match="no CPU fallback"):
        mb.test_auc([1, 0, 1], [[0.1, 0.2, 0.3]], key_rowstart=[0, 1, 3])
