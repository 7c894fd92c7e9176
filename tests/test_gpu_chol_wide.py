"""GPU tests (-m gpu) of the wide Cholesky (ldh > 1000): the factor against numpy's fp64 Cholesky at widths that end mid-panel
and mid-tile, run-to-run bit equality of the factor and the inverse (the look-ahead overlaps the panel chain with the trailing
update on a second stream), and bit equality of the two DMMA shapes the trailing update may issue (m16n8k4 is two m8n8k4
stacked in M).  The hooks are test entry points of the library, not part of its C ABI."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import factored_reference as fr  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def mb():
    import mlease_b200
    return mlease_b200


@pytest.fixture(scope="module")
def hooks(mb):
    from mlease_b200 import _hooks
    return _hooks.bound()


def _check(rc):
    from mlease_b200._native import check
    check(rc)


def _part(D, n, nnz, seed):
    r = np.random.default_rng(seed)
    ci = np.stack([np.sort(r.choice(D, nnz, replace=False)) for _ in range(n)]).astype(np.int32)
    v = r.normal(size=(n, nnz)).astype(np.float32)
    y = (r.random(n) < 0.5).astype(np.int32)
    return np.arange(n + 1, dtype=np.int64) * nnz, ci.reshape(-1), v.reshape(-1), y


def _spd(Dt, seed):
    """A dense SPD matrix with a spread of scales: X X^T / m + diag(0.1 .. 2)."""
    r = np.random.default_rng(seed)
    m = 384
    X = r.normal(size=(Dt, m)) * r.uniform(0.5, 2.0, (Dt, 1))
    H = X @ X.T / m
    H[np.diag_indices(Dt)] += r.uniform(0.1, 2.0, Dt)
    return H


def _factor(hooks, s, H, Dt):
    ldh = fr.ldh_of(Dt)
    L = np.empty((Dt, Dt))
    Y = np.empty((ldh, ldh))
    _check(hooks.mlease_internal_factor(s._h, 0, H.ctypes.data, L.ctypes.data, Y.ctypes.data, None))
    return L, Y


# 2101 / 2303: the last outer panel (256) and the last 128-row tile end mid-way; 4134, 6001: more panels, other remainders
@pytest.mark.parametrize("D", [2100, 2302, 4133, 6000])
def test_factor_against_numpy(mb, hooks, D):
    Dt = D + 1
    H = _spd(Dt, D)
    with mb.AdmmSession(1, D, [1.0]) as s:
        s.add_partition_csr(0, *_part(D, 300, 8, D))
        L, Y = _factor(hooks, s, H, Dt)
        L2, Y2 = _factor(hooks, s, H, Dt)
    ref = np.linalg.cholesky(H)
    err = np.abs(np.tril(L) - ref).max()
    assert err <= 1e-10 * np.abs(ref).max(), err
    # the same H twice: the same bits (the look-ahead's overlap does not change what any element receives)
    assert np.array_equal(L.view(np.uint64), L2.view(np.uint64))
    assert np.array_equal(Y.view(np.uint64), Y2.view(np.uint64))


def test_dmma_16x8x4_matches_8x8x4(mb, hooks):
    """The trailing update issues m16n8k4; each of its elements must take exactly the bits two m8n8k4 give (zero start, one
    4-product step per k4 chunk in ascending k), on operands with mixed signs, a wide exponent range and exact zeros."""
    r = np.random.default_rng(5)
    n, K = 256, 256
    A = r.normal(size=(n, 16, K)) * np.exp2(r.integers(-30, 30, (n, 16, K)))
    B = r.normal(size=(n, 8, K)) * np.exp2(r.integers(-30, 30, (n, 8, K)))
    A[r.random(A.shape) < 0.05] = 0.0
    B[:, :, 100:104] = -B[:, :, 96:100]   # chunks that cancel a previous chunk's products
    D8, D16 = np.empty((n, 16, 8)), np.empty((n, 16, 8))
    _check(hooks.mlease_internal_dmma_shapes(A.ctypes.data, B.ctypes.data, n, K, D8.ctypes.data, D16.ctypes.data))
    assert np.array_equal(D8.view(np.uint64), D16.view(np.uint64)), int((D8.view(np.uint64) != D16.view(np.uint64)).sum())
    ref = np.einsum("tik,tjk->tij", A, B)
    scale = np.einsum("tik,tjk->tij", np.abs(A), np.abs(B))
    assert (np.abs(D8 - ref) <= 1e-13 * scale + 1e-300).all()
