"""The wgmma Gram kernels (csrc/k2_gram.cu) bit for bit on exactly representable data, and entrywise on generic data.

At beta = 0 and offset = 0 the margin is 0, so d = w / 4; with w in {1, 4} and values in {+-1, +-2} every operand
sqrt(d) x (times the CSR kernel's power-of-two scale) is exact in e4m3 and bf16, every product and chain sum is an integer
number of units far below the accumulators' precision, and the Hessian must equal X^T D X + diag(q) computed in float64.
A group of 32 rows in the wrong place, a stale or doubled chain, or a wrong sqrt(d) lane changes it.

The shapes are chosen from the device's SM count so that the CSR consumer loop takes every path: whole ring passes followed
by each tail length, slices shorter than the ring, empty slices, and one slice of hundreds of K-steps.

The entrywise bound |H - H_emu| <= c |A|^T |A| on generic data (A the emulated e4m3 / bf16 operand) keeps checking the
same places once a change makes the Gram no longer bitwise identical."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gram_reference as gr  # noqa: E402

pytestmark = pytest.mark.gpu

Q = 2.0   # prior precision: a power of two keeps the diagonal exact
C_CSR, C_DENSE = gr.ENTRYWISE_C_CSR, gr.ENTRYWISE_C_DENSE


@pytest.fixture(scope="module")
def mb():
    import mlease_b200
    return mlease_b200


@pytest.fixture(scope="module")
def num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _hessian(mb, X, w, D, *, csr, o=None, beta=None, binary=False, tensor=True):
    n = X.shape[0]
    y = (np.arange(n) % 3 == 0).astype(np.int32)
    o = np.zeros(n, np.float32) if o is None else np.asarray(o, np.float32)
    beta = np.zeros(D + 1) if beta is None else beta
    with mb.AdmmSession(1, D, [1.0], binary_feature=binary) as s:
        if csr:
            s.add_partition_csr(0, *gr.csr_arrays(X), y, np.asarray(w, np.float32), o)
        else:
            s.add_partition_dense(0, np.asarray(X.toarray() if sp.issparse(X) else X, np.float32), y, np.asarray(w, np.float32), o)
        _, _, H = s.objective(0, beta, np.zeros(D + 1), np.full(D + 1, Q), want_hessian=True, tensor=tensor)
    return H


def _check_exact(H, X, w, D, what, binary=False):
    Xv = X
    if binary:
        Xv = X.copy()
        Xv.data[:] = 1.0
    H_exact = gr.exact_hessian(Xv, np.asarray(w, np.float64) / 4.0, np.full(D + 1, Q))
    # the premise before the kernel: the intercept diagonal is sum(w) / 4 + q whatever the tiles do
    assert H[D, D] == np.sum(np.asarray(w, np.float64)) / 4.0 + Q, ("exactness premise failed (not a tiling bug)", what, H[D, D])
    bad = np.argwhere(H != H_exact)
    assert bad.size == 0, (what, len(bad), bad[:5].tolist(), [(H[i, j], H_exact[i, j]) for i, j in bad[:5]])


def _exact_csr(n, D, density, seed, w_choices=(1.0, 4.0)):
    rng = np.random.default_rng(seed)
    X, w = gr.exact_values(gr.random_pattern(n, D, density, rng), w_choices, rng)
    return X, w


# ------------------------------------------------------------------------------------------------------------------------
# 1. CSR e4m3 Gram, exact
# ------------------------------------------------------------------------------------------------------------------------
def test_csr_exact_every_consumer_path(mb, num_sms):
    shapes = gr.shapes_covering(num_sms)
    covered = set()
    print("\nCSR Gram shapes on %d SMs: (n, D, slices, K-steps per slice)" % num_sms)
    for i, (n, D) in enumerate(shapes):
        g = gr.gram_geometry(n, D, num_sms, True)
        X, w = _exact_csr(n, D, min(0.1, 12.0 / D), seed=100 + i)
        gr.check_limits(g, X.nnz)
        gr.check_exact_premises(X, w, csr=True)
        print("  ", (n, D, g.slices, sorted(set(g.nk))))
        _check_exact(_hessian(mb, X, w, D, csr=True), X, w, D, (n, D))
        covered |= gr.csr_paths(g)
    assert covered == gr.CSR_TARGETS, gr.CSR_TARGETS - covered


@pytest.mark.parametrize("name", gr.CSR_EDGE_CASES)
def test_csr_exact_structural_edges(mb, num_sms, name):
    X, w, D, binary = gr.csr_edge_case(name)
    g = gr.gram_geometry(X.shape[0], D, num_sms, True)
    gr.check_limits(g, X.nnz)
    gr.check_exact_premises(X, w, csr=True, binary=binary)
    print("\n  ", name, (X.shape[0], D, g.slices, sorted(set(g.nk))))
    _check_exact(_hessian(mb, X, w, D, csr=True, binary=binary), X, w, D, name, binary=binary)


# ------------------------------------------------------------------------------------------------------------------------
# 2. dense bf16 Gram, exact: the wgmma kernel and the SIMT kernel
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tensor", [True, False])
def test_dense_exact(mb, num_sms, tensor):
    shapes = gr.dense_shapes(num_sms)
    seen = set()
    print("\ndense Gram shapes on %d SMs (tensor=%s): (n, D, slices, K-steps per slice)" % (num_sms, tensor))
    for i, (n, D) in enumerate(shapes):
        g = gr.gram_geometry(n, D, num_sms, False)
        gr.check_limits(g, csr=False)
        rng = np.random.default_rng(200 + i)
        X, w = gr.exact_values(gr.random_pattern(n, D, 0.5, rng), (1.0, 4.0), rng)
        gr.check_exact_premises(X.toarray(), w, csr=False)
        print("  ", (n, D, g.slices, sorted(set(g.nk))))
        _check_exact(_hessian(mb, X, w, D, csr=False, tensor=tensor), X, w, D, (n, D, tensor))
        seen |= {"Dp%256=128"} if g.Dp % 256 == 128 else set()
        seen |= {"n%64"} if n % 64 else set()
        seen |= {"nk=0"} if 0 in g.nk else set()
        seen |= {"one slice, D=4000"} if g.slices == 1 and D == 4000 else set()
    assert seen == {"Dp%256=128", "n%64", "nk=0", "one slice, D=4000"}, seen


# ------------------------------------------------------------------------------------------------------------------------
# 3. generic data, entrywise
# ------------------------------------------------------------------------------------------------------------------------
def _entrywise(mb, X, w, o, beta, D, csr):
    A, slack = gr.emulated_operand(X, w, o, beta, csr)
    H = _hessian(mb, X, w, D, csr=csr, o=o, beta=beta)
    H_emu = gr.gram(A) + np.diag(np.full(D + 1, Q))
    return float(gr.entrywise_excess(H, H_emu, A, slack).max()), A


def test_entrywise_csr(mb, num_sms):
    seen = []
    cases = [(n, D, None) for n, D in gr.shapes_covering(num_sms)] + [(3000, 300, 1e4)]
    for i, (n, D, heavy) in enumerate(cases):
        rng = np.random.default_rng(300 + i)
        X, w, o, beta = gr.generic_problem(n, D, min(0.1, 12.0 / D), rng, heavy=heavy)
        gr.check_limits(gr.gram_geometry(n, D, num_sms, True), X.nnz)
        e, A = _entrywise(mb, X, w, o, beta, D, csr=True)
        if heavy is not None:   # the premise of the heavy-tailed case: most operands are e4m3 subnormals
            g = gr.csr_gram_scale(float(np.abs(X.data).max()), float(w.max()))
            a = np.abs(A.data[A.data != 0]) * g
            assert np.mean(a < 2.0 ** -6) > 0.5, np.mean(a < 2.0 ** -6)
        print("\n  CSR entrywise excess", (n, D, heavy), e)
        seen.append(((n, D, heavy), e))
    worst = max(e for _, e in seen)
    print("  CSR entrywise excess, max over shapes:", worst, "bound", C_CSR)
    assert worst <= C_CSR, seen


def test_entrywise_dense(mb, num_sms):
    seen = []
    for i, (n, D) in enumerate(gr.dense_shapes(num_sms)):
        rng = np.random.default_rng(400 + i)
        X, w, o, beta = gr.generic_problem(n, D, 1.0, rng)
        gr.check_limits(gr.gram_geometry(n, D, num_sms, False), csr=False)
        e, _ = _entrywise(mb, X, w, o, beta, D, csr=False)
        print("\n  dense entrywise excess", (n, D), e)
        seen.append(((n, D), e))
    worst = max(e for _, e in seen)
    print("  dense entrywise excess, max over shapes:", worst, "bound", C_DENSE)
    assert worst <= C_DENSE, seen


# ------------------------------------------------------------------------------------------------------------------------
# 4. factorisation of an exact Gram: chol_prep's slice sum and unscale against known numbers
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [700, 1500, 2100])   # ldh 704 (NB = 32 path), 1504 (DMMA), 2112 (explicit inverse, want_hinv)
def test_inverse_of_exact_gram(mb, D):
    X, w = _exact_csr(4000, D, 12.0 / D, seed=500 + D)
    gr.check_exact_premises(X, w, csr=True)
    Hinv = _hessian(mb, X, w, D, csr=True, tensor=2)
    H_exact = gr.exact_hessian(X, w / 4.0, np.full(D + 1, Q))
    err = np.abs(Hinv @ H_exact - np.eye(D + 1)).sum(axis=1).max()
    assert err <= 1e-9, err
