"""The exact sparse CSR Gram (gram_csr_sparse_kernel, csrc/k2_gram.cu) and the data-driven choice between it and the e4m3 wgmma
kernel (session.cu batch_alloc).

The sparse kernel forms only the nonzero products of each row, as integers in units of 2^-18 summed in int64, and rounds each
Gram entry once to fp32.  So on generic data it is within one fp32 rounding of the Gram of the emulated e4m3 operand, and on
exact data (see test_gram_exact.py) it equals X^T D X + diag(q) bit for bit.  The exact data runs through both kernels, forced
with the library's test hook, because the automatic rule now sends those small sparse shapes to the sparse kernel.

The CPU tests pin a Python transcription of the kernel's e4m3 byte -> integer decode against torch's float8_e4m3fn, and the
SATFINITE rounding mirror (gram_reference.e4m3_round) against the NaN codes.  They check the arithmetic, not the CUDA source: the
device decode and the operand pass's conversion are covered only by the GPU tests (exact data bit for bit, generic data within
one rounding)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gram_reference as gr  # noqa: E402

Q = 2.0   # prior precision: a power of two keeps the diagonal exact
AUTO, WGMMA, SPARSE = 0, 1, 2
KINDS = {"wgmma": WGMMA, "sparse": SPARSE}


@pytest.fixture(scope="module")
def mb():
    import mlease_b200
    return mlease_b200


@pytest.fixture(scope="module")
def num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _hooks():
    from mlease_b200._hooks import bound
    return bound()


def _set_kind(s, kind):
    from mlease_b200._native import check
    check(_hooks().mlease_internal_set_csr_gram(s._h, kind))


def _kinds(s):
    """(ADMM batch, scratch batch) CSR Gram kinds of a session (0: no such batch)"""
    from mlease_b200._native import check
    b, sc = C.c_int32(), C.c_int32()
    check(_hooks().mlease_internal_csr_gram(s._h, C.byref(b), C.byref(sc)))
    return b.value, sc.value


def _hessian(mb, X, w, D, kind, o=None, beta=None, binary=False, session_calls=1):
    n = X.shape[0]
    y = (np.arange(n) % 3 == 0).astype(np.int32)
    o = np.zeros(n, np.float32) if o is None else np.asarray(o, np.float32)
    beta = np.zeros(D + 1) if beta is None else beta
    out = []
    with mb.AdmmSession(1, D, [1.0], binary_feature=binary) as s:
        _set_kind(s, kind)
        s.add_partition_csr(0, *gr.csr_arrays(X), y, np.asarray(w, np.float32), o)
        for _ in range(session_calls):
            out.append(s.objective(0, beta, np.zeros(D + 1), np.full(D + 1, Q), want_hessian=True)[2])
        if kind != AUTO:
            assert _kinds(s)[1] == kind
    return out if session_calls > 1 else out[0]


def _check_exact(H, X, w, D, what, binary=False):
    Xv = X
    if binary:
        Xv = X.copy()
        Xv.data[:] = 1.0
    H_exact = gr.exact_hessian(Xv, np.asarray(w, np.float64) / 4.0, np.full(D + 1, Q))
    bad = np.argwhere(H != H_exact)
    assert bad.size == 0, (what, len(bad), bad[:5].tolist(), [(H[i, j], H_exact[i, j]) for i, j in bad[:5]])


# ------------------------------------------------------------------------------------------------------------------------
# exact data, both kernels
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kind", list(KINDS))
def test_exact_covering_shapes(mb, num_sms, kind):
    for i, (n, D) in enumerate(gr.shapes_covering(num_sms)):
        rng = np.random.default_rng(100 + i)
        X, w = gr.exact_values(gr.random_pattern(n, D, min(0.1, 12.0 / D), rng), (1.0, 4.0), rng)
        gr.check_limits(gr.gram_geometry(n, D, num_sms, True), X.nnz)
        gr.check_exact_premises(X, w, csr=True)
        _check_exact(_hessian(mb, X, w, D, KINDS[kind]), X, w, D, (kind, n, D))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("name", gr.CSR_EDGE_CASES)
def test_exact_structural_edges(mb, num_sms, kind, name):
    X, w, D, binary = gr.csr_edge_case(name)
    gr.check_limits(gr.gram_geometry(X.shape[0], D, num_sms, True), X.nnz)
    gr.check_exact_premises(X, w, csr=True, binary=binary)
    _check_exact(_hessian(mb, X, w, D, KINDS[kind], binary=binary), X, w, D, (kind, name), binary=binary)


def _long_uneven_runs(seed):
    """Exact data whose (block 0, group) runs hold 32 rows of 100..127 entries (3 200 - 4 064 entries): the sparse kernel stages
    them in chunks of 256 entries, and most chunk boundaries fall inside a row."""
    rng = np.random.default_rng(seed)
    n, D = 32 * 20 - 5, 255
    dense = np.zeros((n, D), np.float64)
    for r in range(n):
        dense[r, rng.choice(128, size=rng.integers(100, 128), replace=False)] = 1.0
    dense[:, 128:] = rng.random((n, D - 128)) < 0.03
    X, w = gr.exact_values(sp.csr_matrix(dense), (1.0, 4.0), rng)
    return X, w, D


@pytest.mark.gpu
@pytest.mark.parametrize("kind", list(KINDS))
def test_exact_runs_straddling_stage_chunks(mb, num_sms, kind):
    X, w, D = _long_uneven_runs(seed=41)
    gr.check_limits(gr.gram_geometry(X.shape[0], D, num_sms, True), X.nnz)
    gr.check_exact_premises(X, w, csr=True)
    _check_exact(_hessian(mb, X, w, D, KINDS[kind]), X, w, D, (kind, "runs straddling 256-entry chunks"))


# ------------------------------------------------------------------------------------------------------------------------
# generic data, sparse kernel: one fp32 rounding of the emulated operand's Gram
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_generic_within_one_rounding(mb, num_sms):
    cases = [(n, D, None) for n, D in gr.shapes_covering(num_sms)] + [(3000, 300, 1e4)]
    for i, (n, D, heavy) in enumerate(cases):
        rng = np.random.default_rng(300 + i)
        X, w, o, beta = gr.generic_problem(n, D, min(0.1, 12.0 / D), rng, heavy=heavy)
        A, slack = gr.emulated_operand(X, w, o, beta, csr=True)
        if heavy is not None:   # the premise of the heavy-tailed case: most operands are e4m3 subnormals
            g = gr.csr_gram_scale(float(np.abs(X.data).max()), float(w.max()))
            a = np.abs(A.data[A.data != 0]) * g
            assert np.mean(a < 2.0 ** -6) > 0.5, np.mean(a < 2.0 ** -6)
        H = _hessian(mb, X, w, D, SPARSE, o=o, beta=beta)
        H_emu = gr.gram(A) + np.diag(np.full(D + 1, Q))
        excess = np.abs(H - H_emu) - slack - 2.0 ** -23 * np.abs(H_emu)
        assert excess.max() <= 0, ((n, D, heavy), float(excess.max()), np.unravel_index(np.argmax(excess), excess.shape))


# ------------------------------------------------------------------------------------------------------------------------
# repeatability
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_repeatable_bitwise(mb):
    rng = np.random.default_rng(17)
    n, D = 20000, 700
    X, w, o, beta = gr.generic_problem(n, D, 12.0 / D, rng)
    H1, H2 = _hessian(mb, X, w, D, SPARSE, o=o, beta=beta, session_calls=2)
    H3 = _hessian(mb, X, w, D, SPARSE, o=o, beta=beta)
    assert np.array_equal(H1, H2)
    assert np.array_equal(H1, H3)


# ------------------------------------------------------------------------------------------------------------------------
# the automatic choice
# ------------------------------------------------------------------------------------------------------------------------
def _strided_csr(n, D, nnz, seed):
    """n rows of nnz sorted unique columns each, one per stride of D // nnz"""
    rng = np.random.default_rng(seed)
    stride = D // nnz
    ci = (np.arange(nnz, dtype=np.int32)[None, :] * stride + rng.integers(0, stride, (n, nnz), dtype=np.int32)).reshape(-1)
    v = rng.standard_normal(n * nnz, dtype=np.float32)
    return np.arange(n + 1, dtype=np.int64) * nnz, ci, v, (rng.random(n) < 0.3).astype(np.int32)


@pytest.mark.gpu
@pytest.mark.parametrize("D,expect", [(10_000, SPARSE), (500, WGMMA)])
def test_automatic_choice(mb, D, expect):
    """The bench workload's partition shape (1M x 10k, 100 stored values per row: 1 %) picks the sparse kernel; the same rows at
    500 features (20 %, `bench.py --features 500`) keep the wgmma kernel."""
    rp, ci, v, y = _strided_csr(1_000_000, D, 100, seed=D)
    with mb.AdmmSession(1, D, [1.0]) as s:
        s.add_partition_csr(0, rp, ci, v, y)
        s.time_kernel(0, "k1", reps=1)   # allocates the scratch batch, where the rule runs
        assert _kinds(s) == (0, expect)
        s.begin()
        assert _kinds(s)[0] == expect


# ------------------------------------------------------------------------------------------------------------------------
# CPU: the e4m3 decode
# ------------------------------------------------------------------------------------------------------------------------
def e4m3_units(b):
    """k2_gram.cu e4m3_units: the byte's value in integer units of 2^-9"""
    e, m = (b >> 3) & 15, b & 7
    mag = (8 | m) << (e - 1) if e else m
    return -mag if b & 0x80 else mag


def test_e4m3_decode_matches_torch():
    import torch
    codes = torch.arange(256, dtype=torch.int32).to(torch.uint8)
    vals = codes.view(torch.float8_e4m3fn).to(torch.float64).numpy()
    for b in range(256):
        if b in (0x7F, 0xFF):
            assert np.isnan(vals[b])
            continue
        assert e4m3_units(b) == vals[b] * 512, (hex(b), e4m3_units(b), vals[b])
    assert max(abs(e4m3_units(b)) for b in range(256) if b not in (0x7F, 0xFF)) == 229376 < 2 ** 18
    # the row limit of the int64 sums (gram_sparse_max_rows): every row adds at most one product to a cell
    assert (2 ** 27) * 229376 ** 2 < 2 ** 63


def test_satfinite_never_yields_nan_codes():
    """The operand pass rounds with __NV_SATFINITE (mirrored by gram_reference.e4m3_round): every finite input, however large,
    lands on a finite e4m3 value, whose code is never 0x7F / 0xFF."""
    import torch
    x = np.concatenate([np.geomspace(2.0 ** -12, 1e30, 4000), [447.0, 448.0, 449.0, 464.0, 480.0, 512.0, 3.4e38]])
    x = np.concatenate([x, -x, [0.0]])
    r = gr.e4m3_round(x)
    assert np.all(np.isfinite(r)) and np.abs(r).max() == 448.0
    codes = torch.from_numpy(r.astype(np.float32)).to(torch.float8_e4m3fn).view(torch.uint8).numpy()
    assert not np.isin(codes, [0x7F, 0xFF]).any()
    assert np.array_equal(torch.from_numpy(codes).view(torch.float8_e4m3fn).to(torch.float64).numpy(), r)
