"""Exact-data edge cases of the sparse CSR Gram's spans (gram_csr_sparse_kernel, csrc/k2_gram.cu): a warp works on a span of
gram_sparse_span() consecutive 32-row groups (8, i.e. 256 rows, in every case here), stages the bj range of the span in chunks of
448 entries, and enumerates the (bi entry, staged partner) pairs in steps of 32.

Each case runs through both CSR Gram kernels, forced with the library's test hook, and must equal X^T D X + diag(q) bit for bit
(the premises of gram_reference.check_exact_premises).  The CPU tests check that each case's data reaches the path it is named
after, from the span and chunk geometry below."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gram_reference as gr  # noqa: E402
from test_gram_sparse import KINDS, _check_exact, _hessian  # noqa: E402

SPAN, STAGE = 8, 448   # k2_gram.cu SP_SPAN (most groups per span) and SP_STAGE (staged entries per warp and chunk)


def sparse_span(n, D, nnz):
    """kernels.cuh gram_sparse_span: SPAN groups per span, fewer when the mean (block, group) range of the list (nnz + n entries:
    every row has its intercept entry) would not fit 3/4 of a stage chunk."""
    ngroups, nblk = -(-n // 32), gr.padded_width(D) // 128
    per = (nnz + n) / (max(1, nblk) * max(1, ngroups))
    return max(1, min(SPAN, int(0.75 * STAGE / max(per, 1.0))))


CASES = ["short last span, n%32", "runs empty in alternate groups", "row of 128 entries in a block",
         "stage chunks split spans and rows", "intercept cell with w=0 and empty rows"]


def case(name):
    """Exact CSR data -> (X, w, D)."""
    rng = np.random.default_rng(sum(name.encode()))
    if name == "short last span, n%32":
        # n = 40 * 256 + 3 * 32 + 11 = 10 347: 324 groups (the last one 11 rows), 324 % 8 = 4, so the 41st span has 4 groups and
        # the first 9 of the 32 warps take two spans each
        n, D = 40 * 256 + 3 * 32 + 11, 300
        X, w = gr.exact_values(gr.random_pattern(n, D, 0.008, rng), (1.0, 4.0), rng)
        return X, w, D
    if name == "runs empty in alternate groups":
        # block 0 has entries in even groups only, block 1 in odd groups only, and groups 5, 10, 15, ... have none in either: in
        # tiles (1, 0), (2, 0) and (2, 1) (block 2 holds the intercept, every row) each span's two ranges are both nonempty while
        # one of them is empty in half its groups, so entries' rows come from non-adjacent groups
        n, D = 32 * 40 - 9, 300
        dense = np.zeros((n, D), np.float64)
        grp = np.arange(n) // 32
        dense[:, :256] = rng.random((n, 256)) < 0.02
        dense[grp % 2 == 1, :128] = 0
        dense[grp % 2 == 0, 128:256] = 0
        dense[grp % 5 == 0, :256] = 0
        return (*gr.exact_values(sp.csr_matrix(dense), (1.0, 4.0), rng), D)
    if name == "row of 128 entries in a block":
        # rows 37 and 300 hold all 128 columns of block 0: in tile (0, 0) each of their entries owns up to 128 pairs (128 * 129 / 2
        # of the row's pairs are kept), so a batch of 32 of them is 32 * 128 / 32 = 128 steps of 32 pairs.  The other rows are
        # 0.4 % dense (~0.5 entries in block 0), so each span's block-0 range is ~128 + 255 * 0.5 ~ 260 < 448 entries: one chunk
        n, D = 600, 255
        dense = (rng.random((n, D)) < 0.004).astype(np.float64)
        dense[[37, 300], :128] = 1.0
        return (*gr.exact_values(sp.csr_matrix(dense), (1.0, 4.0), rng), D)
    if name == "stage chunks split spans and rows":
        # every row has exactly 3 entries in block 0 and none in blocks 1 .. 7 but the intercept, so a whole span's block-0 range
        # is 256 * 3 = 768 entries: two chunks, [0, 448) and [448, 768), and 448 = 3 * 149 + 1 puts the boundary between the first
        # and second entries of the span's row 149; w = 0 rows (zero bytes) still count in the range, so the boundary stays there
        n, D = 3 * 256 + 100, 1000
        dense = np.zeros((n, D), np.float64)
        for r in range(n):
            dense[r, rng.choice(128, size=3, replace=False)] = 1.0
        return (*gr.exact_values(sp.csr_matrix(dense), (0.0, 1.0, 4.0), rng), D)
    if name == "intercept cell with w=0 and empty rows":
        # D = 127: the intercept is column 127 of block 0, so tile (0, 0) sums the (intercept, intercept) cell in registers; every
        # row has an intercept entry (empty rows too: every 7th row and all of group 9), and w = 0 rows give zero bytes
        n, D = 5 * 256 + 77, 127
        X, w = gr.exact_values(gr.random_pattern(n, D, 0.002, rng), (0.0, 1.0, 4.0), rng)
        X = X.tolil()
        X[::7, :] = 0
        X[9 * 32:10 * 32, :] = 0
        X = X.tocsr()
        X.eliminate_zeros()
        return X, w, D
    raise KeyError(name)


# ------------------------------------------------------------------------------------------------------------------------
# GPU: both kernels, bit for bit
# ------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def mb():
    import mlease_b200
    return mlease_b200


@pytest.fixture(scope="module")
def num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.gpu
@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("name", CASES)
def test_exact_span_edges(mb, num_sms, kind, name):
    X, w, D = case(name)
    gr.check_limits(gr.gram_geometry(X.shape[0], D, num_sms, True), X.nnz)
    gr.check_exact_premises(X, w, csr=True)
    _check_exact(_hessian(mb, X, w, D, KINDS[kind]), X, w, D, (kind, name))


# ------------------------------------------------------------------------------------------------------------------------
# CPU: each case reaches the path it is named after
# ------------------------------------------------------------------------------------------------------------------------
def _layout(name):
    """(data, span, per-entry row and block of the list with its intercept entries, groups)"""
    X, w, D = case(name)
    n = X.shape[0]
    Xb = gr.with_intercept(X).tocsr()
    rows = np.repeat(np.arange(n), np.diff(Xb.indptr))
    return X, w, D, sparse_span(n, D, X.nnz), rows, Xb.indices // 128, -(-n // 32)


@pytest.mark.parametrize("name", CASES)
def test_cases_are_exact(name):
    X, w, D = case(name)
    gr.check_exact_premises(X, w, csr=True)
    gr.check_limits(gr.gram_geometry(X.shape[0], D, 132, True), X.nnz)


def test_short_last_span():
    X, _, _, span, _, _, ngroups = _layout("short last span, n%32")
    assert span == SPAN and X.shape[0] % 32 != 0 and ngroups % span != 0
    assert -(-ngroups // span) > 32   # more spans than warps: some warps take two


def test_runs_empty_in_alternate_groups():
    _, _, _, span, rows, blk, ngroups = _layout("runs empty in alternate groups")
    assert span == SPAN
    grp = rows // 32
    for s in range(-(-ngroups // span)):
        g = set(range(s * span, min(ngroups, (s + 1) * span)))
        in0, in1 = set(grp[blk == 0]) & g, set(grp[blk == 1]) & g
        assert in0 and in1 and not in0 & in1   # both ranges nonempty, never in the same group


def test_row_of_128_entries():
    _, _, _, span, rows, blk, _ = _layout("row of 128 entries in a block")
    assert span == SPAN
    assert np.bincount(rows[blk == 0]).max() == 128
    assert np.bincount(rows[blk == 0] // (32 * span)).max() <= STAGE   # one chunk


def test_stage_chunks_split_spans_and_rows():
    _, _, _, span, rows, blk, _ = _layout("stage chunks split spans and rows")
    assert span == SPAN
    r0 = rows[blk == 0]
    first = r0[r0 < 32 * span]           # the first span's block-0 range, in list order (rows ascending)
    assert len(first) > STAGE
    assert first[STAGE - 1] == first[STAGE]   # the chunk boundary falls inside a row


def test_intercept_cell_with_zero_weights_and_empty_rows():
    X, w, D, span, _, _, _ = _layout("intercept cell with w=0 and empty rows")
    assert span == SPAN and D // 128 == 0   # the intercept (column D) is in block 0: tile (0, 0) is its diagonal tile
    empty = np.diff(X.indptr) == 0
    assert empty.any() and (w == 0).any() and (empty & (w > 0)).any()
