"""The sparse CSR Gram built column by column (gram_csr_column_kernel, csrc/k2_gram.cu) on its row-order operand and the column
index built at upload.

For column c1 of the lower triangle the kernel walks the positions of c1's entries in the row-order operand (row r at
[rowptr[r] + r, rowptr[r + 1] + r], its intercept entry last); the partners of an entry are its row's suffix up to the intercept
word, found by its column.  Each operand word is the e4m3 value in units of 2^-9 as an fp32 (low 20 mantissa bits zero) with the
entry's full column id in those 20 bits.

The GPU tests force the kernel with the library's test hook and require X^T D X + diag(q) bit for bit on exact data
(gram_reference.check_exact_premises) at the structural edges of the walk.  The CPU tests pin a numpy transcription of the word
and of the index layout."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gram_reference as gr  # noqa: E402
from test_gram_sparse import SPARSE, Q, _check_exact, _hessian, _set_kind, e4m3_units  # noqa: E402

VALUE_MASK, COL_MASK = 0xFFF00000, 0x000FFFFF
MAX_COLS = 2 ** 20   # k2_gram.cu gram_sparse_max_cols: D' (features + intercept)
CELLS = 112 * 128    # k2_gram.cu GC_CELLS: the accumulator's cells, a wider column is walked once per window


# ------------------------------------------------------------------------------------------------------------------------
# CPU: the word and the index
# ------------------------------------------------------------------------------------------------------------------------
def encode(byte, col):
    """k2_gram.cu gram_word"""
    return int(np.array([e4m3_units(byte)], np.float32).view(np.uint32)[0]) | col


def decode(w):
    """k2_gram.cu gw_units, gw_col (the conversion truncates toward zero)"""
    return int(np.trunc(np.array([w & VALUE_MASK], np.uint32).view(np.float32)[0])), w & COL_MASK


def test_word_round_trip_every_code():
    for b in range(256):
        if b in (0x7F, 0xFF):   # NaN: the operand pass converts with SATFINITE
            continue
        u = e4m3_units(b)
        assert int(np.array([u], np.float32).view(np.uint32)[0]) & COL_MASK == 0, hex(b)
        for col in (0, 1, 127, 128, 10_000, MAX_COLS - 1):
            w = encode(b, col)
            assert w < 2 ** 32 and decode(w) == (u, col), (hex(b), col)


def row_order_layout(X):
    """(column of every word of the row-order operand, its row, column index offsets [D' + 1], positions): a transcription of
    gram_csr_operand_kernel's word positions and csr_col_index"""
    n, D = X.shape
    Xb = gr.with_intercept(X).tocsr()   # the intercept (column D) is every row's last entry
    col = Xb.indices.astype(np.int64)
    row = np.repeat(np.arange(n), np.diff(Xb.indptr))
    order = np.argsort(col, kind="stable")
    offs = np.searchsorted(col[order], np.arange(D + 2))
    return col, row, offs, order


def test_row_order_and_index_layout():
    rng = np.random.default_rng(3)
    n, D = 777, 300
    X = gr.random_pattern(n, D, 0.02, rng).tolil()
    X[5, :] = 0
    X[9, :] = 1.0
    X = X.tocsr()
    X.eliminate_zeros()
    col, row, offs, pos = row_order_layout(X)
    # row r occupies [rowptr[r] + r, rowptr[r + 1] + r] and ends with its intercept word
    rp = X.indptr
    assert len(col) == X.nnz + n
    for r in (0, 5, 9, n - 1):
        lo, hi = rp[r] + r, rp[r + 1] + r
        assert (row[lo:hi + 1] == r).all() and col[hi] == D
        assert (col[lo:hi] == X.indices[rp[r]:rp[r + 1]]).all()
    # the index lists every column's positions in row order; the intercept's holds every row, empty columns have none
    assert offs[0] == 0 and offs[-1] == len(col) and (np.diff(offs) >= 0).all()
    for c in range(D + 1):
        p = pos[offs[c]:offs[c + 1]]
        assert (col[p] == c).all() and (np.diff(row[p]) > 0).all()
    assert offs[D + 1] - offs[D] == n
    empty = np.setdiff1d(np.arange(D), X.indices)
    assert (offs[empty + 1] == offs[empty]).all()


# ------------------------------------------------------------------------------------------------------------------------
# GPU: exact data, bit for bit
# ------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def mb():
    import mlease_b200
    return mlease_b200


@pytest.fixture(scope="module")
def num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _exact(n, D, density, seed, w_choices=(1.0, 4.0), edit=None):
    rng = np.random.default_rng(seed)
    X = gr.random_pattern(n, D, density, rng).tolil()
    if edit is not None:
        edit(X)
    X = X.tocsr()
    X.eliminate_zeros()
    X.sort_indices()
    return gr.exact_values(X, w_choices, rng)


def _empty_rows(X):   # rows holding only the intercept
    X[::5, :] = 0
    X[40:72, :] = 0


def _empty_cols(X):   # columns 10 .. 139 (across the first block boundary) and the last column hold nothing
    X[:, 10:140] = 0
    X[:, X.shape[1] - 1] = 0


def _full_row(X):     # rows with every column: a suffix of D' words, many 32-word steps
    X[17, :] = 1.0
    X[X.shape[0] - 1, :] = 1.0


def _full_col(X):     # column 5 in every row: its walk has n positions
    X[:, 5] = 1.0


CASES = {
    "intercept-only rows and w = 0": (1000, 300, 0.01, (0.0, 1.0, 4.0), _empty_rows),
    "columns with no entries": (1000, 300, 0.02, (1.0, 4.0), _empty_cols),
    "rows with every column": (700, 300, 0.01, (1.0, 4.0), _full_row),
    "a column in every row": (1500, 200, 0.01, (1.0, 4.0), _full_col),
    "n % 32 != 0, bias at the start of a block": (32 * 37 + 13, 128, 0.03, (1.0, 4.0), None),
    "bias in the middle of a block": (1000, 191, 0.03, (1.0, 4.0), None),
    "bias at the end of a block": (1000, 127, 0.03, (1.0, 4.0), None),
    "bias at the end of block 1, D' = 256": (1000, 255, 0.03, (0.0, 1.0, 4.0), _full_row),
    "D' = 1001": (3000, 1000, 0.01, (1.0, 4.0), _full_col),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_exact_column_edges(mb, num_sms, name):
    n, D, dens, wc, edit = CASES[name]
    X, w = _exact(n, D, dens, sum(name.encode()), wc, edit)
    gr.check_limits(gr.gram_geometry(n, D, num_sms, True), X.nnz)
    gr.check_exact_premises(X, w, csr=True)
    _check_exact(_hessian(mb, X, w, D, SPARSE), X, w, D, name)


@pytest.mark.gpu
def test_exact_beyond_one_window(mb):
    """D' = 14 501 > the 14 336 cells of the accumulator: the low columns are walked in two windows; one row holds every column"""
    n, D = 400, 14_500
    assert (D + 1 + 127) // 128 * 128 > CELLS
    X, w = _exact(n, D, 0.002, 11, edit=_full_row)
    gr.check_exact_premises(X, w, csr=True)
    _check_exact(_hessian(mb, X, w, D, SPARSE), X, w, D, "two windows")


@pytest.mark.gpu
def test_second_build_leaves_no_stale_cell(mb):
    """A build at a generic point, then one at beta = 0 in the same session: the second equals its own exact Hessian"""
    n, D = 2000, 300
    X, w = _exact(n, D, 0.02, 5, edit=_full_row)
    rng = np.random.default_rng(6)
    beta = rng.normal(size=D + 1) * 0.3
    y = (np.arange(n) % 3 == 0).astype(np.int32)
    with mb.AdmmSession(1, D, [1.0]) as s:
        _set_kind(s, SPARSE)
        s.add_partition_csr(0, *gr.csr_arrays(X), y, np.asarray(w, np.float32), np.zeros(n, np.float32))
        H1 = s.objective(0, beta, np.zeros(D + 1), np.full(D + 1, Q), want_hessian=True)[2]
        H2 = s.objective(0, np.zeros(D + 1), np.zeros(D + 1), np.full(D + 1, Q), want_hessian=True)[2]
    assert not np.array_equal(H1, H2)
    _check_exact(H2, X, w, D, "second build")


@pytest.mark.gpu
def test_repeatable_across_sessions(mb):
    rng = np.random.default_rng(23)
    n, D = 30000, 1500
    X, w, o, beta = gr.generic_problem(n, D, 15.0 / D, rng)
    Hs = [_hessian(mb, X, w, D, SPARSE, o=o, beta=beta) for _ in range(2)]
    assert np.array_equal(Hs[0], Hs[1])


def _job(mb, parts, D, lambdas, kind, iters=2):
    with mb.AdmmSession(len(parts), D, lambdas) as s:
        _set_kind(s, kind)
        for p, (X, w) in enumerate(parts):
            n = X.shape[0]
            s.add_partition_csr(p, *gr.csr_arrays(X), (np.arange(n) % 3 == 0).astype(np.int32), np.asarray(w, np.float32))
        s.run(iters)
        return np.stack([s.z(l) for l in range(len(lambdas))])


@pytest.mark.gpu
def test_multi_lambda_job_is_repeatable_and_close_to_wgmma(mb):
    """Three lambdas of two partitions: the cold-start build makes only each group's leader Gram (share), later rebuilds run with
    some problems gated off.  Two runs agree bit for bit, and z stays within the e4m3 operand's reach of the wgmma kernel's."""
    parts = [_exact(3000, 400, 0.02, 40 + p) for p in range(2)]
    z2 = _job(mb, parts, 400, [0.5, 1.0, 4.0], SPARSE)
    assert np.array_equal(z2, _job(mb, parts, 400, [0.5, 1.0, 4.0], SPARSE))
    z1 = _job(mb, parts, 400, [0.5, 1.0, 4.0], 1)
    assert np.all(np.isfinite(z2))
    assert np.abs(z2 - z1).max() <= 1e-3 * max(1.0, np.abs(z1).max()), np.abs(z2 - z1).max()


@pytest.mark.gpu
def test_refused_above_the_column_id_limit(mb):
    """D' = 2^20 + 1: the upload builds no column index and a forced sparse kernel is refused; the rule takes the wgmma kernel"""
    n, D = 64, MAX_COLS
    rng = np.random.default_rng(2)
    rp = np.arange(n + 1, dtype=np.int64) * 2
    ci = np.sort(rng.choice(D, (n, 2), replace=False), axis=1).astype(np.int32).reshape(-1)
    v = np.ones(2 * n, np.float32)
    with mb.AdmmSession(1, D, [1.0]) as s:
        _set_kind(s, SPARSE)
        s.add_partition_csr(0, rp, ci, v, (np.arange(n) % 2).astype(np.int32))
        with pytest.raises(Exception, match="2\\^20"):
            s.time_kernel(0, "k1", reps=1)
