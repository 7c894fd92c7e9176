"""The sparse CSR Gram's operand word (k2_gram.cu sparse_word) and the spans shorter than 8 groups whose rows it encodes.

For a sparse-kernel batch the operand pass writes one 32-bit word per entry of the block-major list: the e4m3 value in integer
units of 2^-9 as an fp32 (whose low 20 mantissa bits are always zero), with the entry's row in its span (32 (group mod span) +
row in group, 8 bits) and its column in the 128-column block (7 bits) in the low 15 bits.  gram_csr_sparse_kernel decodes it
with masks, a shift and one float-to-int conversion.

The CPU tests pin a numpy transcription of the encoder and the decoder, exhaustively over the e4m3 codes, against the byte decode
of test_gram_sparse.py (itself pinned against torch), and check that each span case below reaches the span it is named after.
The GPU tests run the span cases through both CSR Gram kernels, forced with the library's test hook, and require
X^T D X + diag(q) bit for bit."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gram_reference as gr  # noqa: E402
from test_gram_sparse import KINDS, _check_exact, _hessian, e4m3_units  # noqa: E402
from test_gram_sparse_spans import STAGE, sparse_span  # noqa: E402

VALUE_MASK = 0xFFFF8000


# ------------------------------------------------------------------------------------------------------------------------
# CPU: the word format
# ------------------------------------------------------------------------------------------------------------------------
def encode(byte, row_in_span, col):
    """k2_gram.cu sparse_word"""
    f = np.array([e4m3_units(byte)], np.float32).view(np.uint32)[0]
    return int(f) | (row_in_span << 7) | col


def decode(w):
    """k2_gram.cu sw_units, sw_row, sw_col: (units, row in span, column); the conversion truncates toward zero (F2I.TRUNC)"""
    units = int(np.trunc(np.array([w & VALUE_MASK], np.uint32).view(np.float32)[0]))
    return units, (w >> 7) & 255, w & 127


def test_word_round_trip_every_code():
    for b in range(256):
        u = e4m3_units(b)
        f = int(np.array([u], np.float32).view(np.uint32)[0])
        assert f & ~VALUE_MASK & 0xFFFFFFFF == 0 and (f >> 15) & 31 == 0, hex(b)   # the low 20 mantissa bits are free
        for row in (0, 31, 32, 255):
            for col in (0, 127):
                w = encode(b, row, col)
                assert w < 2 ** 32
                assert decode(w) == (u, row, col), (hex(b), row, col, decode(w), u)


def test_word_codes_cover_the_edges():
    units = {b: e4m3_units(b) for b in range(256)}
    assert units[0x00] == 0 and units[0x80] == 0             # both zeros decode to 0 (the sparse kernel skips them)
    assert units[0x01] == 1 and units[0x81] == -1            # the smallest subnormals
    assert units[0x7E] == 229376 and units[0xFE] == -229376  # +-448
    assert encode(0x80, 0, 0) == 0                           # -0 is integer 0 units: an all-zero word
    assert decode(encode(0x80, 255, 127)) == (0, 255, 127)


# ------------------------------------------------------------------------------------------------------------------------
# spans shorter than 8 groups
# ------------------------------------------------------------------------------------------------------------------------
CASES = ["span 5", "span 2", "span 1"]
# per case: rows, light rows' entries in block 0 and in block 1 (columns 128 .. 199), the dense rows (first, count) of the first
# span and their entries in block 0.  D = 200: two 128-column blocks, the intercept (column 200) in block 1
GEOMETRY = {
    # 158 groups, 158 % 5 = 3: a short last span of 3 groups (the last one 13 rows).  The first span's block-0 range is rows
    # 0 .. 9 (2 each), rows 10 .. 29 (40 each), rows 30 .. 159 (2 each): 20 + 800 + 260 entries, so the 448-entry chunk boundary
    # falls after 428 = 40 * 10 + 28 dense entries, inside row 20
    "span 5": (5 * 32 * 31 + 2 * 32 + 13, 2, 1, (10, 20), 40),
    # 81 groups, the last span one group of 5 rows.  First span (64 rows): 3 * 6 + 4 * 60 + 57 * 6 = 600 entries in block 0; the
    # boundary falls after 190 = 6 * 31 + 4 entries of the light rows from row 7 on, inside row 38
    "span 2": (64 * 40 + 5, 6, 2, (3, 4), 60),
    # 61 groups (the last one 19 rows).  First span (32 rows): 2 * 10 + 3 * 70 + 27 * 10 = 500 entries in block 0; the boundary
    # falls after 218 = 10 * 21 + 8 entries of the light rows from row 5 on, inside row 26
    "span 1": (32 * 60 + 19, 10, 2, (2, 3), 70),
}
D = 200


def case(name):
    """Exact CSR data -> (X, w, D)."""
    n, k0, k1, (d0, dn), kd = GEOMETRY[name]
    rng = np.random.default_rng(sum(name.encode()))
    dense = np.zeros((n, D), np.float64)
    for r in range(n):
        if d0 <= r < d0 + dn:
            dense[r, rng.choice(128, size=kd, replace=False)] = 1.0
        else:
            dense[r, rng.choice(128, size=k0, replace=False)] = 1.0
            dense[r, 128 + rng.choice(D - 128, size=k1, replace=False)] = 1.0
    return (*gr.exact_values(sp.csr_matrix(dense), (1.0, 4.0), rng), D)


@pytest.mark.parametrize("name", CASES)
def test_span_cases_are_exact(name):
    X, w, D_ = case(name)
    gr.check_exact_premises(X, w, csr=True)
    gr.check_limits(gr.gram_geometry(X.shape[0], D_, 132, True), X.nnz)


@pytest.mark.parametrize("name", CASES)
def test_span_cases_reach_their_span(name):
    X, _, D_ = case(name)
    n = X.shape[0]
    span = sparse_span(n, D_, X.nnz)
    assert span == int(name.split()[1])
    ngroups = -(-n // 32)
    assert n % 32 != 0   # the last group is short
    if span > 1:
        assert ngroups % span != 0   # and so is the last span
    # the first span's block-0 range in list order (rows ascending) is longer than a stage chunk, and the chunk boundary falls
    # inside a row
    Xb = gr.with_intercept(X).tocsr()
    rows = np.repeat(np.arange(n), np.diff(Xb.indptr))
    blk = Xb.indices // 128
    first = rows[(blk == 0) & (rows < 32 * span)]
    assert len(first) > STAGE and first[STAGE - 1] == first[STAGE]
    # the rows of a span are below 256: the word's 8-bit row field
    assert 32 * span <= 256


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
def test_exact_short_spans(mb, num_sms, kind, name):
    X, w, D_ = case(name)
    gr.check_limits(gr.gram_geometry(X.shape[0], D_, num_sms, True), X.nnz)
    gr.check_exact_premises(X, w, csr=True)
    _check_exact(_hessian(mb, X, w, D_, KINDS[kind]), X, w, D_, (kind, name))
