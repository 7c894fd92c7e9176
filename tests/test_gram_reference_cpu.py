"""CPU checks of the Gram test harness (gram_reference.py): the operand rounding against torch's e4m3 / bf16 casts, the
geometry mirror and its coverage, the exactness premises of every exact data set, and that the exact check and the entrywise
bound catch the tiling and pipeline bugs they exist for.  The bugs are applied to the emulated operand or Gram here, never to
the kernel: a broken ring or parity bit on the device hangs it instead of returning a wrong Hessian."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gram_reference as gr  # noqa: E402


def _torch_round(x, dtype):
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(dtype).to(torch.float32).numpy()


def _with_neighbours(v):
    v = np.asarray(v, np.float32)
    return np.concatenate([v, np.nextafter(v, np.float32(np.inf)), np.nextafter(v, np.float32(-np.inf))])


# ------------------------------------------------------------------------------------------------------------------------
# operand rounding
# ------------------------------------------------------------------------------------------------------------------------
def test_e4m3_round_matches_torch():
    codes = torch.arange(256, dtype=torch.uint8).view(torch.float8_e4m3fn).to(torch.float32).numpy()
    pos = np.unique(np.abs(codes[np.isfinite(codes)]))                      # 0, the subnormals, ..., 448
    mids = (pos[:-1].astype(np.float64) + pos[1:]) / 2                     # the ties, exact in float32
    rng = np.random.default_rng(0)
    rand = np.concatenate([rng.uniform(-448, 448, 100000), np.exp(rng.uniform(np.log(2.0 ** -12), np.log(448.0), 100000))])
    x = _with_neighbours(np.concatenate([pos, mids, rand]))
    x = np.concatenate([x, -x])
    x = x[np.abs(x) <= 448]                                                # torch does not saturate; the kernel's cast does
    assert np.array_equal(gr.e4m3_round(x), _torch_round(x, torch.float8_e4m3fn))
    assert np.array_equal(gr.e4m3_round([500.0, -1e6, 449.0]), [448.0, -448.0, 448.0])   # __NV_SATFINITE


def test_bf16_round_matches_torch():
    hi = np.arange(1 << 16, dtype=np.uint32) << 16
    codes = hi.view(np.float32)
    fin = np.isfinite(codes)
    mids = (hi | 0x8000).view(np.float32)                                   # halfway between a code and the next
    rng = np.random.default_rng(1)
    rand = (rng.normal(size=200000) * np.exp(rng.uniform(-80, 80, 200000))).astype(np.float32)
    x = _with_neighbours(np.concatenate([codes[fin], mids[fin & np.isfinite(mids)], rand]))
    x = x[np.isfinite(x)]
    assert np.array_equal(gr.bf16_round(x), _torch_round(x, torch.bfloat16), equal_nan=True)


# ------------------------------------------------------------------------------------------------------------------------
# geometry
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,D,slices,nk", [(1000, 50, 16, {2}), (333, 255, 6, {1, 2}), (3000, 700, 6, {14, 16}),
                                           (3000, 300, 16, {4, 6}), (20000, 4000, 1, {625})])
def test_csr_geometry_on_132_sms(n, D, slices, nk):
    g = gr.gram_geometry(n, D, 132, True)
    assert (g.slices, set(g.nk)) == (slices, nk)
    assert sum(g.nk) == -(-n // 32)


@pytest.mark.parametrize("num_sms", [132, 114])
def test_shapes_cover_every_consumer_path(num_sms):
    covered = set()
    for n, D in gr.shapes_covering(num_sms):
        g = gr.gram_geometry(n, D, num_sms, True)
        gr.check_limits(g, n * 13)
        covered |= gr.csr_paths(g)
    assert covered == gr.CSR_TARGETS, gr.CSR_TARGETS - covered
    seen = set()
    for n, D in gr.dense_shapes(num_sms):
        g = gr.gram_geometry(n, D, num_sms, False)
        gr.check_limits(g, csr=False)
        seen |= {"Dp%256=128"} if g.Dp % 256 == 128 else set()
        seen |= {"n%64"} if n % 64 else set()
        seen |= {"nk=0"} if 0 in g.nk else set()
        seen |= {"one slice, D=4000"} if g.slices == 1 and D == 4000 else set()
    assert seen == {"Dp%256=128", "n%64", "nk=0", "one slice, D=4000"}, seen


# ------------------------------------------------------------------------------------------------------------------------
# exactness premises of the data sets the GPU tests build
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", gr.CSR_EDGE_CASES)
def test_edge_cases_are_exact(name):
    X, w, D, binary = gr.csr_edge_case(name)
    gr.check_exact_premises(X, w, csr=True, binary=binary)
    gr.check_limits(gr.gram_geometry(X.shape[0], D, 132, True), X.nnz)


def test_exact_builders_stay_on_the_grid():
    rng = np.random.default_rng(2)
    for w_choices in [(1.0, 4.0), (1.0,), (4.0,), (0.0, 1.0, 4.0)]:
        X, w = gr.exact_values(gr.random_pattern(300, 200, 0.1, rng), w_choices, rng)
        gr.check_exact_premises(X, w, csr=True)
        gr.check_exact_premises(X.toarray(), w, csr=False)
    with pytest.raises(AssertionError):   # a value off the grid is refused
        X.data[0] = 3.0
        gr.check_exact_premises(X, w, csr=True)


# ------------------------------------------------------------------------------------------------------------------------
# sensitivity: every corruption below must fail the exact check, and the entrywise bound on generic data
# ------------------------------------------------------------------------------------------------------------------------
N, D = 5000 - 7, 300   # 6 CSR tiles, 16 slices of 10 K-steps: stages are refilled; column blocks 0-127, 128-255, 256-300
GEOM = gr.gram_geometry(N, D, 132, True)
PER = GEOM.nk[0]
Dt = D + 1


def _rows(g):
    return slice(32 * g, min(32 * g + 32, N))


def _blk(b):
    return slice(128 * b, min(128 * b + 128, Dt))


def _tile_add(G, bi, bj, Ai, Aj):
    """Add Ai^T Aj into tile (bi, bj) of the partial and assemble the Hessian from its lower triangle, as the host does."""
    P = G.copy()
    P[_blk(bi), _blk(bj)] += Ai[:, _blk(bi)].T @ Aj[:, _blk(bj)]
    return gr.lower_mirror(P)


def _drop_group(A, pattern, sd_fn):          # one 32-row group missing from one tile
    g = 2 * PER + 3
    return _tile_add(A.T @ A, 2, 1, -A[_rows(g)], A[_rows(g)])


def _neighbour_sqrt_d(A, pattern, sd_fn):    # one row scaled with its neighbour's sqrt(d) (a wrong kmaj_row lane)
    sd, operand = sd_fn
    r = next(r for r in range(32 * PER + 5, N - 1) if sd[r] != sd[r + 1] and pattern[r, :D].any())
    sd2 = sd.copy()
    sd2[r] = sd[r + 1]
    B = operand(sd2)
    return B.T @ B


def _stale_stage(A, pattern, sd_fn):         # K-step 8 of a slice finds the bytes of K-step 0 where it writes none
    g_new, g_old = PER + 8, PER
    assert 8 < PER
    def stale(blk):
        new, old = A[_rows(g_new), _blk(blk)].copy(), A[_rows(g_old), _blk(blk)]
        keep = ~pattern[_rows(g_new), _blk(blk)]
        new[keep] = old[keep]
        return new
    P = A.T @ A
    a_new, b_new = A[_rows(g_new), _blk(2)], A[_rows(g_new), _blk(1)]
    P[_blk(2), _blk(1)] += stale(2).T @ stale(1) - a_new.T @ b_new
    return gr.lower_mirror(P)


def _chain_twice(A, pattern, sd_fn):         # one chain of 4 K-steps promoted into the fp32 sum twice
    rows = slice(32 * (PER + 4), 32 * (PER + 8))
    return _tile_add(A.T @ A, 1, 0, A[rows], A[rows])


def _intercept_missing(A, pattern, sd_fn):   # the intercept entries of one group are missing from the entry list
    B = A.copy()
    B[_rows(3 * PER + 1), D] = 0.0
    return B.T @ B


def _slice_boundary(A, pattern, sd_fn):      # slice 2 starts one group early: the last group of slice 1 counts twice
    g = 2 * PER - 1
    return A.T @ A + A[_rows(g)].T @ A[_rows(g)]


CORRUPTIONS = [_drop_group, _neighbour_sqrt_d, _stale_stage, _chain_twice, _intercept_missing, _slice_boundary]


def _operand(X, w, o, beta, csr):
    pattern = gr.with_intercept(X).toarray() != 0
    operand = lambda sd: gr.emulated_operand(X, w, o, beta, csr, sd=sd)[0].toarray()
    A, slack = gr.emulated_operand(X, w, o, beta, csr)
    return A, slack, pattern, (gr.sqrt_d(X, w, o, beta), operand)


@pytest.fixture(scope="module", params=[True, False], ids=["csr", "dense"])
def exact_and_generic(request):
    csr = request.param
    rng = np.random.default_rng(3)
    X, w = gr.exact_values(gr.random_pattern(N, D, 0.05, rng), (1.0, 4.0), rng)
    gr.check_exact_premises(X, w, csr=csr)
    exact = _operand(X, w, np.zeros(N), np.zeros(Dt), csr)
    Xg, wg, og, bg = gr.generic_problem(N, D, 0.05, rng)
    return csr, exact, _operand(Xg, wg, og, bg, csr)


def test_sensitivity_geometry():
    assert GEOM.slices >= 4 and PER > 8 and GEOM.Dp == 384 and GEOM.ntiles == 6


@pytest.mark.parametrize("corrupt", CORRUPTIONS, ids=[c.__name__.strip("_") for c in CORRUPTIONS])
def test_corruption_is_caught(exact_and_generic, corrupt):
    csr, (A, _, pat, sd_fn), (Ag, slack, patg, sd_fng) = exact_and_generic
    Ad = A.toarray()
    G = Ad.T @ Ad
    assert np.array_equal(gr.lower_mirror(G), G)            # the harness itself: an intact Gram passes
    assert not np.array_equal(corrupt(Ad, pat, sd_fn), G), "the exact check misses it"
    Agd = Ag.toarray()
    G_emu = Agd.T @ Agd
    c = gr.ENTRYWISE_C_CSR if csr else gr.ENTRYWISE_C_DENSE
    assert gr.entrywise_excess(G_emu, G_emu, Ag, slack).max() == 0.0
    excess = gr.entrywise_excess(corrupt(Agd, patg, sd_fng), G_emu, Ag, slack).max()
    assert excess > c, ("the entrywise bound misses it", excess, c)
