"""Plain float64 reference of the Gram kernels (ml-ease_b200/csrc/k2_gram.cu), shared by the Gram tests.

- Operand rounding: e4m3 (the CSR kernel's operand) and bf16 (the dense kernels' operand).
- The split-K geometry the kernels run: tile list, slice count, and the K-steps of every slice.
- Exact data: inputs on which every rounding step of the device Gram is exact, so that the device Hessian must equal
  X^T D X + diag(q) computed in float64 bit for bit.
- Generic data with an emulated operand, and the entrywise error measure |H - H_emu| / (|A|^T |A|).
"""
import functools
from collections import namedtuple

import numpy as np
import scipy.sparse as sp

CSR_STEP, DENSE_STEP = 32, 64   # data rows per K-step: SK (CSR, e4m3 m64n128k32) and GK (dense, bf16 TMA stage)
RING, CHAIN = 8, 4              # CSR ring stages (SST) and wgmma per fp32 promotion (S_CHAIN)
DENSE_MAX_FEATURES = 4095       # session.cu batch_alloc: k1_dense_plan's limit
# Entrywise bounds |H - H_emu| <= c |A|^T |A| of the e4m3 CSR Gram and the bf16 dense Gram: about 4x the largest excess
# test_gram_exact.py measured on an H100 80GB HBM3 (132 SMs, 400 W power limit): 3.04e-4 (CSR) and 3.6e-7 (dense wgmma)
ENTRYWISE_C_CSR = 1.2e-3
ENTRYWISE_C_DENSE = 1.5e-6


# ------------------------------------------------------------------------------------------------------------------------
# operand rounding
# ------------------------------------------------------------------------------------------------------------------------
def bf16_round(a):
    """Round-to-nearest-even of float32 values onto bf16 (__float2bfloat16_rn), returned as float32."""
    u = np.ascontiguousarray(a, np.float32).view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000
    return u.astype(np.uint32).view(np.float32)


def e4m3_round(a):
    """Round-to-nearest-even onto the e4m3 grid (3 mantissa bits, exponents 2^-6 .. 2^8, subnormal step 2^-9), saturating at
    448 like __nv_cvt_float_to_fp8(..., __NV_SATFINITE, __NV_E4M3)."""
    a = np.asarray(a, np.float64)
    mag = np.minimum(np.abs(a), 448.0)
    e = np.clip(np.floor(np.log2(np.maximum(mag, 2.0 ** -20))), -6, 8)
    step = 2.0 ** (e - 3)
    return np.sign(a) * np.minimum(np.round(mag / step) * step, 448.0)   # np.round = half to even


def csr_gram_scale(vmax, wmax):
    """The power-of-two operand scale of the CSR Gram (session.cu fill_problem_data): the largest |sqrt(d) x| goes to [112, 224)."""
    amax = np.float32(0.5) * np.sqrt(np.float32(max(wmax, 1e-30))) * np.float32(max(vmax, 1.0))
    e = np.frexp(np.float32(224.0) / amax)[1]
    return 2.0 ** int(min(60, max(-60, e - 1)))


# ------------------------------------------------------------------------------------------------------------------------
# split-K geometry
# ------------------------------------------------------------------------------------------------------------------------
Geometry = namedtuple("Geometry", "n D Dp ntiles slices nk")


def padded_width(D):
    """Dp of a session with D features: Dt = D + 1, ldx = round_up(Dt, 4) (session.cu mlease_session_create), Dp = round_up(ldx,
    128) (batch_alloc)."""
    ldx = -(-(D + 1) // 4) * 4
    return -(-ldx // 128) * 128


def tile_list(Dp, csr):
    """k2_gram.cu gram_tile_list: lower block-triangle tiles (bi, bj), 128 x 128 (CSR) or 128 x 256 (dense)."""
    cols = 128 if csr else 256
    return [(bi, bj) for bi in range(Dp // 128) for bj in range(-(-Dp // cols)) if bj * cols <= bi * 128 + 127]


def split_k_slices(n, ntiles, Dp, num_sms, nprob=1):
    """session.cu batch_alloc, 'Gram decomposition': the slice count.  It counts 64-row steps for both kernels."""
    ksteps = (max(n, 1) + 63) // 64
    base, cap = ntiles * nprob, max(1, num_sms)
    best, best_eff = 1, 0.0
    for s in range(1, 17):
        if s > ksteps:
            break
        ctas = base * s
        eff = ctas / (((ctas + cap - 1) // cap) * cap)
        if eff > best_eff + 1e-9:
            best_eff, best = eff, s
        if eff >= 0.93 and ctas >= 2 * cap:
            best = s
            break
    while best > 1 and best * Dp * Dp * 4.0 * nprob > 1024.0 ** 3:
        best -= 1
    return best


def slice_steps(n, slices, step):
    """K-steps of every slice: k2_gram.cu gram_wgmma_kernel / gram_csr_wgmma_kernel, 'ksteps_total .. nk'."""
    total = (n + step - 1) // step
    per = (total + slices - 1) // slices
    return [max(0, min(total, (s + 1) * per) - s * per) for s in range(slices)]


def gram_geometry(n, D, num_sms, csr):
    """The tiles, slices and per-slice K-steps (32 rows for CSR, 64 rows for dense) of one objective's Gram build."""
    Dp = padded_width(D)
    ntiles = len(tile_list(Dp, csr))
    slices = split_k_slices(n, ntiles, Dp, num_sms)
    return Geometry(n, D, Dp, ntiles, slices, slice_steps(n, slices, CSR_STEP if csr else DENSE_STEP))


def csr_paths(geom):
    """Which paths of the CSR consumer loop the slices of geom take: whole ring passes followed by a tail of r steps ('ring+r'),
    or a slice shorter than the ring ('nk=k', k < 8); 'single' is one slice of at least 500 steps (the production regime)."""
    t = {"ring+%d" % (k % RING) if k >= RING else "nk=%d" % k for k in geom.nk}
    if geom.slices == 1 and geom.nk[0] >= 500:
        t.add("single")
    return t


CSR_TARGETS = frozenset({"ring+%d" % r for r in range(RING)} | {"nk=%d" % k for k in range(RING)} | {"single"})


def readback_bytes(geom):
    """Host bytes of one Hessian read-back: every slice's fp32 partial (session.cu mlease_objective)."""
    return geom.slices * geom.Dp * geom.Dp * 4


def check_limits(geom, nnz=0, csr=True):
    """The documented limits a test shape must respect before it goes to the device."""
    assert csr or geom.D <= DENSE_MAX_FEATURES, geom
    assert nnz + geom.n < 2 ** 32 - 64, geom
    assert readback_bytes(geom) <= 512 << 20, geom


def _width(nb):
    return 128 * nb - 30   # D whose padded width is nb column blocks, the intercept inside the last block


@functools.lru_cache(maxsize=None)
def shapes_covering(num_sms):
    """Small (n, D) CSR shapes whose Gram builds on a device with num_sms SMs together take every path in CSR_TARGETS.
    Greedy: the candidate that adds the most new paths, the cheapest (n * Dp) first among equals."""
    cands = [(n, _width(nb)) for nb, top in ((1, 8400), (2, 3000), (3, 3000)) for n in range(1, top)]
    geoms = {c: gram_geometry(c[0], c[1], num_sms, True) for c in cands}
    paths = {c: csr_paths(g) for c, g in geoms.items()}
    chosen, covered = [], set()
    # the production regime: one slice of >= 500 steps; the narrowest width that runs one slice at n = 16 001
    for nb in range(1, 33):
        g = gram_geometry(16001, _width(nb), num_sms, True)
        if "single" in csr_paths(g) and readback_bytes(g) <= 256 << 20:
            chosen.append((16001, _width(nb)))
            covered |= csr_paths(g)
            break
    while covered != CSR_TARGETS:
        best = max(cands, key=lambda c: (len(paths[c] - covered), -c[0] * geoms[c].Dp))
        if not paths[best] - covered:
            break
        chosen.append(best)
        covered |= paths[best]
    return tuple(chosen)


def dense_shapes(num_sms):
    """Dense shapes for the bf16 Gram: a width with Dp = 128 mod 256 (the upper half of the last 128 x 256 tile is TMA's
    out-of-bounds fill), n not a multiple of 64, a slice with no K-step, and one slice at D = 4000."""
    shapes = [(1000, 300), (777, 100)]
    for n in range(65, 4000):   # the first n whose slices end in an empty one at D = 300
        if 0 in gram_geometry(n, 300, num_sms, False).nk:
            shapes.append((n, 300))
            break
    n = next(n for n in range(63, 0, -1) if gram_geometry(n, 4000, num_sms, False).slices == 1)
    shapes += [(n, 4000), (700, 4000)]
    return shapes


# ------------------------------------------------------------------------------------------------------------------------
# data sets
# ------------------------------------------------------------------------------------------------------------------------
def random_pattern(n, D, density, rng):
    """A random sparse pattern with sorted unique columns per row (scipy CSR)."""
    m = sp.random(n, D, density=density, format="csr", random_state=rng, data_rvs=lambda k: np.ones(k))
    m.sum_duplicates()
    m.sort_indices()
    return m


def exact_values(pattern, w_choices, rng):
    """Exact data on a pattern: values in {+-1, +-2}, weights drawn from w_choices (subsets of {0, 1, 4}).  At beta = 0 and
    offset = 0 the margin is 0, so d = w / 4 and sqrt(d) is in {0, 0.5, 1}: every e4m3 (x 2^6 .. 2^7) and bf16 operand is exact."""
    X = pattern.copy().astype(np.float64)
    X.data = rng.choice([-2.0, -1.0, 1.0, 2.0], size=X.nnz)
    w = rng.choice(np.asarray(w_choices, np.float64), size=X.shape[0])
    return X, w


def csr_arrays(X):
    """(rowptr int64, colidx int32, vals float32) of a scipy CSR matrix."""
    return X.indptr.astype(np.int64), X.indices.astype(np.int32), X.data.astype(np.float32)


def with_intercept(X):
    n = X.shape[0]
    if sp.issparse(X):
        return sp.hstack([X, sp.csr_matrix(np.ones((n, 1)))], format="csr")
    return np.hstack([np.asarray(X, np.float64), np.ones((n, 1))])


def exact_hessian(X, d, q):
    """X_b^T diag(d) X_b + diag(q) in float64, X_b = X with the intercept column."""
    Xb = with_intercept(X)
    d = np.asarray(d, np.float64)
    if sp.issparse(Xb) and Xb.nnz < 0.05 * np.prod(Xb.shape):
        G = (Xb.T @ sp.diags(d) @ Xb).toarray()
    else:
        Xb = Xb.toarray() if sp.issparse(Xb) else Xb
        G = Xb.T @ (Xb * d[:, None])
    return G + np.diag(q)


CSR_EDGE_CASES = ["empty rows, intercept-only group, empty block, w=0", "runs of 0..4096 entries per (block, group)",
                  "D=127", "D=128", "D=255", "D=256", "binary_feature"]


def csr_edge_case(name):
    """Exact CSR data at the structural edges of the operand assembly -> (X, w, D, binary_feature).  D = 127 / 255 put the
    intercept at the end of a column block, D = 128 / 256 alone in the next one."""
    rng = np.random.default_rng(sum(name.encode()))
    if name == "empty rows, intercept-only group, empty block, w=0":
        n, D = 1000, 300
        X, w = exact_values(random_pattern(n, D, 0.05, rng), (0.0, 1.0, 4.0), rng)
        X = X.tolil()
        X[96:128, :] = 0          # group 3 holds only the intercept entries
        X[::17, :] = 0            # scattered empty rows
        X[:, 128:256] = 0         # column block 1 has no entries at all
        X = X.tocsr()
        X.eliminate_zeros()
        return X, w, D, False
    if name == "runs of 0..4096 entries per (block, group)":
        n, D = 32 * 200 - 3, 255   # 16 slices of 13 K-steps: every stage is refilled, and cleared, at least once
        sizes = [63, 64, 65, 0, 4096, 1, 2, 65, 127, 128, 31]   # 11 is prime to the ring's 8 stages
        dense = np.zeros((n, D), np.float64)
        for grp in range(-(-n // 32)):
            r0 = 32 * grp
            rows = min(32, n - r0)
            k = min(sizes[grp % len(sizes)], rows * 128)
            cells = rng.choice(rows * 128, size=k, replace=False)
            dense[r0 + cells // 128, cells % 128] = 1.0
        dense[:, 128:] = rng.random((n, D - 128)) < 0.03
        X, w = exact_values(sp.csr_matrix(dense), (1.0, 4.0), rng)
        return X, w, D, False
    if name.startswith("D="):
        D = int(name[2:])
        X, w = exact_values(random_pattern(2000 - 11, D, 0.05, rng), (1.0, 4.0), rng)
        return X, w, D, False
    if name == "binary_feature":
        n, D = 3000, 300
        X = random_pattern(n, D, 0.04, rng)
        X.data = rng.normal(size=X.nnz) * 3.0   # stored values are ignored: every listed feature counts as 1
        w = rng.choice([1.0, 4.0], size=n)
        return X, w, D, True
    raise KeyError(name)


def check_exact_premises(X, w, csr, binary=False):
    """Everything that makes the device Gram exact on (X, w) at beta = 0, offset = 0: operands on the e4m3 / bf16 grid, every
    128-row chain sum below 2^11 units of 2^10 (e4m3) and every fp32 total exact.  Returns the operand matrix (with intercept)."""
    sd = np.sqrt(np.asarray(w, np.float64) / 4.0)
    assert np.all(np.isin(sd, [0.0, 0.5, 1.0]))
    Xb = with_intercept(X)
    if binary and sp.issparse(Xb):
        Xb = Xb.copy()
        Xb.data[:] = 1.0
    vals = Xb.data if sp.issparse(Xb) else Xb[Xb != 0]
    assert np.all(np.isin(np.abs(vals), [1.0, 2.0]))
    A = (sp.diags(sd) @ Xb).tocsr() if sp.issparse(Xb) else Xb * sd[:, None]
    a = A.data if sp.issparse(A) else A.ravel()
    n = X.shape[0]
    if csr:
        vmax = 1.0 if binary else float(np.abs(X.data).max() if X.nnz else 0.0)
        g = csr_gram_scale(vmax, float(np.max(w)))
        op = a * g
        assert np.array_equal(e4m3_round(op), op)
        unit = 2.0 ** 10                                             # the smallest product: 32 x 32
        assert np.all(np.isin(np.abs(op[op != 0]), [32.0, 64.0, 128.0])), np.unique(np.abs(op))
        top = float(np.abs(op).max()) ** 2                         # the largest product
        assert top * 128 <= 2 ** 11 * unit                           # a chain of 4 x 32 rows: at most 2^11 units
        assert top * n < 2 ** 24 * unit                              # fp32 total of a slice: an exact integer count of units
    else:
        op = a.astype(np.float32)
        assert np.array_equal(bf16_round(op), op)
        assert np.all(np.isin(np.abs(op[op != 0]), [0.5, 1.0, 2.0]))
        assert float(np.abs(op).max()) ** 2 * n < 2 ** 24 * 0.25   # products are multiples of 2^-2: exact fp32 sums
    return A


def generic_problem(n, D, density, rng, heavy=None):
    """Generic data: normal values, w in U(0.5, 2), a nonzero point and nonzero offsets.  heavy: one stored value set to it."""
    X = random_pattern(n, D, density, rng) if density < 1 else sp.csr_matrix(np.ones((n, D)))
    X = X.astype(np.float64)
    X.data = rng.normal(size=X.nnz).astype(np.float32).astype(np.float64)
    if heavy is not None and X.nnz:
        X.data[X.nnz // 2] = heavy
    w = rng.uniform(0.5, 2.0, n).astype(np.float32)
    o = rng.normal(0, 0.1, n).astype(np.float32)
    k = max(1.0, X.nnz / max(n, 1))
    beta = rng.normal(0, 0.3 / np.sqrt(k), D + 1)
    return X, w, o, beta


def sqrt_d(X, w, o, beta):
    """sqrt(w p (1 - p)) at the margin X_b beta + o, in float64."""
    t = with_intercept(sp.csr_matrix(X)) @ beta + np.asarray(o, np.float64)
    p = 1.0 / (1.0 + np.exp(-np.abs(t)))
    return np.sqrt(np.asarray(w, np.float64) * p * (1.0 - p))


def emulated_operand(X, w, o, beta, csr, rel=2.0 ** -17, sd=None):
    """The device's Gram operand for generic data, rescaled to X's units: sqrt(d) from the margin in float64, rounded to
    float32, times the value, rounded to e4m3 (CSR, with the library's power-of-two scale) or bf16 (dense).
    Returns (A, slack): sqrt(d) on the device differs from this one in its last float32 bits, so an operand that lies within
    rel of a rounding midpoint may round the other way; slack bounds what that can change in every Gram entry.
    sd: use these sqrt(d) instead of the ones at the margin."""
    Xb = with_intercept(sp.csr_matrix(X))
    sd = sqrt_d(X, w, o, beta) if sd is None else sd
    if csr:
        g = csr_gram_scale(float(np.abs(X.data).max()), float(np.max(w)))
        rnd = lambda s: e4m3_round((Xb.data * np.repeat(s * g, np.diff(Xb.indptr))).astype(np.float32)) / g
    else:
        rnd = lambda s: bf16_round((Xb.data * np.repeat(s, np.diff(Xb.indptr))).astype(np.float32)).astype(np.float64)
    mid = rnd(sd.astype(np.float32).astype(np.float64))
    lo, hi = rnd(sd * (1 - rel)), rnd(sd * (1 + rel))
    mk = lambda data: sp.csr_matrix((data, Xb.indices.copy(), Xb.indptr.copy()), shape=Xb.shape)
    A = mk(mid)
    amb = mk(np.abs(hi - lo))
    amb.eliminate_zeros()
    big = mk(np.maximum(np.maximum(np.abs(lo), np.abs(hi)), np.abs(mid)))
    slack = np.asarray((big.T @ amb).toarray() if big.nnz < 0.05 * np.prod(big.shape) else amb.T @ big.toarray()).T
    return A, slack + slack.T


def gram(A):
    """A^T A in float64, sparse or through BLAS, whichever suits A's density."""
    if sp.issparse(A) and A.nnz > 0.05 * np.prod(A.shape):
        A = A.toarray()
    return (A.T @ A).toarray() if sp.issparse(A) else A.T @ A


def entrywise_excess(H, H_emu, A, slack=0.0):
    """|H - H_emu| / (|A|^T |A|) entry by entry, A the emulated operand.  slack (same shape) is first taken off |H - H_emu|:
    see emulated_operand.  Entries with no product at all must match exactly (inf otherwise)."""
    absA = abs(A)
    den = gram(absA)
    num = np.maximum(np.abs(np.asarray(H, np.float64) - H_emu) - slack, 0.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(den > 0, num / np.where(den > 0, den, 1.0), np.where(num > 0, np.inf, 0.0))


def lower_mirror(P):
    """The Hessian the host assembles from a Gram partial: the lower triangle, mirrored (session.cu mlease_objective)."""
    return np.tril(P) + np.tril(P, -1).T
