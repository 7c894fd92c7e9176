"""fp64 reference of the factored Newton direction of wide systems (ldh > 2048).

There the solver never forms H^-1.  The Cholesky factor L of H stays in fp64, Y = L^-1 is built by a recursive inverse whose
merges run in TF32 (merge_tf32_kernel), and Y is stored as bf16 in symmetric storage (ysym_kernel): M[i][j] = Y[max(i,j)][min(i,j)].
Each direction is then Y^T (Y q) by two triangular GEMVs over M (newton_gemv_tri_kernel):
  phase 0   t[r]   = float( sum_{k <= r} M[r][k] qf[k] )      (lower half; qf = float(q))
  phase 1   dir[c] =        sum_{k >= c} M[c][k] t[k]          (upper half, fed with the t phase 0 stored)

Error bound of one output entry (derivation).  Per row, lane l of the warp takes the 8-element chunks k = kbeg + 8 l + 256 i, so a
lane forms at most n = 8 ceil((kend - kbeg) / 256) products.  A bf16 operand times an fp32 vector element is exact in fp32's
24-bit significand only for the vector's leading 16 bits, so the lane's sum is an fp32 FMA chain p = fma(h, x, p) from p = 0:
one rounding per step, |chain - exact| <= gamma_n sum |h x| with gamma_n = n u / (1 - n u), u = 2^-24.  The 32 lane sums are
added in fp64 (warp_sum): 31 roundings of 2^-53, covered by a 1e-13 relative slack.  Phase 0 then rounds the sum to float once:
another u (|exact| + gamma_n sum |h x|).  Phase 0 ranges are [0, min(r0 + 4, Dt)) and phase 1 ranges [r0 & ~7, Dt), with r0 the
first row of the row's 4-row block.  The reference sums themselves are taken in fp64 over exact fp64 products (bf16 x fp32 has at
most 32 significant bits).

Exactly representable factors.  L = I + E with E strictly lower triangular, dyadic entries (+-1/2, +-1/4, +-3/4), and the row
indices of its nonzeros disjoint from its column indices.  Then E^2 = 0, so Y = L^-1 = I - E exactly, H = L L^T has unit pivots and
is exact in fp64, and every product and partial sum of the fp64 factorisation, of the fp64 leaf inverses and of the TF32 merges is
exact (a merge's sums have one nonzero term each: the others are entries of E^2).  On such data Lc, Yinv and Ysym have known bits.
"""
import numpy as np
import scipy.sparse as sp

from gram_reference import bf16_round

WLEAF = 256     # leaf of the recursive inverse (k3_cholesky.cu)
TILE = 128      # TF32 merge tile (TM = TN)
GEMV_RB = 4     # rows per warp block of the triangular GEMVs
U32 = 2.0 ** -24
VALUES = (0.5, -0.25, 0.75, -0.5, 0.25, -0.75)


def ldh_of(Dt):
    return (Dt + 31) // 32 * 32


def merges(ldh):
    """(m, r0, m2) of every merge of the recursive inverse, in the order cholesky_launch_wide runs them: the diagonal blocks
    [r0, r0 + m) and [r0 + m, r0 + m + m2) become one."""
    out, m = [], WLEAF
    while m < ldh:
        for y in range((ldh + 2 * m - 1) // (2 * m)):
            r0 = 2 * y * m
            m2 = min(m, ldh - r0 - m)
            if m2 > 0:
                out.append((m, r0, m2))
        m *= 2
    return out


def exact_pairs(Dt):
    """Nonzeros {(i, j): value} of E (i > j, rows and columns disjoint) that cover: every merge (its L21 block holds a pair, at
    the block's corners and across its first tile boundary), a pair inside every leaf with two rows, both edges of the 128-wide
    tiles in rows and columns, row Dt - 1 and column 0."""
    R, C, pairs = set(), set(), {}

    def add(ti, tj, ilo=0, ihi=None, jlo=0, jhi=None):
        ihi = Dt if ihi is None else min(ihi, Dt)
        jhi = Dt if jhi is None else jhi
        for d in range(128):   # nearest free position to the target (L1 distance d), inside the block
            for i, j in ((ti + di, tj + s * (d - abs(di))) for di in range(-d, d + 1) for s in (1, -1)):
                if ilo <= i < ihi and jlo <= j < jhi and 0 <= j < i and i not in C and j not in R and (i, j) not in pairs:
                    R.add(i); C.add(j); pairs[(i, j)] = VALUES[len(pairs) % len(VALUES)]
                    return
        raise AssertionError("no free position near (%d, %d)" % (ti, tj))

    add(Dt - 1, 0)
    for m, r0, m2 in merges(ldh_of(Dt)):
        a, e = r0 + m, min(r0 + m + m2, Dt) - 1
        blk = dict(ilo=a, ihi=e + 1, jlo=r0, jhi=r0 + m)
        add(a, r0 + m - 1, **blk)
        add(e, r0, **blk)
        if e - a >= TILE:
            add(a + TILE - 1, r0 + TILE, **blk)
            add(a + TILE, r0 + TILE - 1, **blk)
    for l0 in range(0, Dt, WLEAF):
        if min(l0 + WLEAF, Dt) - l0 >= 2:
            add(min(l0 + WLEAF, Dt) - 1 - 5, l0 + 3, ilo=l0, ihi=l0 + WLEAF, jlo=l0, jhi=l0 + WLEAF)
    return pairs


def coverage(Dt, pairs):
    """What the pairs reach: {name: bool}."""
    ij = np.array(list(pairs.keys()))
    i, j = ij[:, 0], ij[:, 1]
    cov = {"row Dt-1": bool((i == Dt - 1).any()), "column 0": bool((j == 0).any()),
           "within-leaf": bool((i // WLEAF == j // WLEAF).any()),
           "tile first row": bool((i % TILE == 0).any()), "tile last row": bool((i % TILE == TILE - 1).any()),
           "tile first column": bool((j % TILE == 0).any()), "tile last column": bool((j % TILE == TILE - 1).any())}
    for m, r0, m2 in merges(ldh_of(Dt)):
        cov["merge m=%d r0=%d m2=%d" % (m, r0, m2)] = bool(((i >= r0 + m) & (i < r0 + m + m2) & (j >= r0) & (j < r0 + m)).any())
    return cov


def exact_system(Dt, pairs):
    """(E sparse, H dense fp64) with H = (I + E)(I + E)^T."""
    ij = np.array(list(pairs.keys()))
    E = sp.csr_matrix((np.array(list(pairs.values())), (ij[:, 0], ij[:, 1])), shape=(Dt, Dt))
    Hs = sp.identity(Dt, format="csr") + E + E.T + E @ E.T
    return E, Hs.toarray()


def ysym_bits(Y, ldh):
    """The bf16 symmetric storage ysym_kernel writes for the lower-triangular Y (Dt x Dt): identity on the padding."""
    Dt = Y.shape[0]
    M = np.eye(ldh, dtype=np.float64)
    M[:Dt, :Dt] = np.tril(Y)
    M = np.where(np.tri(ldh, dtype=bool), M, M.T)   # (a select, not a sum: -0.0 entries keep their sign bit)
    return (bf16_round(M.astype(np.float32)).view(np.uint32) >> 16).astype(np.uint16)


def exact_ysym_bits(ldh, pairs):
    """ysym_bits of Y = I - E straight from the pairs (no dense Y: the 10k-wide case)."""
    bits = np.zeros((ldh, ldh), np.uint16)
    bits[np.arange(ldh), np.arange(ldh)] = 0x3F80   # bf16 1.0
    for (i, j), v in pairs.items():
        b = np.array([-v], np.float32).view(np.uint32)[0] >> 16   # dyadic: exact in bf16
        bits[i, j] = bits[j, i] = b
    return bits


def bits_to_float(bits):
    return (bits.astype(np.uint32) << 16).view(np.float32).astype(np.float64)


def gamma(n):
    n = np.asarray(n, np.float64)
    return n * U32 / (1.0 - n * U32)


def chunk_terms(Dt, phase):
    """n per row: 8 ceil(range / 256) products in one lane's FMA chain."""
    r0 = (np.arange(Dt) // GEMV_RB) * GEMV_RB
    rng = np.minimum(r0 + GEMV_RB, Dt) if phase == 0 else Dt - (r0 & ~7)
    return 8 * ((rng + 255) // 256)


def halves(bits, Dt):
    """(lower incl. diagonal, upper incl. diagonal) of the first Dt rows / columns of a Ysym image, as float32 (bf16 values are
    exact there; half the host memory of fp64 at the 10k width)."""
    M = (bits[:Dt, :Dt].astype(np.uint32) << 16).view(np.float32)
    return np.tril(M), np.triu(M)


def _gemv(M, x, rows=1024):
    """(x @ M^T, |x| @ |M|^T) in fp64 over row blocks of M (no full-size fp64 copy of M)."""
    x = np.asarray(x, np.float64)
    n = M.shape[0]
    exact = np.empty(x.shape[:-1] + (n,))
    s = np.empty_like(exact)
    for r in range(0, n, rows):
        blk = M[r:r + rows].astype(np.float64)
        exact[..., r:r + rows] = x @ blk.T
        s[..., r:r + rows] = np.abs(x) @ np.abs(blk).T
    return exact, s


def phase0(lo, q):
    """(fp64 value of t before its float rounding, entrywise bound on |t_gpu - value|) for vectors q[..., Dt]."""
    exact, s = _gemv(lo, np.asarray(q, np.float32))
    g = gamma(chunk_terms(lo.shape[0], 0))
    return exact, g * s + U32 * (np.abs(exact) + g * s) + 1e-13 * s


def phase1(up, t):
    """(fp64 value of dir, entrywise bound on |dir_gpu - value|), fed with the stored float t[..., Dt]."""
    exact, s = _gemv(up, np.asarray(t, np.float32))
    return exact, gamma(chunk_terms(up.shape[0], 1)) * s + 1e-13 * s


# TF32 merges.  Each operand is rounded double -> float (RN, 2^-24) -> tf32 (cvt.rna, 2^-11): relative error u_t <= 2^-11 + 2^-24,
# so a product of two rounded operands is within 2 u_t + u_t^2 of the exact one.  The tensor cores accumulate in fp32 without a
# guaranteed round-to-nearest: one ulp (2^-23) per addition, gamma_K over the K products of an output.  Mode 1 (T = L21 Y11) is
# thus within c_m |L21| |Y11| of the fp64 product of the GPU's own operands, and mode 2 (Y21 = -Y22 T, T itself inexact) within
# |Y22| bound_T + c_m2 |Y22| (|T| + bound_T).  Every operand of a merge is final when the merge runs (later merges write other
# blocks), so each merge is checked against the GPU's own Lc and Yinv.
U_TF32 = 2.0 ** -11 + 2.0 ** -24


def _c_merge(K):
    return 2 * U_TF32 + U_TF32 ** 2 + K * 2.0 ** -23 / (1 - K * 2.0 ** -23)


def merge_excess(Lc, Y):
    """max over every merge block of |Y21_gpu - (-Y22 L21 Y11)| / bound (Lc, Y: the ldh x ldh padded factor and inverse)."""
    worst = 0.0
    for m, r0, m2 in merges(Lc.shape[0]):
        a, e = r0 + m, r0 + m + m2
        L21, Y11, Y22 = Lc[a:e, r0:a], Y[r0:a, r0:a], Y[a:e, a:e]
        T = L21 @ Y11
        bT = _c_merge(m) * (np.abs(L21) @ np.abs(Y11))
        ref = -(Y22 @ T)
        aY = np.abs(Y22)
        bY = aY @ bT + _c_merge(m2) * (aY @ (np.abs(T) + bT)) + 1e-13 * (aY @ np.abs(T))
        worst = max(worst, excess(Y[a:e, r0:a], ref, bY))
    return worst


def excess(got, ref, bound):
    """max |got - ref| / bound (> 1: outside the bound; NaN counts as outside)."""
    r = np.abs(np.asarray(got, np.float64) - ref) / np.maximum(bound, 1e-300)
    r = np.where(np.isnan(r), np.inf, r)
    return float(r.max())


def spread(Yb, H):
    """Spread of the eigenvalues of Yb H Yb^T (the preconditioned Hessian): max / min."""
    w = np.linalg.eigvalsh(Yb @ H @ Yb.T)
    return float(w[-1] / w[0])
