"""fp64 reference of the explicit-inverse Cholesky (ldh <= 2048): exactly representable systems for the tilings of its two code
paths, and entrywise error bounds for real Hessians.

The two paths (k3_cholesky.cu, cholesky_launch):
  narrow (ldh <= 1000)  NB = 32 panel steps: the 32 x 32 diagonal block factorised and inverted by one warp (chol_diag_block,
                        Ldinv), chol_update_kernel on 64 x 64 lower tiles; Y = L^-1 by trinv_kernel<32> (32-column groups);
                        Hinv = Y^T Y by hinv_syrk_kernel on 64 x 64 tiles
  mid (1000 < ldh)      outer panels of 256 columns (the NB = 32 chain inside, syrk_kernel's 128 x 64 tiles for the trailing update,
                        the next panel's columns first: look-ahead); 256-wide leaves by trinv_kernel<64> (64-column groups), fp64
                        DMMA merges (dgemm_kernel modes 1 and 2, 128 x 64 tiles) and Hinv = Y^T Y (mode 3)

Exactly representable systems.  L = I + E with E strictly lower triangular, dyadic entries (+-1/2, +-1/4, +-3/4) and the row
indices of its nonzeros disjoint from its column indices (so E^2 = 0).  Then Y = L^-1 = I - E and Hinv = Y^T Y = I - E - E^T + E^T E
exactly; H = L L^T = I + E + E^T + E E^T has unit pivots (rsqrt(1) = 1, every column scaling is by 1), and every product and partial
sum the kernels form is a short sum of products of these dyadic values: exact in fp64 whatever the order.  A column of E with two
entries (rows i > i') puts E[i,j] E[i',j] into H[i][i'], which the panel step or trailing update of column j's panel must cancel; a
row with two entries puts off-diagonal values into E^T E, i.e. into Hinv.

Error bounds for a real H (u = 2^-53, gamma_n = n u / (1 - n u); Lc, Ldinv, Y are the GPU's own outputs):
  Factor.  Higham's backward error of Cholesky, |H - L L^T| <= gamma_{n+1} |L| |L^T|, holds for any order of the inner sums.  The
    kernels take r = rsqrt(d) (<= 1 ulp = 2u from 1/sqrt(d)) and form L[j][j] = fl(d r) and L[i][j] = fl(a r) instead of a square
    root and a division: each of those entries carries at most 4u more relative error, so the constant is gamma_{n+5}.  The fp64
    product L L^T of the check adds gamma_n |L| |L^T|.
  Inverse.  Y = L^-1 by blocked substitution: the row block kb is Ldinv[kb] (I - sum_{jb<kb} L[kb][jb] Y[jb]), where the
    32 x 32 inverse Ldinv of the diagonal block Ld comes from its own substitution, |Ld Ldinv - I| <= gamma_36 |Ld| |Ldinv| (the
    pivots' r again).  Writing R for the bracket, L[kb] Y - I = (R_hat - R) + (Ld Ldinv - I) R_hat + Ld (Y[kb] - Ldinv R_hat), so
      |L Y - I| <= gamma_n (I + |L| |Y|) + 2 gamma_36 |Ld| |Ldinv| |R_hat|,   |R_hat| <= |Ld| |Y|  (+ lower order),
    with Ld / Ldinv the block-diagonal matrices of the blocks.  The mid path's merges form Y21 = -Y22 (L21 Y11); their two
    products add gamma_n |L22| |Y22| |L21| |Y11| <= gamma_n (|L| |Y|)^2 to the residual of the merged block, and the inexact Y22
    they multiply adds |I - L22 Y22| |L21 Y11| -- both covered by a gamma_n (|L| |Y|) (|L| |Y|) term.  The fp64 check product adds
    gamma_n |L| |Y|.
  Hinv.  Every entry is one dot product of two columns of the GPU's Y: |Hinv - Y^T Y| <= gamma_n |Y|^T |Y|, plus gamma_n for the
    check's own product.
"""
import numpy as np
import scipy.sparse as sp

from factored_reference import VALUES, ldh_of, merges

NB = 32          # panel width / diagonal block
TB = 64          # chol_update_kernel / hinv_syrk_kernel tile, trinv_kernel<64> column group
WNB = 256        # outer panel of the mid path
CHOL_WIDE_MIN = 1000
DM, DN = 128, 64  # DMMA tiles (syrk_kernel, dgemm_kernel)
U = 2.0 ** -53
SENTINEL = np.uint64(0xFFFFFFFFFFFFFFFF)


def is_mid(ldh):
    return ldh > CHOL_WIDE_MIN


def chol_pairs(Dt):
    """Nonzeros {(i, j): value} of E (i > j, rows and columns disjoint) for the tilings of the explicit-inverse Cholesky; see
    coverage() for what they reach."""
    ldh = ldh_of(Dt)
    R, C, pairs = set(), set(), {}

    def add(ti, tj, ilo=0, ihi=None, jlo=0, jhi=None, need=None):
        ihi = Dt if ihi is None else min(ihi, Dt)
        jhi = Dt if jhi is None else min(jhi, Dt)
        for d in range(256):   # nearest free position to the target (L1 distance d), inside the block
            for i, j in ((ti + di, tj + s * (d - abs(di))) for di in range(-d, d + 1) for s in (1, -1)):
                if ilo <= i < ihi and jlo <= j < jhi and 0 <= j < i and i not in C and j not in R and (i, j) not in pairs \
                        and (need is None or need(i, j)):
                    R.add(i); C.add(j); pairs[(i, j)] = VALUES[len(pairs) % len(VALUES)]
                    return (i, j)
        return None

    add(Dt - 1, 0)
    # every 32 x 32 diagonal block (chol_diag_block, Ldinv, the 32-column groups of trinv_kernel<32>)
    for k0 in range(0, Dt, NB):
        if min(k0 + NB, Dt) - k0 >= 2:
            add(min(k0 + NB, Dt) - 1 - (k0 // NB) % 7, k0 + (k0 // NB) % 5, ilo=k0, ihi=k0 + NB, jlo=k0, jhi=k0 + NB)
    # both edges of every 64-wide tile: even tiles in rows, odd tiles in columns (a row index used by E cannot be a column index)
    for t0 in range(0, Dt, TB):
        for e in (t0, t0 + TB - 1):
            if e >= Dt:
                continue
            if (t0 // TB) % 2 == 0:
                add(e, max(0, e - TB - 3), ilo=e, ihi=e + 1, jhi=e)
            else:
                add(min(Dt - 1, e + TB + 5), e, jlo=e, jhi=e + 1, ilo=e + 1)
    # columns with two entries in different 64-row tiles below their panel: H[i][i'] = E[i,j] E[i',j] is cancelled by the
    # trailing update (narrow: chol_update_kernel; mid: the look-ahead columns of the next outer panel and the rest)
    step = WNB if is_mid(ldh) else 4 * TB
    for c in range(0, Dt, step):
        j = add(c + 7, c + 5, jlo=c, jhi=c + step, ilo=c + step, ihi=c + 2 * step)   # i in the next panel
        if j is None:
            continue
        jj = j[1]
        # a second entry of column jj, two panels down if there is room (the rest of the trailing update), else in the next
        for lo, nd in ((c + 2 * step, None), (c + step, lambda i, _: i // TB != j[0] // TB), (c + step, None)):
            if add(lo + 70, jj, jlo=jj, jhi=jj + 1, ilo=lo, ihi=lo + step, need=nd):
                break
    # rows with two entries in different 64-column tiles: E^T E off the diagonal of Hinv
    for r in range(TB + 10, Dt, 3 * TB + 17):
        p = add(r, r - TB - 9, ilo=r, ihi=r + TB)
        if p is not None:
            add(p[0], p[1] - TB - 1, ilo=p[0], ihi=p[0] + 1, jhi=p[1] - (p[1] % TB))
    # every merge of the mid path's inverse (the L21 block of each: its corners)
    if is_mid(ldh):
        for m, r0, m2 in merges(ldh):
            a, e = r0 + m, min(r0 + m + m2, Dt) - 1
            blk = dict(ilo=a, ihi=e + 1, jlo=r0, jhi=r0 + m)
            add(a, r0 + m - 1, **blk)
            add(e, r0, **blk)
    return pairs


def coverage(Dt, pairs):
    """What the pairs reach: {name: bool}.  Every value must be True."""
    ldh = ldh_of(Dt)
    ij = np.array(list(pairs.keys()))
    i, j = ij[:, 0], ij[:, 1]
    cov = {"row Dt-1": bool((i == Dt - 1).any()), "column 0": bool((j == 0).any())}
    for k0 in range(0, Dt, NB):
        if min(k0 + NB, Dt) - k0 >= 2:
            cov["diagonal block %d" % k0] = bool(((i // NB == k0 // NB) & (j // NB == k0 // NB)).any())
        cov["32-column group %d" % k0] = bool((j // NB == k0 // NB).any()) or k0 + 1 >= Dt
    for t0 in range(0, Dt, TB):
        cov["64-column group %d" % t0] = bool((j // TB == t0 // TB).any()) or t0 + 1 >= Dt
        first = ((i == t0) | (j == t0)).any()
        last = t0 + TB - 1 >= Dt or ((i == t0 + TB - 1) | (j == t0 + TB - 1)).any()
        cov["64-tile %d both edges" % t0] = bool(first and last)
    wide = Dt > 2 * TB   # room for pairs across tiles
    for name, sel in (("64-tile first row", i % TB == 0), ("64-tile last row", i % TB == TB - 1),
                      ("64-tile first column", j % TB == 0), ("64-tile last column", j % TB == TB - 1)):
        cov[name] = bool(sel.any()) or not wide
    # columns with two entries: (i, i') in different 64-row tiles below the column's panel
    cols = {}
    for (a, b) in pairs:
        cols.setdefault(b, []).append(a)
    twice = [(b, sorted(r)) for b, r in cols.items() if len(r) >= 2 and len({x // TB for x in r}) >= 2]
    cov["column with two entries in different 64-row tiles"] = bool(twice) or not wide
    rows = {}
    for (a, b) in pairs:
        rows.setdefault(a, []).append(b)
    cov["row with two entries in different 64-column tiles"] = any(len({x // TB for x in c}) >= 2 for c in rows.values()) or not wide
    if is_mid(ldh):
        for c in range(0, ldh, WNB):
            cov["outer panel %d" % c] = bool(((j >= c) & (j < c + WNB)).any()) or c + 1 >= Dt
            if c + WNB < Dt:
                # look-ahead: column j in panel c, a product landing in panel c + 1's columns
                cov["look-ahead columns of panel %d" % (c + WNB)] = any(
                    c <= b < c + WNB and len(r) >= 2 and any(c + WNB <= x < c + 2 * WNB for x in r) for b, r in cols.items())
        for m, r0, m2 in merges(ldh):
            cov["merge m=%d r0=%d m2=%d" % (m, r0, m2)] = bool(((i >= r0 + m) & (i < r0 + m + m2) & (j >= r0) & (j < r0 + m)).any())
        for ti in range(0, Dt, DM):
            cov["128-row DMMA tile %d" % ti] = bool(((i >= ti) & (i < ti + DM)).any())
        for tj in range(0, Dt - 1, DN):   # (the last column, Dt - 1, is a row of E: no pair can start there)
            cov["64-column DMMA tile %d" % tj] = bool(((j >= tj) & (j < tj + DN)).any())
    return cov


def assert_coverage(Dt, pairs):
    missing = [k for k, v in coverage(Dt, pairs).items() if not v]
    assert not missing, missing


def exact_system(Dt, pairs):
    """(E dense, H) with H = (I + E)(I + E)^T (fp64, exact)."""
    ij = np.array(list(pairs.keys()))
    E = sp.csr_matrix((np.array(list(pairs.values())), (ij[:, 0], ij[:, 1])), shape=(Dt, Dt))
    H = (sp.identity(Dt, format="csr") + E + E.T + E @ E.T).toarray()
    return E.toarray(), H


def exact_outputs(E):
    """The buffers the kernels must leave for H = (I + E)(I + E)^T: Lc (Dt x Dt, zero above the diagonal), Yinv and Hinv (ldh x ldh,
    identity padding, Yinv zero above the diagonal), Ldinv (ldh x 32: the inverse of every 32 x 32 diagonal block of L)."""
    Dt = E.shape[0]
    ldh = ldh_of(Dt)
    Ep = np.zeros((ldh, ldh))
    Ep[:Dt, :Dt] = E
    Lc = np.eye(Dt) + E
    Y = np.eye(ldh) - Ep
    Hinv = np.eye(ldh) - Ep - Ep.T + Ep.T @ Ep
    Ldinv = np.stack([Y[r, (r // NB) * NB:(r // NB) * NB + NB] for r in range(ldh)])
    return dict(L=Lc, Y=Y, Hinv=Hinv, Ldinv=Ldinv)


def bits(a):
    """Raw bits with -0.0 read as +0.0 (a kernel that stores -acc or -0 * x may leave either sign of zero)."""
    a = np.asarray(a, np.float64)
    return np.where(a == 0.0, 0.0, a).view(np.uint64)


def same_bits(a, b):
    return np.array_equal(bits(a), bits(b))


def is_sentinel(a):
    return bool((np.asarray(a, np.float64).view(np.uint64) == SENTINEL).all())


def gamma(n):
    return n * U / (1.0 - n * U)


def _blockdiag(M, ldh):
    out = np.zeros((ldh, ldh))
    for k0 in range(0, ldh, NB):
        out[k0:k0 + NB, k0:k0 + NB] = M[k0:k0 + NB]
    return out


def factor_excess(H, L):
    """max |H - L L^T| / bound over the lower triangle (L: the GPU's Dt x Dt factor, lower triangle read)."""
    n = H.shape[0]
    L = np.tril(L)
    aL = np.abs(L)
    bound = (gamma(n + 5) + gamma(n)) * (aL @ aL.T)
    return _excess(np.tril(H - L @ L.T), np.tril(bound))


def inverse_excess(L, Y, Ldinv):
    """max |L Y - I| / bound (L: Dt x Dt factor; Y: ldh x ldh; Ldinv: ldh x 32), over the first Dt rows / columns."""
    Dt = L.shape[0]
    ldh = Y.shape[0]
    Lp = np.eye(ldh)
    Lp[:Dt, :Dt] = np.tril(L)
    Yl = np.tril(Y)
    aL, aY = np.abs(Lp), np.abs(Yl)
    LY = aL @ aY
    Ld = np.abs(_blockdiag(np.stack([Lp[r, (r // NB) * NB:(r // NB) * NB + NB] for r in range(ldh)]), ldh))
    Ldi = np.abs(_blockdiag(Ldinv, ldh))
    n = ldh
    bound = (gamma(n + 36) + gamma(n)) * (np.eye(ldh) + LY) + 2 * gamma(36) * (Ld @ (Ldi @ (Ld @ aY)))
    if is_mid(ldh):
        bound += gamma(n) * (LY @ LY)
    return _excess((Lp @ Yl - np.eye(ldh))[:Dt, :Dt], bound[:Dt, :Dt])


def hinv_excess(Y, Hinv):
    """max |Hinv - Y^T Y| / bound (ldh x ldh, the GPU's own lower-triangular Y)."""
    n = Y.shape[0]
    Yl = np.tril(Y)
    aY = np.abs(Yl)
    return _excess(Hinv - Yl.T @ Yl, 2 * gamma(n) * (aY.T @ aY))


def _excess(diff, bound):
    r = np.abs(diff) / np.maximum(bound, 1e-300)
    r = np.where(np.isnan(r), np.inf, r)
    return float(r.max())


# ---- quasi-Newton direction on the explicit inverse (k1_reduce_decide_kernel's first loop, newton_gemv_kernel, newton_solve_kernel)
# Ring order: pair j (0 = newest) sits in slot (count - 1 - j) % BFGS_M, npairs = min(count, BFGS_M).
#   first loop (newest..oldest):  a_j = rho_j (s_j . q);  q -= a_j y_j                              (q starts at g)
#   GEMV:                         r = Hinv q  (the Dt x Dt part of the GPU's own Hinv)
#   scale:                        r *= h0_scale   (between the GEMV and the second loop; skipped when h0_scale == 1)
#   second loop (oldest..newest): c_j = a_j - rho_j (y_j . r);  r += c_j s_j;        dir = -r
# Running error bound (every sum is an fp64 sum of Dt products in some order, |fl(sum) - sum| <= gamma_Dt sum |terms|; every
# product and update one or two roundings of u): the same recursion on absolute values carries e_q, e_a, e_r, e_c:
#   e_d = gamma_Dt |s|.|q| + |s|.e_q,   e_a = |rho| e_d + u |a|,   e_q += e_a |y| + 2u (|q| + |a y|)
#   e_r = |Hinv| e_q + gamma_Dt |Hinv| |q|,   then e_r = h0 e_r + u |r|
#   e_c = e_a + |rho| (|y|.e_r + gamma_Dt |y|.|r|) + 2u (|a| + |rho y.r|),   e_r += e_c |s| + 2u (|r| + |c s|)
# The magnitudes are the reference's (longdouble), which differ from the GPU's by far less than the bound's slack of 1 %.
BFGS_M = 6


def two_loop(Hinv, g, S, Y, rho, count, h0, dtype=np.longdouble, fault=None):
    """(dir, entrywise bound on |dir_gpu - dir|) of the direction above, computed in `dtype`.  fault (emulations the tests must
    reject): "slot" reads the ring one slot off, "reverse" runs the pairs in reverse order in both loops, "h0_first" applies h0 to
    the gradient before the first loop instead of between the GEMV and the second loop."""
    Dt = len(g)
    H = np.asarray(Hinv[:Dt, :Dt], dtype)
    aH = np.abs(H)
    gn = gamma(Dt)
    npairs = min(int(count), BFGS_M)
    slots = [((count - j) if fault == "slot" else (count - 1 - j)) % BFGS_M for j in range(npairs)]
    if fault == "reverse":
        slots = slots[::-1]
    q = np.asarray(g, dtype).copy()
    if fault == "h0_first":
        q = q * dtype(h0)
    eq = np.zeros(Dt, dtype)
    a, ea = {}, {}
    for sl in slots:
        s, y, rh = np.asarray(S[sl], dtype), np.asarray(Y[sl], dtype), dtype(rho[sl])
        d = s @ q
        ed = gn * (np.abs(s) @ np.abs(q)) + np.abs(s) @ eq
        a[sl] = rh * d
        ea[sl] = abs(rh) * ed + U * abs(a[sl])
        q = q - a[sl] * y
        eq = eq + ea[sl] * np.abs(y) + 2 * U * (np.abs(q) + np.abs(a[sl] * y))
    r = H @ q
    er = aH @ eq + gn * (aH @ np.abs(q))
    if fault != "h0_first":
        r = r * dtype(h0)
        er = dtype(h0) * er + U * np.abs(r)
    for sl in slots[::-1]:
        s, y, rh = np.asarray(S[sl], dtype), np.asarray(Y[sl], dtype), dtype(rho[sl])
        d = y @ r
        c = a[sl] - rh * d
        ec = ea[sl] + abs(rh) * (np.abs(y) @ er + gn * (np.abs(y) @ np.abs(r))) + 2 * U * (abs(a[sl]) + abs(rh * d))
        r = r + c * s
        er = er + ec * np.abs(s) + 2 * U * (np.abs(r) + np.abs(c * s))
    return (-r).astype(np.float64), (er * 1.01).astype(np.float64) + 1e-300


def direction_excess(dir_gpu, phi0, dirnorm, g, ref, bound):
    """max error / bound of dir, of phi0 = dir . g (fp64 sum of Dt products of the GPU's dir) and of dirnorm = max |dir|."""
    ed = _excess(dir_gpu - ref, bound)
    ag = np.abs(g)
    ep = _excess(np.array([phi0 - ref @ g]), np.array([ag @ bound + gamma(len(g)) * (np.abs(dir_gpu) @ ag)]))
    en = _excess(np.array([dirnorm - np.abs(ref).max()]), np.array([bound.max()]))
    return ed, ep, en
