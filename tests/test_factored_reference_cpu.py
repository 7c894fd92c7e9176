"""CPU checks of tests/factored_reference.py: the premises of the exactly representable factors, their coverage of the recursive
inverse at every width the GPU tests use, and that the bounds of the direction emulation are tight enough to catch the defects a
kernel of this shape could have."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import factored_reference as fr  # noqa: E402

WIDTHS = [2049, 2080, 2303, 10001]   # Dt of D = 2048, 2079, 2302, 10000


@pytest.mark.parametrize("Dt", WIDTHS)
def test_exact_pairs_premises_and_coverage(Dt):
    pairs = fr.exact_pairs(Dt)
    rows = {i for i, _ in pairs}
    cols = {j for _, j in pairs}
    assert not rows & cols
    assert all(0 <= j < i < Dt for i, j in pairs)
    assert set(pairs.values()) <= {0.5, -0.5, 0.25, -0.25, 0.75, -0.75}
    cov = fr.coverage(Dt, pairs)
    assert all(cov.values()), [k for k, v in cov.items() if not v]
    if Dt == 10001:   # the benchmark width: merges up to m = 8192, whose second block is 1824 rows (of which 1809 below Dt)
        assert (8192, 0, 1824) in fr.merges(fr.ldh_of(Dt))
    if Dt <= 2303:
        E, H = fr.exact_system(Dt, pairs)
        Ed = E.toarray()
        assert not (Ed @ Ed).any()
        L = np.eye(Dt) + Ed
        assert np.array_equal(np.linalg.cholesky(H), L)   # unit pivots, exact in fp64
        Y = np.eye(Dt) - Ed
        assert np.array_equal(Y @ L, np.eye(Dt))


def test_exact_bits_catch_flips_transposes_and_merge_tiles():
    """The bitwise check of Yinv / Ysym on exact data fails for one flipped element, a transposed tile, and a merge tile that is
    skipped or applied twice."""
    Dt = 2303
    ldh = fr.ldh_of(Dt)
    pairs = fr.exact_pairs(Dt)
    E, _ = fr.exact_system(Dt, pairs)
    Y = np.eye(ldh)
    Y[:Dt, :Dt] -= E.toarray()
    ref = fr.ysym_bits(Y[:Dt, :Dt], ldh)
    assert np.array_equal(fr.bits_to_float(ref)[:Dt, :Dt], np.tril(Y[:Dt, :Dt]) + np.tril(Y[:Dt, :Dt], -1).T)
    (i, j), v = next(iter(pairs.items()))
    bad = Y.copy(); bad[i, j] = -bad[i, j]
    assert not np.array_equal(bad, Y) and not np.array_equal(fr.ysym_bits(bad[:Dt, :Dt], ldh), ref)
    for m, r0, m2 in fr.merges(ldh):
        inside = [(a, b) for a, b in pairs if r0 + m <= a < r0 + m + m2 and r0 <= b < r0 + m]
        a, b = inside[0]
        ti, tj = (a - r0 - m) // fr.TILE * fr.TILE + r0 + m, (b - r0) // fr.TILE * fr.TILE + r0
        tile = (slice(ti, ti + fr.TILE), slice(tj, tj + fr.TILE))
        for corrupt in ("skip", "twice", "transpose"):
            bad = Y.copy()
            if corrupt == "skip":
                bad[tile] = 0.0
            elif corrupt == "twice":
                bad[tile] *= 2.0
            else:
                blk = bad[tile].copy()
                bad[tile] = blk.T[:blk.shape[0], :blk.shape[1]] if blk.shape[0] == blk.shape[1] else 0.0
            assert not np.array_equal(bad, Y), (m, r0, corrupt)
            assert not np.array_equal(fr.ysym_bits(bad[:Dt, :Dt], ldh), ref), (m, r0, corrupt)


def _generic(Dt, seed):
    """A wide-ish SPD Hessian (Gram of random sparse rows + prior), its bf16 factored inverse, and two vectors."""
    rng = np.random.default_rng(seed)
    A = rng.normal(size=(3 * Dt, Dt)) * (rng.random((3 * Dt, Dt)) < 0.02)
    H = A.T @ A * 0.25 + np.eye(Dt)
    Y = np.linalg.inv(np.linalg.cholesky(H))
    bits = fr.ysym_bits(Y, fr.ldh_of(Dt))
    q = rng.normal(size=(2, Dt)).astype(np.float32)
    return H, Y, bits, q


@pytest.mark.parametrize("Dt", [611, 2303])
def test_direction_bounds_catch_corruptions(Dt):
    """Each defect below must push at least one entry past the entrywise bound of the emulation on this data (the GPU test asserts
    every entry inside it), while the fp32 arithmetic the kernel actually performs stays inside."""
    H, Y, bits, q = _generic(Dt, Dt)
    lo, up = fr.halves(bits, Dt)
    t_ex, b0 = fr.phase0(lo, q)
    t = t_ex.astype(np.float32)
    d_ex, b1 = fr.phase1(up, t)
    # the kernel's own arithmetic: per-lane fp32 FMA chains in chunk order, fp64 across lanes -- inside the bound
    qf = q[0].astype(np.float32)
    for r in (0, 5, Dt // 2, Dt - 1):
        r0 = r // 4 * 4
        lanes = np.zeros(32, np.float32)
        for k in range(0, min(r0 + 4, Dt), 8):
            ln = (k // 8) % 32
            for e in range(8):
                if k + e <= r:
                    lanes[ln] = np.float32(lanes[ln] + np.float32(lo[r, k + e]) * qf[k + e])
        assert abs(np.float32(lanes.astype(np.float64).sum()) - t_ex[0, r]) <= b0[0, r]
    assert fr.excess(t, t_ex, b0) <= 1.0 and fr.excess(d_ex, d_ex, b1) == 0.0
    # a mirror block one row off (upper block (c-block 3, k-block 20) read one row of Y further down)
    upb = up.copy()
    cs, ks = slice(96, 128), slice(640 % Dt, 672 % Dt) if Dt > 672 else slice(480, 512)
    upb[cs, ks] = fr.bits_to_float(bits)[ks.start + 1:ks.stop + 1, cs].T
    assert fr.excess(fr.phase1(upb, t)[0], d_ex, b1) > 1.0
    # the diagonal dropped in either phase
    assert fr.excess(fr.phase0(np.tril(lo, -1), q)[0].astype(np.float32), t_ex, b0) > 1.0
    assert fr.excess(fr.phase1(np.triu(up, 1), t)[0], d_ex, b1) > 1.0
    # the last partial 8-element chunk dropped (Dt % 8 != 0)
    k8 = Dt & ~7
    assert k8 < Dt
    lob, upb = lo.copy(), up.copy()
    lob[:, k8:] = 0.0; upb[:, k8:] = 0.0
    assert fr.excess(fr.phase0(lob, q)[0].astype(np.float32), t_ex, b0) > 1.0
    assert fr.excess(fr.phase1(upb, t)[0], d_ex, b1) > 1.0
    # a member given another member's vector, in either phase
    assert fr.excess(fr.phase0(lo, q[::-1])[0].astype(np.float32), t_ex, b0) > 1.0
    assert fr.excess(fr.phase1(up, t[::-1])[0], d_ex, b1) > 1.0
    # a stale t (phase 1 fed with the t of the previous vector)
    assert fr.excess(fr.phase1(up, t[[1, 1]])[0][0], d_ex[0], b1[0]) > 1.0
    # the preconditioner the bf16 factor gives: close to the identity on a well-conditioned H
    Yb = fr.bits_to_float(bits)[:Dt, :Dt]
    Yb = np.tril(Yb)
    assert fr.spread(Yb, H) < 1.1


def test_merge_bound_accepts_tf32_rounding_and_catches_tile_defects():
    """The per-merge TF32 bound: the fp64 inverse with each merge's operands rounded to TF32 stays inside; a merge tile that is
    skipped, applied twice or written transposed does not."""
    Dt = 600
    ldh = fr.ldh_of(Dt)
    H, Y, _, _ = _generic(Dt, 3)
    Lc = np.eye(ldh)
    Lc[:Dt, :Dt] = np.linalg.cholesky(H)
    Yp = np.eye(ldh)
    Yp[:Dt, :Dt] = Y
    assert fr.merge_excess(Lc, Yp) < 1e-3

    def tf32(a):   # double -> float -> tf32 (round to nearest, ties away: cvt.rna)
        u = np.asarray(a, np.float32).view(np.uint32).astype(np.uint64)
        return ((u + 0x1000) & 0xFFFFE000).astype(np.uint32).view(np.float32).astype(np.float64)

    Yt = Yp.copy()
    for m, r0, m2 in fr.merges(ldh):
        a, e = r0 + m, r0 + m + m2
        T = (tf32(Lc[a:e, r0:a]) @ tf32(Yt[r0:a, r0:a])).astype(np.float32).astype(np.float64)
        Yt[a:e, r0:a] = -(tf32(Yt[a:e, a:e]) @ tf32(T)).astype(np.float32)
    assert 1e-3 < fr.merge_excess(Lc, Yt) <= 1.0
    m, r0, m2 = fr.merges(ldh)[0]   # (m = 256: whole 128 x 128 tiles)
    tile = (slice(r0 + m, r0 + m + fr.TILE), slice(r0, r0 + fr.TILE))
    for corrupt in ("skip", "twice", "transpose"):
        bad = Yt.copy()
        bad[tile] = 0.0 if corrupt == "skip" else (2.0 * bad[tile] if corrupt == "twice" else bad[tile].T)
        assert fr.merge_excess(Lc, bad) > 1.0, corrupt
