"""CPU self-tests of tests/k1_reference.py: the fp64 reference of the K1 gradient pass against the oracle, every kernel's fp32 order
of operations (emulated in numpy) inside its per-column bound, and seeded defects outside it (the bound is not too loose)."""
import numpy as np
import pytest

import k1_reference as kr
from oracle import oracle as orc

BIG = 1e30   # prior variance: the oracle's prior term vanishes


def _orc_data(case, part):
    if "X" in case:
        return orc.Csr.from_dense(case["X"], case["response"], case["weight"], case["offset"])
    return orc.Csr(part.rowptr, part.colidx, part.vals, case["response"], case["weight"], case["offset"], part.Dg)


def _tol(part, ref):
    """Per-column tolerance: 1e-12 of the column's magnitude sum_i |x_ic r_i| (bias: sum |r_i|), plus what the oracle's q = 1 - p in
    fp64 can lose per row (2^-52 w_i |x_ic|), which matters only on columns listed by rows with tiny q."""
    x = np.abs(part.vals.astype(np.float64))
    w = part.w.astype(np.float64)
    s = 1e-12 * np.bincount(part.colidx, x * np.abs(ref.r[part.rows]), part.Dt) + 2.0 ** -52 * np.bincount(part.colidx, x * w[part.rows], part.Dt)
    s[-1] = 1e-12 * np.abs(ref.r).sum() + 2.0 ** -52 * w.sum()
    return s


@pytest.mark.parametrize("dense,edge,dup", [(True, False, False), (False, False, False), (True, True, False), (False, True, False),
                                            (False, True, True)])
def test_reference_matches_oracle_synthetic(dense, edge, dup):
    case, part = kr.synth(11, 700, 40, dense=dense, edge=edge, dup=dup)
    for beta in kr.make_betas(40, 2, 3, edge_seed=11 if edge else None):
        ref = kr.reference(part, beta)
        data = _orc_data(case, part)
        f, g = orc.objective("grad", data, beta, np.zeros(part.Dt), np.full(part.Dt, BIG))
        assert abs(f - ref.f) <= 1e-12 * ref.loss_rows.sum()
        assert abs(orc.objective("fun", data, beta, np.zeros(part.Dt), np.full(part.Dt, BIG)) - ref.f) <= 1e-12 * ref.loss_rows.sum()
        present = np.zeros(part.Dt, bool); present[part.colidx] = True; present[-1] = True
        assert np.all(np.abs(g - ref.g)[present] <= _tol(part, ref)[present])
        assert np.all(ref.g[~present] == 0.0)   # columns no row lists are exactly 0


def test_reference_matches_oracle_on_fixture(fixture_data):
    d = fixture_data
    part = kr.Part.from_csr(d.rowptr, d.colidx, d.val, d.response, d.weight, d.offset, d.n_features)
    rng = np.random.default_rng(0)
    beta = rng.normal(0, 0.1, part.Dt).astype(np.float32).astype(np.float64)
    ref = kr.reference(part, beta)
    f, g = orc.objective("grad", d, beta, np.zeros(part.Dt), np.full(part.Dt, BIG))
    assert abs(f - ref.f) <= 1e-12 * ref.loss_rows.sum()
    present = np.zeros(part.Dt, bool); present[part.colidx] = True; present[-1] = True
    assert np.all(np.abs(g - ref.g)[present] <= _tol(part, ref)[present])


def test_labels_and_binary_features():
    assert list(kr.labels([1, 0, -1])) == [1, -1, -1]
    case, part = kr.synth(2, 50, 12, binary=True)
    assert np.all(part.vals == 1.0)


PLANS = [kr.Plan("dense", RT=8, chunks=3), kr.Plan("dense", RT=4, chunks=5), kr.Plan("fused", seg_rows=97, chunks=0),
         kr.Plan("fused", seg_rows=1000, chunks=0), kr.Plan("fx", chunks=7), kr.Plan("fx", chunks=1), kr.Plan("csr", chunks=5)]


def _cases(plan, standard):
    dense = plan.kind == "dense"
    if standard:
        return [kr.synth(21, 900, 37, dense=dense)]
    return [kr.synth(22, 900, 37, dense=dense, edge=True, empty_rows=not dense),
            kr.synth(23, 333, 200, dense=dense, nnz=30),
            kr.synth(24, 500, 61, dense=dense, edge=True, dup=plan.kind == "csr")]


def _fix(plan, part):
    if plan.kind == "fused":
        return kr.Plan("fused", seg_rows=plan.seg_rows, chunks=-(-part.n // plan.seg_rows))
    return plan


@pytest.mark.parametrize("plan", PLANS, ids=lambda p: "%s-%d-%d-%d" % (p.kind, p.RT, p.seg_rows, p.chunks))
@pytest.mark.parametrize("standard", [True, False])
def test_emulation_within_bound(plan, standard):
    for i, (case, part) in enumerate(_cases(plan, standard)):
        plan_p = _fix(plan, part)
        edge_seed = {0: 22, 2: 24}.get(i) if not standard else None
        for beta in kr.make_betas(part.Dg, 2, 5 + i, edge_seed=edge_seed):
            ref = kr.reference(part, beta)
            err = kr.row_errors(part, ref, plan_p)
            g, f, sd = kr.emulate(part, beta, plan_p)
            bnd, _ = kr.grad_bound(part, ref, plan_p, err)
            ratio = kr.ratio(g - ref.g, bnd)
            assert np.all(ratio <= 1.0), (i, int(np.argmax(ratio)), ratio.max())
            assert abs(f - ref.f) <= kr.loss_bound(part, ref, plan_p, err)
            assert np.all(np.abs(sd.astype(np.float64) - ref.sd) <= kr.sd_bound(ref, err))


@pytest.mark.parametrize("plan", PLANS, ids=lambda p: "%s-%d-%d-%d" % (p.kind, p.RT, p.seg_rows, p.chunks))
@pytest.mark.parametrize("defect", kr.DEFECTS + ("wrong_lambda",))
def test_seeded_defect_violates_bound(plan, defect):
    (case, part), = _cases(plan, True)
    plan_p = _fix(plan, part)
    betas = kr.make_betas(part.Dg, 2, 7)
    ref = kr.reference(part, betas[0])
    bnd, _ = kr.grad_bound(part, ref, plan_p)
    if defect == "wrong_lambda":
        g, _, _ = kr.emulate(part, betas[1], plan_p)
    else:
        g, _, _ = kr.emulate(part, betas[0], plan_p, defect=defect)
    assert np.any(np.abs(g - ref.g) > bnd), defect


def test_fixed_point_resolution_follows_the_kernel():
    """e_hi and kbits as k1_csr_fx_kernel derives them (2^e_hi * bound in [2^28, 2^29), kbits = 30 - bit length of the rows per CTA)."""
    case, part = kr.synth(3, 1000, 20)
    for per in (1, 2, 3, 1000, 16384, 16385):
        e_hi, kbits, res = kr.fx_scales(part, per)
        bound = np.float32(per) * np.float32(part.w.max()) * np.float32(max(np.abs(part.vals).max(), 1.0))
        assert 2.0 ** 28 <= float(bound) * 2.0 ** e_hi < 2.0 ** 29
        assert kbits == min(24, 30 - per.bit_length())
        assert res == 0.5 * 2.0 ** (-kbits - e_hi)
