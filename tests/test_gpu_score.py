"""RegressionTest scoring and RegressionTestLoglik (-m gpu) record by record against fp64 numpy.

mlease_score: each pred must be float32 of the exact value of offset + intercept term + sum of model[c] x_c (the products exact, the
sum exact, one rounding to fp64 then to fp32).  The kernel sums in fp64 in its own order, so its value lies within
(k + 2) 2^-53 sum |terms| of the exact one; only a record whose interval straddles an fp32 rounding boundary may land one ulp
off, and the test counts those.

mlease_test_loglik: a numpy replica of the reference's rounding points -- every record's loglik as float, every combiner block's
double sum cast to float, float(sum / count) at the end; with combiner_block = 0 no cast at all.  The device sums a block in its own
order, so a block's float is pinned exactly unless its double-sum interval straddles a rounding boundary, where either neighbour
is accepted."""
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

U64 = 2.0 ** -53
REPORT = {}


@pytest.fixture(scope="module")
def mb():
    import mlease_b200
    return mlease_b200


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    for k in sorted(REPORT):
        print("%-40s %s" % (k, REPORT[k]))


def _split(a):
    """a = hi + lo, each with at most 26 significant bits: hi * x and lo * x are exact in fp64 for an fp32 x"""
    c = a * 134217729.0
    hi = c - (c - a)
    return hi, a - hi


def score_reference(rowptr, colidx, vals, model, offset, ncr, binary):
    """-> (fp64 rounding of the exact value, bound on |kernel fp64 value - exact|) per record"""
    Dg = len(model) - 1
    b = float(model[Dg])
    ic = -math.log((ncr - 1) + ncr * math.exp(-b))
    x = np.ones(len(colidx)) if binary else np.asarray(vals, np.float32).astype(np.float64)
    m = np.asarray(model, np.float64)[colidx]
    hi, lo = _split(m)
    ph, pl = hi * x, lo * x
    absp = np.abs(m * x)
    n = len(rowptr) - 1
    ref, bnd = np.zeros(n), np.zeros(n)
    for i in range(n):
        s, e = int(rowptr[i]), int(rowptr[i + 1])
        o = 0.0 if offset is None else float(offset[i])
        ref[i] = math.fsum(list(ph[s:e]) + list(pl[s:e]) + [ic, o])
        k = e - s
        bnd[i] = (k + 3) * U64 * (float(absp[s:e].sum()) + abs(ic) + abs(o)) * (1 + 1e-9) + abs(ic) * 2.0 ** -50
    return ref, bnd


def check_preds(pred, ref, bnd, tag):
    """pred == float32(ref) unless [ref - bnd, ref + bnd] straddles an fp32 rounding boundary; there pred is one of the two
    neighbours.  Counts the straddling records."""
    lo, hi = (ref - bnd).astype(np.float32), (ref + bnd).astype(np.float32)
    want = ref.astype(np.float32)
    pinned = lo == hi
    bad = np.flatnonzero(pinned & (pred.view(np.uint32) != want.view(np.uint32)) & ~((pred == 0) & (want == 0)))
    assert len(bad) == 0, (tag, bad[:8], pred[bad[:8]], want[bad[:8]])
    loose = np.flatnonzero(~pinned)
    assert np.all((pred[loose] >= lo[loose]) & (pred[loose] <= hi[loose])), tag
    w = want[loose]
    assert np.all((pred[loose] >= np.nextafter(w, np.float32(-np.inf))) & (pred[loose] <= np.nextafter(w, np.float32(np.inf)))), tag
    REPORT["score one-ulp allowance " + tag] = "%d of %d records" % (len(loose), len(pred))
    assert len(loose) <= max(2, len(pred) // 50), (tag, len(loose))
    return len(loose)


def _rows(rng, lens, Dg):
    cols = [np.sort(rng.choice(Dg, size=k, replace=False)) for k in lens]
    rp = np.cumsum([0] + list(lens)).astype(np.int64)
    return rp, np.concatenate(cols).astype(np.int32)


LENS = [0, 1, 31, 32, 33, 1100, 0, 5, 64, 65, 2, 31, 33]


def _model(rng, Dg, kind):
    if kind == "cancel":   # pairs of large terms of opposite sign: a small value with a large sum of magnitudes
        m = np.repeat(rng.uniform(20, 60, (Dg + 1) // 2), 2)[:Dg] * np.tile([1.0, -1.0], (Dg + 1) // 2)[:Dg]
        m = m * (1 + rng.normal(0, 1e-3, Dg))
    else:
        m = rng.normal(0, 1, Dg) * np.exp2(rng.integers(-8, 8, Dg))
    return np.append(m, rng.normal(0, 2))


@pytest.mark.parametrize("ncr", [1, 3])
@pytest.mark.parametrize("with_offset", [True, False])
@pytest.mark.parametrize("kind", ["plain", "cancel", "binary"])
def test_score_csr(mb, ncr, with_offset, kind):
    rng = np.random.default_rng(100 + ncr * 10 + with_offset * 3 + len(kind))
    Dg = 1500
    lens = LENS + list(rng.integers(0, 120, 2000))
    rp, ci = _rows(rng, lens, Dg)
    if kind == "cancel":   # whole pairs in every row: columns 2j and 2j + 1 with the same value, their coefficients nearly opposite
        rp = (rp // 2 * 2).astype(np.int64)
        ci = (ci[:rp[-1]] // 2 * 2).astype(np.int32)
        ci[1::2] = ci[0::2] + 1
    v = rng.normal(0, 1, len(ci)).astype(np.float32)
    if kind == "cancel":
        v[1::2] = v[0::2]
    v[:4] = [-0.0, 1e-42, 3e3, -7.0]
    model = _model(rng, Dg, kind)
    o = rng.normal(0, 4, len(rp) - 1).astype(np.float32) if with_offset else None
    binary = kind == "binary"
    pred = mb.score(v, model, rowptr=rp, colidx=ci, offset=o, num_click_replicates=ncr, binary_feature=binary)
    ref, bnd = score_reference(rp, ci, v, model, o, ncr, binary)
    check_preds(pred, ref, bnd, "csr %s ncr=%d offset=%d" % (kind, ncr, with_offset))


@pytest.mark.parametrize("on_device", [False, True])
def test_score_dense_wide_rows(mb, on_device):
    """Dense rows ldx = Dg + 3 floats apart (the padding NaN: never read), from the host and from a device tensor."""
    rng = np.random.default_rng(200 + on_device)
    n, Dg = 1300, 1100
    X = rng.normal(0, 1, (n, Dg + 3)).astype(np.float32)
    X[:, Dg:] = np.nan
    X[0, :3] = [-0.0, 1e-42, 1e3]
    model = _model(rng, Dg, "plain")
    o = rng.normal(0, 4, n).astype(np.float32)
    arg = X
    if on_device:
        import torch
        arg = torch.from_numpy(X).cuda()
    pred = mb.score(arg, model, offset=o)
    rp = np.arange(n + 1, dtype=np.int64) * Dg
    ci = np.tile(np.arange(Dg, dtype=np.int32), n)
    ref, bnd = score_reference(rp, ci, X[:, :Dg].reshape(-1), model, o, 1, False)
    check_preds(pred, ref, bnd, "dense ldx>Dg %s" % ("device" if on_device else "host"))


def test_score_refusals(mb):
    """colidx == Dg (the intercept's slot of the model) is refused, not added as a feature; so is a decreasing rowptr, in
    mlease_score, mlease_score_var and mlease_score_keyed.  Both stay inside the arrays they describe."""
    Dg = 6
    model = np.arange(Dg + 1, dtype=np.float64)
    rp = np.array([0, 2, 4], np.int64)
    ci = np.array([0, 1, 2, Dg], np.int32)
    v = np.ones(4, np.float32)
    with pytest.raises(mb.MleaseError) as e:
        mb.score(v, model, rowptr=rp, colidx=ci)
    assert e.value.code == 1 and "colidx" in e.value.message
    rpd = np.array([0, 3, 1, 4], np.int64)   # rows overlap; every entry inside [0, 4]
    ci = np.array([0, 1, 2, 3], np.int32)
    with pytest.raises(mb.MleaseError) as e:
        mb.score(v, model, rowptr=rpd, colidx=ci)
    assert e.value.code == 1 and "rowptr" in e.value.message
    with pytest.raises(mb.MleaseError) as e:
        mb.score_var(rpd, ci, v, model, var=np.ones(Dg + 1))
    assert e.value.code == 1 and "rowptr" in e.value.message
    with pytest.raises(mb.MleaseError) as e:
        mb.score_keyed(v, np.array([0, 3], np.int64), rpd, ci, Dg, np.array([0, 2], np.int64), np.array([0, Dg], np.int32),
                       np.array([0.5, 0.25], np.float32))
    assert e.value.code == 1 and "rowptr" in e.value.message


# ---- test log-likelihood -----------------------------------------------------------------------------------------------------------
def _record_ll(resp, pred, weight):
    """float32 per record (the fp64 value cast), and whether the cast is pinned against the device's few-ulp fp64 error"""
    p = pred.astype(np.float64)
    w = np.ones(len(p)) if weight is None else weight.astype(np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        v = np.where(resp == 1, -np.log1p(np.exp(-p)) * w, -np.log1p(np.exp(p)) * w)
    d = np.abs(v) * 2.0 ** -49
    with np.errstate(invalid="ignore"):
        pinned = ((v - d).astype(np.float32) == (v + d).astype(np.float32)) | ~np.isfinite(v)
    return v.astype(np.float32), pinned


def _block_floats(ll, block):
    """per block: the lowest and highest float the device's double sum of the block can be cast to (its error is within
    (m + 16) 2^-53 sum |x| for m records: a 256-stride loop, 5 shuffle levels, 8 warp partials)"""
    lo, hi = [], []
    for b0 in range(0, len(ll), block):
        x = ll[b0:b0 + block].astype(np.float64)
        s = math.fsum(x)
        bd = (len(x) + 16) * U64 * float(np.abs(x).sum())
        lo.append(float(np.float32(s - bd)))
        hi.append(float(np.float32(s + bd)))
    return np.array(lo), np.array(hi)


def loglik_replica(resp, pred, weight, combiner_block, cast_internal=False):
    """-> (lowest, highest) float the reference's rounding points allow, and the count; lowest == highest when every block is
    pinned.  None when a record's float depends on the last ulps of its fp64 value (data to avoid).  cast_internal: cast the
    internal 4096-record blocks of combiner_block = 0 as if they were combiner blocks (the replica of a wrong library)."""
    ll, pinned = _record_ll(resp, pred, weight)
    if not pinned.all():
        return None
    cnt = float(len(ll)) if weight is None else math.fsum(weight.astype(np.float64))
    if combiner_block > 0 or cast_internal:
        # the host adds the block floats in order in double (monotone in each), then one division and the cast
        lo, hi = _block_floats(ll, combiner_block if combiner_block > 0 else 4096)
        return np.float32(np.cumsum(lo)[-1] / cnt), np.float32(np.cumsum(hi)[-1] / cnt), cnt
    # no cast: the blocks' double sums added in order in double, then divided -- the exact total within both summations' bounds
    x = ll.astype(np.float64)
    tot = math.fsum(x)
    nb = -(-len(x) // 4096)
    bd = (4096 + 16 + nb + 2) * U64 * float(np.abs(x).sum())
    q_lo, q_hi = (tot - bd) / cnt, (tot + bd) / cnt
    return np.float32(q_lo - abs(q_lo) * 2 * U64), np.float32(q_hi + abs(q_hi) * 2 * U64), cnt


def _check_loglik(got, cnt, lo, hi, rcnt, tag):
    assert cnt == rcnt, (tag, cnt, rcnt)
    if lo == hi:
        assert got == lo, (tag, got, lo)
        REPORT.setdefault("loglik pinned", 0)
        REPORT["loglik pinned"] += 1
    else:
        assert lo <= got <= hi and hi <= np.nextafter(lo, np.float32(np.inf)), (tag, got, lo, hi)
        REPORT.setdefault("loglik one-ulp allowance", 0)
        REPORT["loglik one-ulp allowance"] += 1


def _ll_data(seed, n, weights):
    rng = np.random.default_rng(seed)
    resp = rng.integers(-1, 2, n).astype(np.int32)
    pred = rng.normal(0, 3, n).astype(np.float32)
    sel = rng.random(n)
    pred[sel < 0.03] = 30.0
    pred[(sel >= 0.03) & (sel < 0.06)] = -30.0
    pred[(sel >= 0.06) & (sel < 0.08)] = 100.0
    pred[(sel >= 0.08) & (sel < 0.10)] = -100.0
    big = (sel >= 0.10) & (sel < 0.12)   # +-800 where the record's value is -0: +800 with response 1, -800 otherwise
    pred[big] = np.where(resp[big] == 1, 800.0, -800.0)
    w = None
    if weights == "weights":
        w = (rng.integers(0, 33, n) / 16.0).astype(np.float32)   # sums exact in any order; zeros included
    return resp, pred, w


N_LL = 3 * 4096 + 125   # four internal blocks, the last partial; not a multiple of 7


@pytest.mark.parametrize("weights", ["weights", "absent"])
@pytest.mark.parametrize("block", [1, 7, N_LL - 1, N_LL, N_LL + 1])
def test_loglik_combiner_blocks(mb, weights, block):
    resp, pred, w = _ll_data(300 + block % 97, N_LL, weights)
    got, cnt = mb.test_loglik(resp, pred, w, combiner_block=block)
    rep = loglik_replica(resp, pred, w, block)
    assert rep is not None
    lo, hi, rcnt = rep
    _check_loglik(got, cnt, lo, hi, rcnt, "block %d %s" % (block, weights))
    # responses 0 and -1 are the same label
    r2 = resp.copy()
    r2[r2 == 0] = -1
    got2, _ = mb.test_loglik(r2, pred, w, combiner_block=block)
    assert got2.view(np.uint32) == got.view(np.uint32)


@pytest.mark.parametrize("weights", ["weights", "absent"])
def test_loglik_no_combiner(mb, weights):
    """combiner_block = 0: no float cast anywhere but the last.  The data is chosen so that casting each internal block would give
    another float, so a cast that should not be there is seen."""
    for seed in range(400, 600):
        resp, pred, w = _ll_data(seed, N_LL, weights)
        rep = loglik_replica(resp, pred, w, 0)
        if rep is None:
            continue
        lo, hi, rcnt = rep
        clo, chi, _ = loglik_replica(resp, pred, w, 0, cast_internal=True)
        if lo == hi and clo == chi and clo != lo:
            break
    else:
        pytest.fail("no data found on which a per-block cast changes the result")
    got, cnt = mb.test_loglik(resp, pred, w, combiner_block=0)
    _check_loglik(got, cnt, lo, hi, rcnt, "no combiner %s seed %d" % (weights, seed))


def test_loglik_minus_inf_and_refusal(mb):
    """-800 with response 1: the record's value is -log1p(exp(800)) = -inf in double, and so is the result; response 5 is
    refused."""
    resp = np.array([1, 0, 1, -1, 1], np.int32)
    pred = np.array([0.5, -800.0, -800.0, 800.0 - 1600.0, 800.0], np.float32)
    w = np.array([1.0, 2.0, 0.5, 1.0, 1.0], np.float32)
    for block in (0, 2):
        got, cnt = mb.test_loglik(resp, pred, w, combiner_block=block)
        assert got == -np.inf and cnt == 5.5
    bad = resp.copy()
    bad[3] = 5
    with pytest.raises(mb.MleaseError) as e:
        mb.test_loglik(bad, pred, w, combiner_block=0)
    assert e.value.code == 1 and "response" in e.value.message
