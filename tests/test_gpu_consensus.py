"""GPU tests (-m gpu) of the ADMM consensus step (K4, csrc/k4_consensus.cu) and the host values it reads (session.cu), bit for bit
(up to the sign of a zero and the payload of a NaN) against the numpy replica consensus_reference.py, through the test hook
mlease_internal_consensus (not part of the C ABI):

- each stage (reset, init, pack, consensus) on injected states over widths Dt = 8, 256 (one CTA), 257 (the intercept alone in
  CTA 1), 1001 (padding) and 10001 (40 CTAs), 1 / 3 / 5 lambdas, all partitions local or a subset (local sum, global P), dense,
  CSR, fused multi-lambda CSR and matrix-free batches, L2 with and without lambda.map and penalize_intercept, L1 with values on the
  band edge; padding, the exchange's failed-fit slot, the diff sentinel and the Ctrl fields K4 does not own are checked by bytes;
- real iterations: local_step, the state read back, the public consensus (once with a perturbed exchange sum, as another rank's
  share would make it), the state read back again, all against the replica applied to the first read-back;
- the estimated start gradient g_t of the fused batches against the exact data-term gradient at x_p;
- the hook's refusals."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import consensus_reference as cr  # noqa: E402

pytestmark = pytest.mark.gpu
f32 = np.float32
PAD64, PAD32 = -12345.678, f32(-1234.5)   # padding sentinels (no kernel may write [Dt, ldx) outside reset)
EXCH_LAST, DIFF_SENT = 123.25, -7.0        # the failed-fit slot; a diff the launcher must zero (a negative double's bits would win the atomicMax)
RATIOS = []                                 # measured error ratios of the estimated start gradient (printed at the end of the module)


@pytest.fixture(scope="module")
def mb():
    import mlease_b200
    yield mlease_b200
    if RATIOS:
        print("\nestimated start gradient: max error / (|H|inf xtol max(|x|inf, 1e-2)) = %.3g (of %d x-updates); reordered formula >= %.3g"
              % (max(r[0] for r in RATIOS), len(RATIOS), min(r[1] for r in RATIOS)))


def _same(a, b):
    """Bit for bit, up to the sign of a zero and the payload of a NaN."""
    a = np.ascontiguousarray(a)
    b = np.ascontiguousarray(b, a.dtype)
    u = {8: np.uint64, 4: np.uint32}[a.dtype.itemsize]
    return bool(((a.view(u) == b.view(u)) | ((a == 0) & (b == 0)) | (np.isnan(a) & np.isnan(b))).all())


def _first_bad(a, b):
    a, b = np.asarray(a), np.asarray(b, np.asarray(a).dtype)
    return np.argwhere(~((a == b) | (np.isnan(a) & np.isnan(b))))[:4].tolist()


def _rows(r, kind, n, D, nnz=3):
    """(arrays for add_partition_*, k1_reference.Part): dense rows, CSR rows with sorted unique columns (fused / matrix-free), or
    CSR rows that repeat a column (general CSR: no fused K1)."""
    import k1_reference as k1
    y = (r.random(n) < 0.5).astype(np.int32)
    if kind == "dense":
        X = r.normal(size=(n, D)).astype(np.float32)
        return dict(X=X, response=y), k1.Part.from_dense(X, y, np.ones(n), np.zeros(n))
    k = min(nnz, D)
    ci = np.stack([np.sort(r.choice(D, k, replace=False)) for _ in range(n)]).astype(np.int32)
    if kind == "csr":
        ci[:, -1] = ci[:, 0]   # a repeated column in every row
    v = (r.normal(size=(n, k)) / np.sqrt(k)).astype(np.float32)
    rp = np.arange(n + 1, dtype=np.int64) * k
    arr = dict(rowptr=rp, colidx=ci.reshape(-1), vals=v.reshape(-1), response=y)
    return arr, k1.Part.from_csr(rp, ci.reshape(-1), v.reshape(-1), y, np.ones(n), np.zeros(n), D)


class _Sess:
    """An ADMM session of P partitions (those in `parts` resident) x L lambdas; kind: "dense", "csr" (general CSR, Gram path),
    "fused" (sorted unique CSR rows, fused multi-lambda K1 when L <= 4) or "mf" (matrix-free, hessian_policy 2)."""

    def __init__(self, mb, kind, D, P, L, parts=None, n=400, reg=2, lmap=None, pen=False, coef=0.0, epsilon=1e-4, seed=0):
        from mlease_b200.admm import _internal_consensus
        self.hook = _internal_consensus
        r = np.random.default_rng(seed + D + 7 * P + 31 * L)
        self.kind, self.D, self.P, self.L, self.reg, self.pen, self.coef, self.eps = kind, D, P, L, reg, pen, coef, epsilon
        self.parts = list(range(P)) if parts is None else sorted(parts)
        self.lambdas = [0.5 + 1.5 * l for l in range(L)]
        self.rhos = [1.0, 0.7, 2.5, 0.3, 1.9][:L]
        self.lmap = lmap
        self.s = mb.AdmmSession(P, D, self.lambdas, self.rhos, regularizer=reg, penalize_intercept=pen, lambda_map=lmap,
                                rho_adapt_coefficient=coef, epsilon=epsilon, hessian_policy=2 if kind == "mf" else 0)
        self.s.__enter__()
        self.data = {}
        for p in self.parts:
            arr, part = _rows(r, "csr" if kind == "csr" else ("dense" if kind == "dense" else "fused"), n, D)
            if kind == "dense":
                self.s.add_partition_dense(p, arr["X"], arr["response"])
            else:
                self.s.add_partition_csr(p, arr["rowptr"], arr["colidx"], arr["vals"], arr["response"])
            self.data[p] = part
        self.s.begin()
        self.info = self.hook(self.s, read=False)["info"]
        i = self.info
        self.nprob, self.Dt, self.ldx, self.nlocal, self.fused = i["nprob"], i["Dt"], i["ldx"], i["nlocal"], bool(i["fused"])
        assert (i["L"], i["P"], i["nlocal"], i["Dt"], i["regularizer"]) == (L, P, len(self.parts), D + 1, reg)
        assert i["nprob"] == len(self.parts) * L and i["ldx"] % 4 == 0 and i["ldx"] >= i["Dt"]
        want = dict(dense=(0, 0, 0), csr=(1, 0, 0), fused=(1, int(L <= 4), 0), mf=(1, i["fused"], 1))[kind]
        assert (i["csr"], i["fused"], i["matrix_free"]) == want, (kind, i)
        self.wz = cr.z_weights(P, self.lambdas, self.rhos, D, self.ldx, lambda_map=lmap, penalize_intercept=pen)
        self.thr = cr.l1_thresholds(P, self.lambdas, self.rhos) if reg == 1 else None

    def close(self):
        self.s.__exit__(None, None, None)

    def state(self, r):
        nprob, L, Dt, ldx = self.nprob, self.L, self.Dt, self.ldx
        vec = np.full((nprob, 5, ldx), PAD64)
        vec[:, :, :Dt] = r.normal(size=(nprob, 5, Dt))
        vec[:, cr.Q, :Dt] = r.uniform(0.5, 3.0, (nprob, Dt))
        fvec = np.full((nprob, 3, ldx), PAD32, f32)
        fvec[:, :, :Dt] = r.normal(size=(nprob, 3, Dt)).astype(f32)
        z = np.full((L, ldx), PAD64)
        z[:, :Dt] = r.normal(size=(L, Dt))
        exch = r.normal(size=L * Dt + 1) * self.P
        exch[-1] = EXCH_LAST
        ctrl = np.tile(np.array([3, 7, self.info["k1_grid"]], np.int32), (nprob, 1))
        return dict(vec=vec, fvec=fvec, z=z, exch=exch, diff=np.full(L, DIFF_SENT), ctrl=ctrl)

    def run(self, stages, st, it=1, leps=0.01):
        self.s.begin()
        return self.hook(self.s, stages, st, iter=it, liblinear_eps=leps)

    def check(self, out, exp, tag, keys=("vec", "fvec", "z", "exch", "diff")):
        for k in keys:
            assert _same(out[k], exp[k]), (tag, k, _first_bad(out[k], exp[k]))
        assert (out["ctrl"] == exp["ctrl"]).all(), (tag, "ctrl", out["ctrl"][:4].tolist(), exp["ctrl"][:4].tolist())
        assert (out["ctrl_raw"][0] == out["ctrl_raw"][1]).all(), (tag, "a Ctrl field K4 does not own changed")
        assert _same(out["wz"], self.wz), (tag, "wz")
        if self.reg == 1:
            assert _same(out["l1thr"], self.thr), (tag, "l1thr")


# (kind, D, P, local partitions or None, L, regularizer, lambda.map, penalize_intercept, rho.adapt.coefficient)
CASES = [
    ("dense", 7, 2, None, 1, 2, False, False, 0.0),
    ("dense", 255, 5, (0, 2, 3), 3, 2, True, True, 0.289),
    ("dense", 1000, 1, None, 5, 1, False, False, 0.0),
    ("csr", 256, 3, None, 5, 2, False, False, 0.1),
    ("csr", 1000, 2, None, 3, 1, False, False, 0.0),
    ("fused", 7, 3, (1,), 3, 2, False, True, 0.0),
    ("fused", 256, 4, (1, 3), 3, 1, False, False, 0.0),
    ("fused", 1000, 2, None, 1, 2, True, False, 0.0),
    ("fused", 10000, 4, (0, 3), 3, 2, False, False, 0.289),
    ("mf", 255, 5, (0, 2, 3), 5, 2, False, False, 0.0),
    ("mf", 1000, 3, (1, 2), 3, 2, False, True, 0.0),
    ("mf", 10000, 5, (0, 2, 3), 1, 1, False, False, 0.0),
]


def _lmap(D, r):
    m = (np.abs(r.normal(size=D)) * 3).astype(np.float32)
    m[::4] = 0.0
    m[1::7] = -1.5
    return m


def _ids(c):
    return "%s-D%d-P%d%s-L%d-%s%s%s%s" % (c[0], c[1], c[2], "" if c[3] is None else "loc" + "".join(map(str, c[3])), c[4], "L1" if c[5] == 1 else "L2",
                                          "-map" if c[6] else "", "-pen" if c[7] else "", "-coef" if c[8] else "")


@pytest.mark.parametrize("case", CASES, ids=_ids)
def test_stages_bitwise(mb, case):
    kind, D, P, parts, L, reg, lm, pen, coef = case
    r = np.random.default_rng(D * 13 + L)
    S = _Sess(mb, kind, D, P, L, parts, reg=reg, lmap=_lmap(D, r) if lm else None, pen=pen, coef=coef)
    try:
        Dt, nl = S.Dt, S.nlocal
        rho1 = [cr.rho_eff(x, 1) for x in S.rhos]
        # reset (as begin() runs it)
        st = S.state(r)
        out = S.run(["reset"], st)
        exp = cr.reset(st, L, Dt, rho1)
        S.check(out, exp, "reset")
        assert _same(out["rho"], rho1)
        # init on an injected z (L2 only, as begin_initialized)
        if reg == 2:
            st = S.state(r)
            S.check(S.run(["init"], st), cr.init(st, L, Dt), "init")
        # pack
        st = S.state(r)
        out = S.run(["pack"], st)
        S.check(out, cr.pack(st, L, Dt, nl), "pack")
        # consensus: the largest |dz| of each lambda in the last CTA, at a lane != 0 where the width has one; distinct rho per lambda
        for it, leps, tag in ((1, 0.01, "big diff"), (3, 1e-6, "diff 0 -> stop"), (2, 1e-6, "NaN")):
            st = S.state(r)
            if reg == 1:
                t = S.thr
                for l in range(L):   # means on the band edges and one ulp outside (exact when P is a power of two), large intercept
                    base = l * Dt
                    vals = [t[l], -t[l], np.nextafter(t[l], np.inf), -np.nextafter(t[l], np.inf), np.nextafter(t[l], 0), 0.0]
                    for j, v in enumerate(vals[:max(0, Dt - 1)]):
                        st["exch"][base + j] = v * P
                    st["exch"][base + Dt - 1] = 1e3 * P * (1 + l)
            zn = cr.consensus(st, L, Dt, P, nl, S.wz, [1.0] * L, l1thr=S.thr)["z"]
            last_cta = (Dt - 1) // 256 * 256
            kb = max(range(last_cta, Dt), key=lambda k: (k % 32 != 0, k))
            st["z"][:, :Dt] = zn[:, :Dt] * (1 + 1e-9 * r.normal(size=(L, Dt)))
            for l in range(L):
                st["z"][l, kb] = zn[l, kb] + 1.0 + 0.5 * l
            if tag.startswith("diff 0"):
                st["z"][:, :Dt] = zn[:, :Dt]
            if tag == "NaN":
                st["exch"][0 * Dt + Dt - 1] = np.nan          # lambda 0: NaN at the intercept -> its diff is NaN
                if L > 1:
                    st["exch"][1 * Dt + min(1, Dt - 2)] = np.nan   # lambda 1: a NaN coefficient is skipped
            rho_next = [cr.rho_eff(x, it + 1, coef=coef) for x in S.rhos]
            out = S.run(["consensus"], st, it=it, leps=leps)
            exp = cr.consensus(st, L, Dt, P, nl, S.wz, rho_next, l1thr=S.thr, fused=S.fused)
            S.check(out, exp, "consensus " + tag)
            assert _same(out["rho"], rho_next), (tag, out["rho"], rho_next)
            mx, mn, stop = cr.finish(exp["diff"], leps, S.eps)
            assert _same(np.float64(out["maxdiff"]), np.float64(mx)) and _same(np.float64(out["mindiff"]), np.float64(mn)), (tag, out["maxdiff"], mx, out["mindiff"], mn)
            assert out["stop"] == stop, tag
            if tag == "big diff":
                assert (exp["diff"] >= 1.0).all() and stop == 0
            if tag.startswith("diff 0"):
                assert stop == 1 and mx == 0.0
            if tag == "NaN":
                assert np.isnan(out["diff"][0]) and (L == 1 or np.isfinite(out["diff"][1]))
            if not S.fused:   # g_t, skip_eval and k1_chunks belong to the fused K1's problems only
                assert (out["vec"][:, cr.GT] == st["vec"][:, cr.GT]).all() and (out["ctrl"] == st["ctrl"]).all()
        # begin() and begin_initialized(z0, 2.5), read back without stages
        S.s.begin()
        rd = S.hook(S.s)
        z0 = np.full((L, S.ldx), 0.0)
        exp = cr.reset(dict(vec=rd["vec"], fvec=rd["fvec"], z=rd["z"], exch=rd["exch"], diff=rd["diff"], ctrl=rd["ctrl"]), L, Dt, rho1)
        S.check(rd, exp, "begin()", keys=("vec", "fvec", "z"))
        assert (rd["ctrl"][:, :2] == 0).all() and _same(rd["rho"], rho1)
        if reg == 2:
            z0[:, :Dt] = r.normal(size=(L, Dt))
            S.s.begin(z0[:, :Dt], 2.5)
            rd = S.hook(S.s)
            rho_b = [cr.rho_eff(x, 1, boost_rate=2.5) for x in S.rhos]
            exp = cr.reset(dict(vec=rd["vec"], fvec=rd["fvec"], z=rd["z"], exch=rd["exch"], diff=rd["diff"], ctrl=rd["ctrl"]), L, Dt, rho_b)
            exp["z"] = z0
            exp = cr.init(exp, L, Dt)
            S.check(rd, exp, "begin_initialized", keys=("vec", "fvec", "z"))
            assert _same(rd["rho"], rho_b)
    finally:
        S.close()


# ---------------------------------------------------------------------------------------------------------------------------------
# real iterations


def _grad_hess_inf(part, x):
    """The exact data-term gradient at float(x) (k1_reference) and |H + diag(q)|inf pieces: the row sums of |X^T D X| (fp64)."""
    import k1_reference as k1
    import scipy.sparse as sp
    ref = k1.reference(part, x)
    rows = part.rows
    Xs = sp.csr_matrix((part.vals.astype(np.float64), (rows, part.colidx)), shape=(part.n, part.Dt))
    Xs = sp.hstack([Xs[:, :part.Dg], sp.csr_matrix(np.ones((part.n, 1)))]).tocsr()
    d = part.w.astype(np.float64) * ref.p * ref.q
    H = (Xs.T @ sp.diags(d) @ Xs).tocsr()
    return ref.g, np.asarray(abs(H).sum(axis=1)).ravel()


GT_C = 0.5   # measured on an H100: at most 0.064 over the 100 x-updates of test_real_iterations (c chosen ~8x above); the
#             formula with the new q and m gave ratios >= 218

# (kind, D, P, local partitions or None, L, regularizer, rows per partition, boost, rho.adapt.coefficient)
REAL = [
    ("dense", 60, 3, None, 2, 2, 400, 0.0, 0.0),
    ("csr", 300, 3, (0, 2), 3, 1, 1500, 0.0, 0.0),
    ("fused", 300, 3, None, 3, 2, 1500, 2.5, 0.289),
    ("mf", 300, 2, None, 2, 2, 1500, 0.0, 0.3),
    ("fused", 10000, 4, None, 3, 2, 3000, 0.0, 0.0),   # the benchmark's shape, small
]


@pytest.mark.parametrize("case", REAL, ids=lambda c: "%s-D%d-P%d-L%d" % (c[0], c[1], c[2], c[4]))
def test_real_iterations(mb, case):
    import torch
    kind, D, P, parts, L, reg, n, boost, coef = case
    S = _Sess(mb, kind, D, P, L, parts, n=n, reg=reg, coef=coef, epsilon=1e-4, seed=5)
    s = S.s
    try:
        r = np.random.default_rng(3)
        if boost:
            s.begin(r.normal(size=(L, S.Dt)) * 0.1, boost)
        Dt = S.Dt
        exch = torch.zeros(L * Dt, dtype=torch.float64, device="cuda")
        for it in range(1, 5):
            s.local_step(exch)
            torch.cuda.synchronize()
            pre = S.hook(s)
            if it == 2:   # another rank's share of the sum
                exch += torch.from_numpy(r.normal(size=L * Dt) * 1e-3).cuda()
            S_sum = exch.cpu().numpy()
            leps = float(s.stats()["liblinear_epsilon"])
            md, stop = s.consensus(exch)
            post = S.hook(s)
            st = {k: pre[k] for k in ("vec", "fvec", "z", "ctrl")}
            st.update(exch=np.append(S_sum, EXCH_LAST), diff=np.zeros(L))
            rho_next = [cr.rho_eff(x, it + 1, boost_rate=boost, coef=coef) for x in S.rhos]
            exp = cr.consensus(st, L, Dt, P, S.nlocal, S.wz, rho_next, l1thr=S.thr, fused=S.fused)
            tag = "iteration %d" % it
            for k in ("vec", "fvec", "z", "diff"):
                assert _same(post[k], exp[k]), (tag, k, _first_bad(post[k], exp[k]))
            assert (post["ctrl"] == exp["ctrl"]).all(), tag
            assert _same(post["rho"], rho_next)
            mx, mn, stp = cr.finish(exp["diff"], leps, S.eps)
            assert _same(np.float64(md), np.float64(mx)) and int(stop) == stp, (tag, md, mx)
            if S.fused:
                _check_estimate(S, pre, post, tag)
            exch.zero_()
    finally:
        S.close()


def _check_estimate(S, pre, post, tag):
    """g_t after the consensus estimates the data-term gradient at x_p from the old prior: x_p minimised data(x) + q/2 |x - m|^2 up to
    the last, unevaluated Newton correction d (|d|inf <= xtol max(|x_p|inf, 1e-2)), so the error is the objective's gradient at x_p,
    ~ (H + q) d: bounded by GT_C |H + diag(q)|inf xtol max(|x_p|inf, 1e-2).  The same formula with the NEW q and m must break it."""
    L = S.L
    xtol = 2e-7
    for pi, p in enumerate(S.parts):
        for l in range(L):
            b = pi * L + l
            x = pre["vec"][b, cr.BETA, :S.Dt]
            q_old = pre["vec"][b, cr.Q, :S.Dt]
            g, hrow = _grad_hess_inf(S.data[p], x)
            scale = (hrow + q_old).max() * xtol * max(np.abs(x).max(), 1e-2)
            err = np.abs(post["vec"][b, cr.GT, :S.Dt] - g).max() / scale
            bad = -post["vec"][b, cr.Q, :S.Dt] * (x - post["vec"][b, cr.M, :S.Dt])
            err_bad = np.abs(bad - g).max() / scale
            RATIOS.append((err, err_bad))
            assert err <= GT_C, (tag, p, l, err)
            assert err_bad > 10 * GT_C, (tag, p, l, err_bad)


# ---------------------------------------------------------------------------------------------------------------------------------
# refusals (all before any launch)


def test_refusals(mb):
    from mlease_b200._native import MleaseError, lib
    from mlease_b200.admm import _internal_consensus
    r = np.random.default_rng(9)
    arr, _ = _rows(r, "fused", 200, 20)
    with mb.AdmmSession(2, 20, [1.0], regularizer=1) as s:
        s.add_partition_csr(0, arr["rowptr"], arr["colidx"], arr["vals"], arr["response"])
        with pytest.raises(MleaseError, match="begin"):
            _internal_consensus(s, read=False)
        s.begin()
        S = _internal_consensus(s)   # a read without stages
        st = {k: S[k] for k in ("vec", "fvec", "z", "exch", "diff", "ctrl")}
        for mask in (16, -1):
            with pytest.raises(MleaseError, match="stage mask"):
                _internal_consensus(s, mask, st)
        with pytest.raises(MleaseError, match="L2"):
            _internal_consensus(s, ["init"], st)
        with pytest.raises(MleaseError, match="iter >= 1"):
            _internal_consensus(s, ["consensus"], st, iter=0)
        bad = dict(st, ctrl=np.tile([0, 0, S["info"]["k1_grid"] + 1], (S["info"]["nprob"], 1)))
        with pytest.raises(MleaseError, match="k1_chunks"):
            _internal_consensus(s, ["pack"], bad)
        info = np.zeros(12, np.int32)
        fn = lib().mlease_internal_consensus
        rc = fn(s._h, 4, None, None, None, None, None, None, None, None, None, None, None, None, info.ctypes.data)
        assert rc != 0 and b"null" in lib().mlease_last_error()
