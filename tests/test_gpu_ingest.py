"""The upload path of a session partition (-m gpu) against numpy, through the read-only hooks partition_info / partition_data:
labels, weights and offsets as stored; dense rows staged from the host through several two-buffer chunks (the last one partial)
and from a strided device tensor, bit for bit, with the intercept column and the padding; the CSR scalars that set the fixed-point
scales of the CSR K1 and Hv passes (vmax, rowl1, wmax), the Gram product count, the sorted-rows flag that picks the deterministic
kernels; the binary.feature rewrite; an all-empty partition's gradient; and the refusals of malformed input, each of which stays
inside the buffers it describes."""
import numpy as np
import pytest

import k1_reference as kr

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24
REPORT = []


@pytest.fixture(scope="module")
def mb():
    import mlease_b200
    return mlease_b200


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    for line in REPORT:
        print(line)


def _hooks():
    from mlease_b200 import _hooks
    return _hooks


def _csr(rows):
    """list of (cols, vals) -> rowptr, colidx, vals"""
    rp = np.cumsum([0] + [len(c) for c, _ in rows]).astype(np.int64)
    ci = np.concatenate([np.asarray(c, np.int32) for c, _ in rows] or [np.zeros(0, np.int32)]).astype(np.int32)
    v = np.concatenate([np.asarray(x, np.float32) for _, x in rows] or [np.zeros(0, np.float32)]).astype(np.float32)
    return rp, ci, v


def _labels(rng, n):
    return rng.integers(-1, 2, n).astype(np.int32), rng.uniform(0.25, 4.0, n).astype(np.float32), rng.normal(0, 3, n).astype(np.float32)


# ---- labels ----------------------------------------------------------------------------------------------------------------------
def test_labels_weights_offsets(mb):
    rng = np.random.default_rng(1)
    n, Dg = 3001, 12
    resp = rng.integers(-1, 2, n).astype(np.int32)
    w = rng.uniform(0, 3, n).astype(np.float32)
    w[::17] = 0.0
    w[5] = np.float32(1e-40)              # subnormal
    w[2999] = np.float32(7.5000005)       # the lone largest, in the last warp of rows
    o = rng.normal(0, 5, n).astype(np.float32)
    o[7] = -0.0
    rp, ci, v = _csr([([i % Dg], [1.0]) for i in range(n)])
    s = mb.AdmmSession(2, Dg, [1.0])
    s.add_partition_csr(0, rp, ci, v, resp, w, o)
    s.add_partition_csr(1, rp, ci, v, resp)   # no weight, no offset
    H = _hooks()
    info = H.partition_info(s, 0)
    d = H.partition_data(s, 0, info)
    np.testing.assert_array_equal(d["y"], np.where(resp == 1, 1, -1).astype(np.int8))
    assert set(np.unique(resp)) == {-1, 0, 1}
    np.testing.assert_array_equal(d["w"].view(np.uint32), w.view(np.uint32))
    np.testing.assert_array_equal(d["o"].view(np.uint32), o.view(np.uint32))
    assert info["wmax"] == w.max() and info["n"] == n and info["nnz"] == n and info["csr"]
    d1 = H.partition_data(s, 1)
    np.testing.assert_array_equal(d1["y"], d["y"])
    np.testing.assert_array_equal(d1["w"], np.ones(n, np.float32))
    np.testing.assert_array_equal(d1["o"].view(np.uint32), np.zeros(n, np.uint32))
    assert H.partition_info(s, 1)["wmax"] == np.float32(1.0)
    s.close()


@pytest.mark.parametrize("what", ["response 2", "weight -1", "weight nan"])
def test_label_refusals(mb, what):
    rng = np.random.default_rng(2)
    n, Dg = 300, 8
    resp, w, o = _labels(rng, n)
    if what == "response 2":
        resp[n - 1] = 2
    elif what == "weight -1":
        w[n // 2] = -1.0
    else:
        w[3] = np.nan
    rp, ci, v = _csr([([i % Dg], [1.0]) for i in range(n)])
    s = mb.AdmmSession(1, Dg, [1.0])
    with pytest.raises(mb.MleaseError) as e:
        s.add_partition_csr(0, rp, ci, v, resp, w, o)
    assert e.value.code == 1 and ("response" if what.startswith("response") else "weight") in e.value.message
    with pytest.raises(mb.MleaseError) as e:     # not left behind half-added
        _hooks().partition_info(s, 0)
    assert "not resident" in e.value.message
    s.close()


# ---- dense rows ------------------------------------------------------------------------------------------------------------------
def test_dense_staging_host_and_device(mb):
    """A host partition streamed through 4 staging chunks (the last one of 17 rows) and the same rows from a device tensor whose
    rows are ldx_in = 4100 floats apart: X bit for bit in both, column Dg = 1, padding = +0, and the same K1 gradient bits."""
    import torch
    Dg, ld_in, n = 4093, 4100, 24569
    chunk = max(1, (128 << 20) // (4 * ld_in))
    nchunks = -(-n // chunk)
    assert nchunks >= 4 and n % chunk != 0
    REPORT.append("dense staging: %d rows of %d floats in %d chunks of %d rows, the last of %d" % (n, ld_in, nchunks, chunk, n - (nchunks - 1) * chunk))
    rng = np.random.default_rng(3)
    X = rng.standard_normal((n, ld_in), dtype=np.float32)
    X[:, Dg:] = np.nan                        # past Dg: never read
    for r in (0, chunk - 1, chunk, 2 * chunk + 5, n - 1):
        X[r, :7] = [-0.0, 1e-42, -1e-45, 3e30, -3e30, 1.0, 0.0]
    resp, w, o = _labels(rng, n)
    s = mb.AdmmSession(2, Dg, [1.0])
    s.add_partition_dense(0, X, resp, w, o)
    Xd = torch.from_numpy(X).cuda()
    assert Xd.stride(0) == ld_in
    s.add_partition_dense(1, Xd, resp, w, o)
    H = _hooks()
    ldx = (Dg + 1 + 3) // 4 * 4
    for pid in (0, 1):
        info = H.partition_info(s, pid)
        assert (info["n"], info["nnz"], info["csr"], info["ldx"]) == (n, 0, False, ldx)
        assert info["wmax"] == w.max()
        got = H.partition_data(s, pid, info)
        np.testing.assert_array_equal(got["y"], np.where(resp == 1, 1, -1).astype(np.int8))
        np.testing.assert_array_equal(got["w"], w)
        np.testing.assert_array_equal(got["o"], o)
        G = got["X"]
        for r0 in range(0, n, 2048):   # in slices: no full-size temporaries
            a, b = G[r0:r0 + 2048], X[r0:r0 + 2048]
            bad = np.flatnonzero((a[:, :Dg].view(np.uint32) != b[:, :Dg].view(np.uint32)).any(axis=1))
            assert len(bad) == 0, (pid, "rows differ", r0 + bad[:8], "chunk", (r0 + bad[0]) // chunk)
            assert np.all(a[:, Dg] == 1.0), (pid, r0)
            assert np.all(a[:, Dg + 1:].view(np.uint32) == 0), (pid, r0)
        del G, got
    del Xd
    torch.cuda.empty_cache()
    s.begin()
    beta = np.random.default_rng(4).normal(0, 0.01, Dg + 1)
    res = H.batch_grad(s, np.stack([beta, beta]))
    assert res["kind"] == "dense" and np.all(np.isfinite(res["g"][0]))
    np.testing.assert_array_equal(res["g"][0].view(np.uint64), res["g"][1].view(np.uint64))
    assert res["f"][0] == res["f"][1]
    s.close()


# ---- CSR scalars ---------------------------------------------------------------------------------------------------------------
def _row_l1_bounds(rp, v):
    a = np.abs(v.astype(np.float64))
    k = np.diff(rp)
    l1 = np.add.reduceat(a, rp[:-1]) if len(a) else np.zeros(len(k))
    l1[k == 0] = 0.0
    return float((l1 * (1 - k * U32)).max()), float((l1 * (1 + k * U32)).max())


def test_csr_scalars(mb):
    """vmax = max |v| exactly (with -0.0, subnormals and a lone large value), rowl1 within the fp32 row-sum bound of the fp64
    row-L1 maximum, gram_pairs = sum (k + 1)(k + 2) / 2 exactly, and the lists of a sorted partition built."""
    rng = np.random.default_rng(5)
    n, Dg = 5000, 700
    rows = []
    for i in range(n):
        k = int(rng.choice([0, 1, 2, 7, 31, 32, 33, 64])) if i % 97 else 600
        c = np.sort(rng.choice(Dg, size=k, replace=False))
        x = rng.normal(0, 1, k).astype(np.float32) * np.float32(2.0 ** rng.integers(-20, 20))
        rows.append((c, x))
    rp, ci, v = _csr(rows)
    v[3] = -0.0
    v[10:20] = np.float32(1e-41) * np.arange(1, 11, dtype=np.float32)
    r = 4321 + int(np.flatnonzero(np.diff(rp)[4321:] >= 2)[0])
    v[int(rp[r]) + 1] = np.float32(-6.0e25)   # the lone largest |value|, second in its row
    assert (np.abs(v) == np.float32(6.0e25)).sum() == 1
    resp, w, o = _labels(rng, n)
    s = mb.AdmmSession(1, Dg, [1.0])
    s.add_partition_csr(0, rp, ci, v, resp, w, o)
    H = _hooks()
    info = H.partition_info(s, 0)
    assert info["vmax"] == np.abs(v).max() == np.float32(6.0e25)
    lo, hi = _row_l1_bounds(rp, v)
    assert lo <= float(info["rowl1"]) <= hi, (info["rowl1"], lo, hi)
    k = np.diff(rp).astype(np.int64)
    assert info["gram_pairs"] == int(((k + 1) * (k + 2) // 2).sum())
    assert info["csr_unique"] and info["block_major"] and info["gram_col_index"]
    assert info["wmax"] == w.max()
    np.testing.assert_array_equal(H.partition_data(s, 0, info)["vals"].view(np.uint32), v.view(np.uint32))
    s.close()


def _sorted_rows(rng, n, Dg, k):
    c = np.sort(np.stack([rng.choice(Dg, size=k, replace=False) for _ in range(min(n, 64))]), axis=1)
    return np.tile(c, (-(-n // len(c)), 1))[:n].astype(np.int32)


@pytest.mark.parametrize("case", ["repeat in the last row", "descent in the last row", "repeat past row 1048576"])
def test_csr_unique_flag(mb, case):
    """One row breaks the strictly increasing column order: csr_unique is 0 and the lists of the sorted kernels are not built."""
    rng = np.random.default_rng(6)
    Dg = 40
    n = 1_100_000 if "past" in case else 3000
    cols = _sorted_rows(rng, n, Dg, 2)
    bad = 1_050_000 if "past" in case else n - 1
    cols[bad] = [9, 9] if "repeat" in case else [20, 3]
    rp = np.arange(n + 1, dtype=np.int64) * 2
    v = rng.uniform(0.5, 1.5, 2 * n).astype(np.float32)
    resp, w, o = _labels(rng, n)
    s = mb.AdmmSession(2, Dg, [1.0])
    s.add_partition_csr(0, rp, cols.reshape(-1), v, resp, w, o)
    good = _sorted_rows(rng, 3000, Dg, 2)
    s.add_partition_csr(1, np.arange(3001, dtype=np.int64) * 2, good.reshape(-1), v[:6000], resp[:3000], w[:3000], o[:3000])
    H = _hooks()
    info = H.partition_info(s, 0)
    assert not info["csr_unique"], case
    assert not info["block_major"] and not info["k1_segments"] and info["gram_pairs"] == 0
    assert H.partition_info(s, 1)["csr_unique"]
    s.close()


# ---- binary.feature ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("on_device", [False, True])
def test_binary_feature(mb, on_device):
    rng = np.random.default_rng(7)
    n, Dg = 2000, 300
    rows = [(np.sort(rng.choice(Dg, size=int(rng.integers(0, 90)), replace=False)), None) for _ in range(n)]
    rows = [(c, rng.normal(0, 50, len(c)).astype(np.float32)) for c, _ in rows]
    rp, ci, v = _csr(rows)
    v[:5] = [0.0, -0.0, -7.0, 1e-42, 3e30]
    keep = v.copy()
    resp, w, o = _labels(rng, n)
    s = mb.AdmmSession(1, Dg, [1.0], binary_feature=True)
    if on_device:
        import torch
        t = [torch.from_numpy(a).cuda() for a in (rp, ci, v)]
        s.add_partition_csr(0, t[0], t[1], t[2], resp, w, o)
        torch.cuda.synchronize()
        np.testing.assert_array_equal(t[2].cpu().numpy().view(np.uint32), keep.view(np.uint32))
    else:
        s.add_partition_csr(0, rp, ci, v, resp, w, o)
    H = _hooks()
    info = H.partition_info(s, 0)
    np.testing.assert_array_equal(v.view(np.uint32), keep.view(np.uint32))
    np.testing.assert_array_equal(H.partition_data(s, 0, info)["vals"], np.ones(len(v), np.float32))
    assert info["vmax"] == 1.0 and info["rowl1"] == np.float32(np.diff(rp).max())
    s.close()


# ---- an empty partition ----------------------------------------------------------------------------------------------------------
def test_empty_partition_gradient(mb):
    """nnz = 0: every row empty.  The gradient is the intercept's alone, within the fp64 reference's bound; the features' are 0."""
    rng = np.random.default_rng(8)
    n, Dg = 777, 9
    resp, w, o = _labels(rng, n)
    rp = np.zeros(n + 1, np.int64)
    ci, v = np.zeros(0, np.int32), np.zeros(0, np.float32)
    s = mb.AdmmSession(1, Dg, [1.0])
    s.add_partition_csr(0, rp, ci, v, resp, w, o)
    H = _hooks()
    info = H.partition_info(s, 0)
    assert info["nnz"] == 0 and info["vmax"] == 0 and info["rowl1"] == 0
    s.begin()
    part = kr.Part.from_csr(rp, ci, v, resp, w, o, Dg)
    beta = rng.normal(0, 0.5, Dg + 1)
    res = H.batch_grad(s, beta[None, :])
    ref = kr.reference(part, beta)
    plan = kr.plan_from_info(res, 0, n)
    bnd, _ = kr.grad_bound(part, ref, plan, kr.row_errors(part, ref, plan))
    assert np.all(res["g"][0][:Dg] == 0.0)
    assert np.all(kr.ratio(res["g"][0] - ref.g, bnd) <= 1.0), (res["g"][0][Dg], ref.g[Dg], bnd[Dg])
    assert abs(res["f"][0] - ref.f) <= kr.loss_bound(part, ref, plan)
    s.close()


# ---- refusals ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("col", ["Dg", "-1"])
def test_colidx_out_of_range(mb, col):
    """A column id outside [0, Dg) is reported by the next session call (the checks of a partition run while the next one
    uploads), naming the partition."""
    rng = np.random.default_rng(9)
    n, Dg = 500, 16
    rp, ci, v = _csr([([i % 7, 8 + i % 5], [1.0, 2.0]) for i in range(n)])
    ci[len(ci) - 1 if col == "Dg" else 0] = Dg if col == "Dg" else -1
    resp, w, o = _labels(rng, n)
    s = mb.AdmmSession(2, Dg, [1.0])
    s.add_partition_csr(1, rp, ci, v, resp, w, o)
    ci2 = ci.copy()
    ci2[ci2 < 0] = 0
    ci2[ci2 >= Dg] = 0
    with pytest.raises(mb.MleaseError) as e:
        s.add_partition_csr(0, rp, ci2, v, resp, w, o)
    assert e.value.code == 1 and "partition 1" in e.value.message and "out of range" in e.value.message
    s.close()


def _overlapping_rowptr():
    """rowptr that decreases once, every entry inside [0, rowptr[n]]: rows 1 and 3 overlap row 2."""
    rp = np.array([0, 4, 2, 6, 3, 8], np.int64)
    ci = np.array([0, 1, 2, 3, 4, 5, 6, 7], np.int32)
    return rp, ci, np.ones(8, np.float32)


def test_decreasing_rowptr_session(mb):
    rng = np.random.default_rng(10)
    rp, ci, v = _overlapping_rowptr()
    n = len(rp) - 1
    resp, w, o = _labels(rng, n)
    s = mb.AdmmSession(1, 8, [1.0])
    s.add_partition_csr(0, rp, ci, v, resp, w, o)
    with pytest.raises(mb.MleaseError) as e:
        _hooks().partition_info(s, 0)
    assert e.value.code == 1 and "partition 0" in e.value.message and "rowptr" in e.value.message
    s.close()


def test_decreasing_rowptr_naive_train(mb):
    rng = np.random.default_rng(11)
    rp, ci, v = _overlapping_rowptr()
    n = len(rp) - 1
    resp, w, o = _labels(rng, n)
    with pytest.raises(mb.MleaseError) as e:
        mb.naive_train(v, np.array([0, n], np.int64), resp, [1.0], rowptr=rp, colidx=ci, num_features=8, weight=w, offset=o)
    assert e.value.code == 1 and "rowptr" in e.value.message
