"""Seeded inputs of the fused CSR K1 golden cases (tests/test_gpu_k1_fused_stream.py, tests/golden/make_k1_fused_stream.py).

One case per lambda count L = 1 .. 4 (LP = 1, 2, 4, 4).  Every partition has 4097 rows, cut by k1f_plan into 9 segments of 456 rows
(the last one 449 rows).  The rows exercise what the kernel's streaming has to get right:
- rows longer than the 112 register-resident entries of phase A (every 37th row holds 113 .. 290 entries);
- an empty segment (segment 4: all its rows are empty);
- segment starts at every residue of the CSR entry index mod 8, i.e. every 2-byte residue of the 16-bit column ids and every
  4-byte residue of the fp32 values mod 16 bytes (the last row of the previous segment is lengthened to get there);
- L = 1 runs at 50 000 features, so that column ids >= 32768 occur (16-bit ids must not sign-extend)."""
import hashlib

import numpy as np

import k1_reference as kr

N_ROWS = 4097
SEG_ROWS, SEGS = 456, 9     # k1f_plan at 4097 rows on 132 SMs: 9 segments (whole 512-row blocks), ceil(4097 / 9) rows each
EMPTY_SEG = 4
# target residue (mod 8) of the first entry of each segment; segment 5 starts where the empty segment 4 does
TARGET = {0: 0, 1: 1, 2: 2, 3: 3, 4: 4, 6: 6, 7: 7, 8: 5}


def case_shape(L):
    """-> (partitions, features, lambdas)."""
    if L == 1:
        return 1, 50000, [1.0]
    return 2, 301, [0.5 * (l + 1) for l in range(L)]


def make_part(seed, D):
    """One partition: dict(rowptr, colidx, vals, response, weight, offset) and its k1_reference Part."""
    rng = np.random.default_rng(seed)
    n = N_ROWS
    lens = rng.integers(1, 40, n)
    longr = np.arange(n) % 37 == 11
    lens[longr] = rng.integers(113, 291, longr.sum())
    lens[EMPTY_SEG * SEG_ROWS:(EMPTY_SEG + 1) * SEG_ROWS] = 0
    for s in range(1, SEGS):
        if s not in TARGET:
            continue
        last = s * SEG_ROWS - 1
        start = int(lens[:s * SEG_ROWS].sum())
        lens[last] += (TARGET[s] - start) % 8
    rowptr = np.zeros(n + 1, np.int64)
    rowptr[1:] = np.cumsum(lens)
    cols = [np.sort(rng.choice(D, size=int(k), replace=False)) for k in lens]
    colidx = np.concatenate(cols).astype(np.int32)
    vals = rng.normal(size=len(colidx)).astype(np.float32)
    response = (rng.random(n) < 0.5).astype(np.int32)
    weight = rng.uniform(0.5, 2.0, n).astype(np.float32)
    offset = rng.normal(0, 0.1, n).astype(np.float32)
    arr = dict(rowptr=rowptr, colidx=colidx, vals=vals, response=response, weight=weight, offset=offset)
    return arr, kr.Part.from_csr(rowptr, colidx, vals, response, weight, offset, D)


def make_case(L):
    """-> (arrays of each partition, Parts, W [P L, Dt] points, V [P L, Dt] Hv vectors, digest of all inputs)."""
    P, D, _ = case_shape(L)
    built = [make_part(1300 + 10 * L + p, D) for p in range(P)]
    arrs, parts = [a for a, _ in built], [p for _, p in built]
    W = []
    for p in range(P):
        W += kr.make_betas(D, L, 1400 + 10 * L + p)
    W = np.array(W)
    V = np.random.default_rng(1500 + L).normal(size=W.shape)
    h = hashlib.sha256()
    for a in arrs:
        for k in sorted(a):
            h.update(np.ascontiguousarray(a[k]).tobytes())
    h.update(W.tobytes()); h.update(V.tobytes())
    return arrs, parts, W, V, h.hexdigest()


def run_case(mb, L):
    """The gradient pass (with sqrt(d)), the Hv pass and the Hessian-diagonal pass of case L through the solver's launchers.
    -> dict(g, f, sd [P L, n], hv, diag, info (of the gradient pass), digest)."""
    from mlease_b200._native import check, ptr
    from mlease_b200 import _hooks
    P, D, lambdas = case_shape(L)
    arrs, parts, W, V, digest = make_case(L)
    fn = _hooks.bound().mlease_internal_batch_hv
    with mb.AdmmSession(P, D, lambdas, hessian_policy=2) as s:
        for p, a in enumerate(arrs):
            s.add_partition_csr(p, a["rowptr"], a["colidx"], a["vals"], a["response"], a["weight"], a["offset"])
        s.begin()
        info = _hooks.batch_grad(s, W, rows=[N_ROWS] * P, want_sd=True)
        out = dict(g=info["g"], f=info["f"], sd=np.stack(info["sd"]), info=info, digest=digest)
        for mode, name in ((1, "hv"), (2, "diag")):
            o = np.zeros_like(W)
            check(fn(s._h, mode, ptr(W), ptr(V), ptr(o)))
            out[name] = o
    return out
