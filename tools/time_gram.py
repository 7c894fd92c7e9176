#!/usr/bin/env python
"""Times one CSR Gram build with each kernel (e4m3 wgmma, exact sparse) on the same upload, at several densities at D = 10k plus
the bench shape (1M x 10k x 1 %) and `bench.py --features 500` (1M x 500 x 20 %), through mlease_time_kernel; prints which kernel
the automatic rule picks for each and a least-squares fit of the cost constants of batch_alloc's rule (csrc/batch.cu).
OUT=path also writes the table as JSON.  SHAPES=bench keeps the bench shape only.
WHICH=cholesky: times the factorisation + inverse of one 10k-wide system instead (ROWS=100000 keeps the data small).
Scratch tool for kernel work on a GPU box, not part of the product."""
import ctypes as C
import json
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "ml-ease_b200"))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
import mlease_b200 as mb  # noqa: E402
from mlease_b200 import _hooks  # noqa: E402
from mlease_b200._native import check  # noqa: E402

WGMMA, SPARSE = 1, 2
dev = torch.device("cuda:0")
REPS = int(os.environ.get("REPS", 3))


def session(n, D, nnz):
    beta = (np.random.default_rng(7).normal(size=D) / np.sqrt(nnz)).astype(np.float32)
    rp, ci, vv, y = bench.gen_sparse(0, n, D, nnz, beta, dev, chunk=max(1000, min(250_000, 200_000_000 // D)))
    s = mb.AdmmSession(1, D, [1.0], device=0)
    s.add_partition_csr(0, rp, ci, vv, y)
    del rp, ci, vv, y
    torch.cuda.empty_cache()
    return s


def time_gram(s, kind):
    """ms per build with the kernel `kind` (0: the automatic choice), and the kind that ran"""
    L = _hooks.bound()
    check(L.mlease_internal_set_csr_gram(s._h, kind))
    ms = s.time_kernel(0, "gram", reps=REPS)
    b, sc = C.c_int32(), C.c_int32()
    check(L.mlease_internal_csr_gram(s._h, C.byref(b), C.byref(sc)))
    return ms, sc.value


def main():
    if os.environ.get("WHICH", "gram") == "cholesky":
        n, D = int(os.environ.get("ROWS", 100000)), 10000
        with session(n, D, 100) as s:
            # factorisation + inverse of ONE 10k-wide system (factored direction: TF32 merges of the inverse)
            ms = s.time_kernel(0, "cholesky", reps=3)
            print("cholesky+inverse ms per factorisation", ms)
        return
    # (rows, features, stored values per row): the row counts keep each upload near 10^8 stored values
    shapes = [(1_000_000, 10_000, 100), (1_000_000, 500, 100), (1_000_000, 10_000, 30), (1_000_000, 10_000, 150),
              (1_000_000, 10_000, 200), (300_000, 10_000, 300), (100_000, 10_000, 1000), (30_000, 10_000, 2000)]
    if os.environ.get("SHAPES") == "bench":
        shapes = shapes[:1]
    print("device:", torch.cuda.get_device_name(0))
    rows = []
    for n, D, nnz in shapes:
        with session(n, D, nnz) as s:
            ms_w, _ = time_gram(s, WGMMA)
            ms_s, _ = time_gram(s, SPARSE)
            _, auto = time_gram(s, 0)
        Dp = (D + 1 + 127) // 128 * 128   # ldx rounds D + 1 up to a multiple of 4; Dp to 128
        nblk = Dp // 128
        tiles, groups = nblk * (nblk + 1) // 2, (n + 31) // 32
        r = dict(n=n, D=D, nnz=nnz, density=nnz / D, ms_wgmma=ms_w, ms_sparse=ms_s, auto="sparse" if auto == SPARSE else "wgmma",
                 macs_wgmma=tiles * 128.0 * 128.0 * 32.0 * groups, pairs=n * (nnz + 1) * (nnz + 2) / 2.0,
                 entries=float(n * (nnz + 1)), cells=0.5 * Dp * (Dp + 1.0), reads=(nblk + 1.0) * n * (nnz + 1))
        rows.append(r)
        print("n %8d D %6d nnz/row %5d (%5.2f %%): wgmma %9.3f ms  sparse %9.3f ms  auto %s" %
              (n, D, nnz, 100.0 * nnz / D, ms_w, ms_s, r["auto"]), flush=True)
    fit = {}
    full = rows   # every shape here has more columns than the sparse kernel's grid
    if len(full) >= 3:
        # the rule's models, relative least squares (every shape weighs the same):
        #   sparse  s = s/pair * pairs + s/entry * entries (column positions) + s/cell * cells of the lower triangle (epilogues)
        #   wgmma   s = s/MAC * MACs + s/read * entries read (the producers' run loads)
        for name, key, cols in (("sparse", "ms_sparse", ("pairs", "entries", "cells")), ("wgmma", "ms_wgmma", ("macs_wgmma", "reads"))):
            A = np.array([[r[c] for c in cols] for r in full])
            t = np.array([r[key] * 1e-3 for r in full])
            c, *_ = np.linalg.lstsq(A / t[:, None], np.ones(len(full)), rcond=None)
            fit[name] = dict(zip(cols, c))
            print("%s fit (s per unit):" % name, {k: "%.3e" % v for k, v in fit[name].items()})
            for r in full:
                print("   %s model %9.3f ms  measured %9.3f ms  (%d x %d x %d)" %
                      (name, 1e3 * sum(ci * r[k] for ci, k in zip(c, cols)), r[key], r["n"], r["D"], r["nnz"]))
    if os.environ.get("OUT"):
        with open(os.environ["OUT"], "w") as f:
            json.dump(dict(device=torch.cuda.get_device_name(0), rows=rows, fit=fit), f, indent=1)


if __name__ == "__main__":
    main()
