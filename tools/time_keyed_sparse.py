"""Time the keyed CSR fits with dense outputs (mlease_naive_train, mlease_item_model_train) against the same fits with sparse
outputs (mlease_naive_train_sparse, mlease_item_model_train_sparse) on the shapes of tools/time_keyed_wide.py: 4096 keys x ~200 rows x
20 entries a row, each key's entries drawn from its own pool of 64 - 256 columns, at several dictionary widths; NaiveTrain with one
lambda, ItemModelTrain with one (intercept, default) pair without and with the posterior variance.  Time by CUDA events around each
call, median of --reps after one warm-up call; a call returns when its work is done, so this includes its host side (the checks, the
output arrays it fills).  Then one shape only the sparse calls can run: 50 000 keys of 1 - 8 rows over 2 000 000 features, whose
dense output would be 800 GB a lambda.

    python tools/time_keyed_sparse.py
    python tools/time_keyed_sparse.py --features 20000 --no-big

Prints one JSON line per (entry point, output, width) with the card's name and power limit first; a call that fails is reported with
its error."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from time_keyed_wide import data, timed  # noqa: E402


def big_data(K, D, seed=1):
    """K keys of 1 - 8 rows, each row 20 sorted unique columns of the key's pool of 40 random columns of [0, D)"""
    rng = np.random.default_rng(seed)
    nk = rng.integers(1, 9, K)
    ci, rl = [], []
    for k in range(K):
        p = np.unique(rng.integers(0, D, 40))
        pick = np.sort(np.argsort(rng.random((nk[k], len(p))), axis=1)[:, :20], axis=1)
        ci.append(p[pick].reshape(-1)); rl.append(np.full(nk[k], pick.shape[1]))
    ci = np.concatenate(ci).astype(np.int32)
    rp = np.concatenate([[0], np.cumsum(np.concatenate(rl))]).astype(np.int64)
    v = rng.standard_normal(len(ci), dtype=np.float32)
    y = (rng.random(int(nk.sum())) < 0.4).astype(np.int32)
    return np.concatenate([[0], np.cumsum(nk)]).astype(np.int64), rp, ci, v, y


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keys", type=int, default=4096)
    ap.add_argument("--rows", type=int, default=200)
    ap.add_argument("--features", default="2000,20000,200000")
    ap.add_argument("--entries", type=int, default=20, help="entries a row")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-big", action="store_true", help="skip the 50 000 x 2 000 000 shape")
    a = ap.parse_args()
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "ml-ease_b200"))
    import mlease_b200 as mb
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"card": card.splitlines()}), flush=True)

    def calls(krs, rp, ci, v, y, D, dense):
        kw = dict(rowptr=rp, colidx=ci, num_features=D)
        nt = mb.naive_train if dense else mb.naive_train_sparse
        it = mb.item_model_train if dense else mb.item_model_train_sparse
        return {"naive_train": lambda: nt(v, krs, y, [1.0], **kw),
                "item_model_train": lambda: it(v, krs, y, [2.0], [1.0], **kw),
                "item_model_train_var": lambda: it(v, krs, y, [2.0], [1.0], compute_var=True, **kw)}

    def run(krs, rp, ci, v, y, D, outputs):
        for out in outputs:
            for name, fn in calls(krs, rp, ci, v, y, D, out == "dense").items():
                rec = {"call": name, "output": out, "keys": len(krs) - 1, "rows": int(krs[-1]), "nnz": int(rp[-1]), "features": D}
                try:
                    ms, res = timed(fn, a.reps)
                    rec.update(ms=round(ms, 2))
                    del res
                except Exception as e:   # reported, and the next shape runs
                    rec.update(error=str(e)[:300])
                print(json.dumps(rec), flush=True)

    for D in map(int, a.features.split(",")):
        krs, rp, ci, v, y = data(a.keys, a.rows, D, (min(64, D), min(256, D)), a.entries)
        run(krs, rp, ci, v, y, D, ("dense", "sparse"))
    if not a.no_big:
        D = 2000000
        run(*big_data(50000, D), D, ("sparse",))


if __name__ == "__main__":
    main()
