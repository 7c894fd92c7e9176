"""Time mlease_naive_train and mlease_item_model_train on CSR keys over a wide dictionary: fixed keys (K keys x ~rows rows x 20
entries a row by default, each key's entries drawn from its own pool of 64 - 256 columns spread over the dictionary) at several dictionary
widths.  Time by CUDA events around each call, median of --reps after one warm-up call; a call returns when its work is done, so
this includes its host side (the checks, the output arrays it fills).

    python tools/time_keyed_wide.py --features 2000,20000,200000
    python tools/time_keyed_wide.py --features 256 --pool 256,256 --rows 1 --entries 256 --dump /tmp/a   # every key full width

Prints one JSON line per (entry point, width); a call that fails (e.g. out of device memory) is reported with its error.  --dump DIR
writes each call's models (and variances) as .npy files, so the outputs of two builds can be compared file for file.  --root chooses
the source tree whose build is timed (default: this one).  The host outputs are L x K x (num_features + 1) doubles: 6.6 GB per
lambda at 4096 keys and 200 000 features.  The card's name and power limit are printed with the numbers."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np


def data(K, rows, D, pool, entries, seed=0):
    rng = np.random.default_rng(seed)
    nk = rng.integers(max(1, rows * 3 // 4), rows * 5 // 4 + 1, K)
    rp, ci = [np.zeros(1, np.int64)], []
    off = 0
    for k in range(K):
        P = int(rng.integers(pool[0], pool[1] + 1))
        cols = np.sort(rng.choice(D, P, replace=False)).astype(np.int32) if P < D else np.arange(D, dtype=np.int32)
        e = min(entries, P)
        pick = np.sort(np.argsort(rng.random((nk[k], P)), axis=1)[:, :e], axis=1)
        ci.append(cols[pick].reshape(-1))
        rp.append(off + e * np.arange(1, nk[k] + 1, dtype=np.int64))
        off += e * nk[k]
    ci = np.concatenate(ci)
    rp = np.concatenate(rp)
    n = int(nk.sum())
    v = rng.standard_normal(len(ci), dtype=np.float32)
    beta = rng.standard_normal(D, dtype=np.float32) * np.float32(0.3)
    z = np.add.reduceat(v * beta[ci], rp[:-1]) if len(ci) else np.zeros(n, np.float32)
    y = (rng.random(n, dtype=np.float32) < 1 / (1 + np.exp(-z))).astype(np.int32)
    krs = np.concatenate([[0], np.cumsum(nk)]).astype(np.int64)
    return krs, rp, ci, v, y


def timed(fn, reps):
    import torch
    fn()   # warm-up: modules, allocator
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keys", type=int, default=4096)
    ap.add_argument("--rows", type=int, default=200)
    ap.add_argument("--features", default="2000,20000,200000")
    ap.add_argument("--pool", default="64,256", help="min,max columns of a key's pool")
    ap.add_argument("--entries", type=int, default=20, help="entries a row")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--var", action="store_true", help="ItemModelTrain with compute_var")
    ap.add_argument("--dump", default="", help="write the models here as .npy")
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    a = ap.parse_args()
    sys.path.insert(0, os.path.join(os.path.abspath(a.root), "ml-ease_b200"))
    import mlease_b200 as mb
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"card": card.splitlines(), "root": os.path.abspath(a.root)}), flush=True)
    pool = tuple(int(x) for x in a.pool.split(","))
    if a.dump:
        os.makedirs(a.dump, exist_ok=True)
    for D in map(int, a.features.split(",")):
        krs, rp, ci, v, y = data(a.keys, a.rows, D, (min(pool[0], D), min(pool[1], D)), a.entries)
        calls = {
            "naive_train": lambda: mb.naive_train(v, krs, y, [1.0], rowptr=rp, colidx=ci, num_features=D),
            "item_model_train": lambda: mb.item_model_train(v, krs, y, [2.0], [1.0], rowptr=rp, colidx=ci, num_features=D, compute_var=a.var),
        }
        for name, fn in calls.items():
            rec = {"call": name, "keys": a.keys, "rows": int(krs[-1]), "nnz": int(rp[-1]), "features": D}
            try:
                ms, out = timed(fn, a.reps)
                rec.update(ms=round(ms, 2), fits_per_s=round(a.keys / ms * 1e3, 1))
                if a.dump:
                    for i, arr in enumerate(x for x in out if x is not None and x.dtype == np.float64):
                        np.save(os.path.join(a.dump, "%s_%d_%d.npy" % (name, D, i)), arr)
                del out
            except Exception as e:   # reported, and the next shape runs
                rec.update(error=str(e)[:300])
            print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
