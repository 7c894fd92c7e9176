"""Time NaiveTrain at the cfg5 shape (dense, 1k rows x 256 features per key): K keys resident, K keys streamed through one GPU,
and the same K sharded over 1, 2, 4, 8 GPUs the way the keyed jobs shard them (contiguous key ranges, one host thread per device).

    python tools/time_keyed_scale.py --keys 8192 --stream-keys 24576 --gpus 1,2,4,8
    python tools/time_keyed_scale.py --keys 4096 --stream-keys 4096 --score-keys 4096 --budget 4000000000

--score-keys adds streamed scoring (mlease_score_keyed under the --budget cap) of the same rows as a CSR of every feature, one
model per key; its fits_per_s counts the keys scored.  Prints one JSON line per run: fits/s and, for streamed fits, the share of
the staging time (host copy into the pinned ring + H2D, on a staging thread) hidden behind the solve.  Streamed scoring queues its
copies from the calling thread: it prints the staging time only.  The full 100k-key size needs ~103 GB of host RAM (X alone is
102.4 GB); --keys / --stream-keys choose
what runs, and runs of the same K share one data set.  The card's
name and power limit are printed with the numbers."""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np



def data(K, rows, D, seed=0):
    """float32 throughout: X is the only large array (K * rows * D * 4 bytes)"""
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((K * rows, D), dtype=np.float32)
    beta = rng.standard_normal(D, dtype=np.float32) / np.float32(np.sqrt(D))
    y = (rng.random(K * rows, dtype=np.float32) < 1 / (1 + np.exp(-(X @ beta)))).astype(np.int32)
    return X, y, np.arange(K + 1, dtype=np.int64) * rows


def fit(X, y, krs, devs):
    """NaiveTrain over len(devs) devices: contiguous equal-cost key ranges (every key has the same rows), one thread each."""
    import mlease_b200 as mb
    K = len(krs) - 1
    cuts = [K * s // len(devs) for s in range(len(devs) + 1)]
    out, err = [None] * len(devs), []

    def run(s):
        a, b = krs[cuts[s]], krs[cuts[s + 1]]
        try:
            out[s] = mb.naive_train(X[a:b], krs[cuts[s]:cuts[s + 1] + 1] - a, y[a:b], [1.0], device=devs[s])[0]
        except Exception as e:
            err.append(e)
    ts = [threading.Thread(target=run, args=(s,)) for s in range(len(devs))]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    if err:
        raise err[0]
    return np.concatenate(out, axis=1)


def score(X, krs, ci, model):
    """mlease_score_keyed of X's rows as a CSR listing every feature (ci: the column ids of at least X's rows), key k's rows scored
    with model[k]"""
    import mlease_b200 as mb
    n, D = X.shape
    K = len(krs) - 1
    mp = np.arange(K + 1, dtype=np.int64) * (D + 1)
    mc = np.tile(np.arange(D + 1, dtype=np.int32), K)
    return mb.score_keyed(X.reshape(-1), krs, np.arange(n + 1, dtype=np.int64) * D, ci[:n * D], D, mp, mc, model.reshape(-1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keys", type=int, default=8192)
    ap.add_argument("--stream-keys", type=int, default=0, help="K of the streamed one-GPU run (0: none)")
    ap.add_argument("--rows", type=int, default=1000)
    ap.add_argument("--features", type=int, default=256)
    ap.add_argument("--gpus", default="1")
    ap.add_argument("--score-keys", type=int, default=0, help="K of the streamed scoring run (0: none)")
    ap.add_argument("--budget", type=int, default=0, help="cap the device bytes of the streamed runs (forces streaming on a large GPU)")
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))), help="the checkout whose package runs")
    a = ap.parse_args()
    sys.path.insert(0, os.path.join(os.path.abspath(a.root), "ml-ease_b200"))
    import torch

    from mlease_b200 import _hooks
    ndev = torch.cuda.device_count()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"card": card.splitlines(), "devices": ndev, "root": os.path.abspath(a.root)}), flush=True)
    runs = [("resident", a.keys, [1])] + [("sharded", a.keys, [g]) for g in map(int, a.gpus.split(",")) if g > 1]
    if a.stream_keys:
        runs.append(("streamed", a.stream_keys, [1]))
    if a.score_keys:
        runs.append(("score_streamed", a.score_keys, [1]))
    cached = [None, None]   # [K, (X, y, krs)]
    for name, K, (g,) in runs:
        if g > ndev:
            print(json.dumps({"run": name, "keys": K, "gpus": g, "measured": False, "reason": "only %d devices" % ndev}), flush=True)
            continue
        _hooks.set_keyed_budget(a.budget if name.endswith("streamed") else 0)
        if cached[0] != K:
            cached[:] = [K, None]          # the previous data set is released before the next one is made
            cached[1] = data(K, a.rows, a.features)
        X, y, krs = cached[1]
        if name == "score_streamed":
            model = np.random.default_rng(1).standard_normal((K, a.features + 1), dtype=np.float32) / np.float32(16)
            ci = np.tile(np.arange(a.features, dtype=np.int32), len(X))
            run = lambda X, y, krs, devs: score(X, krs, ci, model[:len(krs) - 1])   # noqa: E731
        else:
            run = fit
        run(X[:krs[64]], y[:krs[64]], krs[:65], list(range(g)))          # warm-up: modules, allocator
        t0 = time.perf_counter()
        run(X, y, krs, list(range(g)))
        dt = time.perf_counter() - t0
        bounds, streamed, stage_ms, wait_ms = _hooks.keyed_last_call()
        rec = {"run": name, "keys": K, "rows": a.rows, "features": a.features, "gpus": g, "seconds": round(dt, 3), "fits_per_s": round(K / dt, 1),
               "streamed": streamed, "chunks": len(bounds) - 1}
        if streamed and name == "score_streamed":
            rec.update(stage_ms=round(stage_ms, 1))
        elif streamed:
            rec.update(stage_ms=round(stage_ms, 1), wait_ms=round(wait_ms, 1), hidden=round(1 - wait_ms / stage_ms, 3) if stage_ms else None)
        print(json.dumps(rec), flush=True)
        del X, y


if __name__ == "__main__":
    main()
