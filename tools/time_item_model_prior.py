"""Time ItemModelTrain under per-key priors (mlease_item_model_train_prior) against the same fits without them
(mlease_item_model_train_sparse) on the shape of tools/time_keyed_sparse.py: 4096 keys x ~200 rows x 20 entries a row, each key's
entries drawn from its own pool of 64 - 256 of 200 000 features, over a 3 x 3 (intercept, default) lambda grid with the posterior
variance; priors on every column a key lists plus a quarter as many prior-only columns and the intercept, a third of the variances 0.
Calls are timed by CUDA events, alternating the two, median of --reps after one warm-up each; a call returns when its work is done.
Then one call of each under torch.profiler gives the device time of the kernels the priors add or change.

    python tools/time_item_model_prior.py [--reps 5] [--out /tmp/prior_trace.json]

Prints one JSON line per measurement, the card's name and power limit first."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from time_keyed_wide import data  # noqa: E402

KERNELS = ("prior_check_kernel", "prior_only_count_kernel", "prior_init_kernel", "naive_init_kernel", "local_init_kernel",
           "sparse_gather_kernel", "span_present_kernel")


def priors(krs, rp, ci, D, seed=1):
    """every listed column of each key, plus 25 % prior-only columns and the intercept; means N(0, 0.5), variances U(0.05, 2) or 0"""
    rng = np.random.default_rng(seed)
    pp, pc = [0], []
    for k in range(len(krs) - 1):
        listed = np.unique(ci[rp[krs[k]]:rp[krs[k + 1]]])
        extra = np.setdiff1d(rng.integers(0, D, max(1, len(listed) // 4)), listed)
        c = np.concatenate([np.union1d(listed, extra), [D]]).astype(np.int32)
        pc.append(c); pp.append(pp[-1] + len(c))
    pc = np.concatenate(pc)
    pm = rng.normal(0, 0.5, len(pc))
    pv = np.where(rng.random(len(pc)) < 1 / 3, 0.0, rng.uniform(0.05, 2.0, len(pc)))
    return np.array(pp, np.int64), pc, pm, pv


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keys", type=int, default=4096)
    ap.add_argument("--rows", type=int, default=200)
    ap.add_argument("--features", type=int, default=200000)
    ap.add_argument("--entries", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="", help="write the profiler's trace here")
    a = ap.parse_args()
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "ml-ease_b200"))
    import torch
    import mlease_b200 as mb
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"card": card.splitlines()}), flush=True)
    D = a.features
    krs, rp, ci, v, y = data(a.keys, a.rows, D, (64, 256), a.entries)
    pp, pc, pm, pv = priors(krs, rp, ci, D)
    il, dl = [0.5, 2.0, 8.0], [0.3, 1.0, 4.0]
    kw = dict(rowptr=rp, colidx=ci, num_features=D, compute_var=True)
    calls = {"sparse": lambda: mb.item_model_train_sparse(v, krs, y, il, dl, **kw),
             "prior": lambda: mb.item_model_train_prior(v, krs, y, il, dl, prior_ptr=pp, prior_col=pc, prior_mean=pm, prior_var=pv, **kw)}
    print(json.dumps({"keys": a.keys, "rows": int(krs[-1]), "nnz": int(rp[-1]), "features": D, "grid": len(il) * len(dl),
                      "prior_entries": int(pp[-1])}), flush=True)
    for fn in calls.values():
        fn()   # warm-up: modules, allocator
    ts = {name: [] for name in calls}
    for _ in range(a.reps):
        for name, fn in calls.items():
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            fn()
            e.record()
            e.synchronize()
            ts[name].append(s.elapsed_time(e))
    ms = {name: float(np.median(t)) for name, t in ts.items()}
    for name in calls:
        print(json.dumps({"call": name, "ms_median": round(ms[name], 2), "ms_all": [round(t, 2) for t in ts[name]]}), flush=True)
    print(json.dumps({"overhead_pct": round(100.0 * (ms["prior"] / ms["sparse"] - 1.0), 2)}), flush=True)
    from torch.profiler import ProfilerActivity, profile
    for name, fn in calls.items():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        tot, per = 0.0, {}
        for ev in prof.events():
            if ev.device_type.name != "CUDA":
                continue
            t = ev.device_time_total / 1000.0 if hasattr(ev, "device_time_total") else ev.cuda_time_total / 1000.0
            tot += t
            for kname in KERNELS:
                if kname in ev.name:
                    per[kname] = per.get(kname, 0.0) + t
        print(json.dumps({"call": name, "device_ms": round(tot, 2), "kernel_ms": {k: round(x, 3) for k, x in per.items()}}),
              flush=True)
        if a.out and name == "prior":
            prof.export_chrome_trace(a.out)


if __name__ == "__main__":
    main()
