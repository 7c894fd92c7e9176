"""Time ItemModelTrain with the full posterior (mlease_item_model_train_cov) against the sparse call with the diagonal variance
(mlease_item_model_train_sparse, compute_var), one (intercept, default) pair, on two shapes:

    A' = 4096 keys x ~200 rows x 256 of 256 features (every key at the global width of 257 columns); the covariance output is
         4096 * 257 * 258 / 2 doubles = 1.09 GB, so the call with blocks is expected to be bound by that copy;
    W  = 4096 keys x ~200 rows x 20 entries a row from pools of 64 - 256 of 200 000 features (every key in its own space).

The cov call runs with and without out_cov.  Scoring: the shape's own rows under the models of a cov fit over the shape's grid (G = 1
at A', G = 4 at W), mlease_score_keyed_cov against mlease_score_keyed_var with the same models' diagonal variances.  CUDA events around each call, median of --reps after one warm-up call; a call returns when
its work is done, so this includes its host side.  Then, unless --no-profile, one cov call and one cov scoring call per shape under
torch.profiler (a run of its own): the summed device time of the posterior's kernels (row weights, Hessian assembly, the gather), of K3's Cholesky and inverse
kernels (the fits' own Newton rebuilds included) and of every kernel and copy of the call.

    python tools/time_item_model_cov.py
    python tools/time_item_model_cov.py --shapes W --reps 3

Prints one JSON line per (shape, call) with the card's name and power limit first; a call that fails is reported with its error."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from time_keyed_wide import data, timed  # noqa: E402

SHAPES = {"A'": dict(K=4096, rows=200, D=256, pool=(256, 256), entries=256, grid=([2.0], [1.0])),
          "W": dict(K=4096, rows=200, D=200000, pool=(64, 256), entries=20, grid=([2.0, 0.5], [1.0, 0.25]))}
# the posterior's kernels by name: row weights, the Hessian, K3's factorisation and inverse, the gather
GROUPS = {"rowweights": ("postvar_rowweight",), "hessian": ("postvar_hess_batch",),
          "factor_inverse": ("chol_", "trinv", "hinv_syrk", "dmma", "dgemm"), "gather": ("cov_gather",),
          "score_cov": ("score_keyed_cov_kernel",), "score_pred": ("score_keyed_kernel", "keyed_table_scatter")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="A',W")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-profile", action="store_true")
    a = ap.parse_args()
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "ml-ease_b200"))
    import mlease_b200 as mb
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"card": card.splitlines()}), flush=True)
    for name in a.shapes.split(","):
        s = SHAPES[name]
        krs, rp, ci, v, y = data(s["K"], s["rows"], s["D"], s["pool"], s["entries"])
        kw = dict(rowptr=rp, colidx=ci, num_features=s["D"])
        calls = {"sparse_var": lambda: mb.item_model_train_sparse(v, krs, y, [2.0], [1.0], compute_var=True, **kw),
                 "cov_var_only": lambda: mb.item_model_train_cov(v, krs, y, [2.0], [1.0], want_cov=False, **kw),
                 "cov": lambda: mb.item_model_train_cov(v, krs, y, [2.0], [1.0], **kw)}
        for call, fn in calls.items():
            rec = {"shape": name, "call": call, "keys": s["K"], "rows": int(krs[-1]), "nnz": int(rp[-1]), "features": s["D"]}
            try:
                ms, res = timed(fn, a.reps)
                rec.update(ms=round(ms, 2))
                if call == "cov":
                    rec.update(cov_bytes=int(res[5].nbytes))
                del res
            except Exception as e:   # reported, and the next call runs
                rec.update(error=str(e)[:300])
            print(json.dumps(rec), flush=True)
        il, dl = s["grid"]
        kp, cols, models, var, cp, cov = mb.item_model_train_cov(v, krs, y, il, dl, **kw)
        G = len(il) * len(dl)
        mp, mc, mv = mb.keyed_models_for_scoring(kp, cols, models)
        sp, sv = mb.keyed_cov_for_scoring(kp, cp, cov)
        _, _, vv = mb.keyed_models_for_scoring(kp, cols, var)
        vd = np.repeat(1.0 / np.array([d for _ in il for d in dl], np.float32), s["K"]).astype(np.float32)
        score = {"score_keyed_var": lambda: mb.score_keyed_var(v, krs, rp, ci, s["D"], mp, mc, mv, mp, mc, vv, vd),
                 "score_keyed_cov": lambda: mb.score_keyed_cov(v, krs, rp, ci, s["D"], mp, mc, mv, sp, sv, vd)}
        for call, fn in score.items():
            ms, _ = timed(fn, a.reps)
            print(json.dumps({"shape": name, "call": call, "G": G, "rows": int(krs[-1]), "ms": round(ms, 2)}), flush=True)
        if a.no_profile:
            continue
        import torch
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            calls["cov"]()
            score["score_keyed_cov"]()
            torch.cuda.synchronize()
        ms = {g: 0.0 for g in GROUPS}
        total = 0.0
        for ev in prof.events():
            if ev.device_type.name != "CUDA":
                continue
            t = ev.time_range.elapsed_us() / 1000.0
            total += t
            for g, keys in GROUPS.items():
                if any(k in ev.name for k in keys):
                    ms[g] += t
        print(json.dumps({"shape": name, "profile": "cov", "kernel_ms": {g: round(t, 2) for g, t in ms.items()},
                          "all_device_ms": round(total, 2)}), flush=True)


if __name__ == "__main__":
    main()
