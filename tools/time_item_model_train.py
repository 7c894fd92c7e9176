"""Time ItemModelTrain's device call (mlease_item_model_train) on an H100: a 3 x 3 (intercept lambda x default lambda) grid on two
shapes, with and without the batched posterior variance, and the per-key route it replaces (one session, upload, fit_partition and
posterior_variance per key and grid point).  Prints the card name and power limit first: the figures hold for that card only.

  A  NaiveTrain-like: 20 000 keys x 200 rows x 256 of 256 features
  B  wide sparse:     10 000 keys x 500 rows x 100 of 10 000 features

Call time = host clock around one call ending in a device synchronise (the call returns its results on the host), after a warm-up
call on the first keys.  Variance kernel time = the postvar_* kernels of one call under torch.profiler, in a run of its own."""
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "ml-ease_b200"))
import mlease_b200 as mb  # noqa: E402

IL, DL = [1.0, 10.0, 100.0], [0.1, 1.0, 10.0]


def problem(K, rows, nnz, D):
    g = torch.Generator(device="cuda").manual_seed(0)
    n = K * rows
    krs = np.arange(K + 1, dtype=np.int64) * rows
    rp = torch.arange(n + 1, dtype=torch.int64, device="cuda") * nnz
    if nnz == D:
        ci = torch.arange(D, dtype=torch.int32, device="cuda").repeat(n)
    else:
        ci = torch.sort(torch.randint(0, D, (n, nnz), generator=g, dtype=torch.int32, device="cuda"), dim=1).values.reshape(-1)
    v = torch.randn(n * nnz, generator=g, device="cuda") * (1.0 / np.sqrt(nnz))
    y = torch.randint(0, 2, (n,), generator=g, dtype=torch.int32, device="cuda")
    means = np.random.default_rng(0).normal(0, 1, K)
    return dict(krs=krs, rp=rp, ci=ci, v=v, y=y, means=means, D=D, K=K, rows=rows, nnz=nnz)


def call(p, var, K=None):
    K = p["K"] if K is None else K
    n = K * p["rows"]
    return mb.item_model_train(p["v"][:n * p["nnz"]], p["krs"][:K + 1], p["y"][:n], IL, DL, rowptr=p["rp"][:n + 1], colidx=p["ci"][:n * p["nnz"]],
                               num_features=p["D"], intercept_prior_mean=p["means"][:K], compute_var=var)


def per_key_route(p, keys, budget_s=120.0):
    """ms per key of the per-key route: session + upload + (fit_partition + posterior_variance) per grid point"""
    D, rows, nnz = p["D"], p["rows"], p["nnz"]
    rp = (torch.arange(rows + 1, dtype=torch.int64) * nnz).numpy()
    t0 = time.perf_counter()
    done = 0
    for k in keys:
        a = k * rows * nnz
        ci, v, y = (t.cpu().numpy() for t in (p["ci"][a:a + rows * nnz], p["v"][a:a + rows * nnz], p["y"][k * rows:(k + 1) * rows]))
        with mb.AdmmSession(1, D, [1.0], epsilon=0.0) as s:
            s.add_partition_csr(0, rp, ci, v, y)
            for il in IL:
                for dl in DL:
                    q = np.full(D + 1, 1.0 / (1.0 / np.float64(np.float32(dl)))); q[D] = 1.0 / (1.0 / np.float64(np.float32(il)))
                    m = np.zeros(D + 1); m[D] = p["means"][k]
                    x, _ = s.fit_partition(0, np.zeros(D + 1), m, q)
                    s.posterior_variance(0, x, q)
        done += 1
        if time.perf_counter() - t0 > budget_s:
            break
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / done, done


def main():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="AB", help="which shapes to run: A, B or AB")
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print("card:", q.stdout.strip(), flush=True)
    for name, K, rows, nnz, D in (("A", 20000, 200, 256, 256), ("B", 10000, 500, 100, 10000)):
        if name not in args.shapes:
            continue
        p = problem(K, rows, nnz, D)
        fits = K * len(IL) * len(DL)
        call(p, True, K=500)                           # warm-up: module load, first allocations
        torch.cuda.synchronize()
        res = {}
        for var in (False, True):
            t0 = time.perf_counter()
            call(p, var)
            torch.cuda.synchronize()
            res[var] = time.perf_counter() - t0
            print("%s %d keys x %d rows x %d of %d, 3 x 3 grid, compute_var=%d: call %.2f s, %.0f fits/s"
                  % (name, K, rows, nnz, D, var, res[var], fits / res[var]), flush=True)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            call(p, True)
            torch.cuda.synchronize()
        kt = {e.key: e.device_time_total / 1e3 for e in prof.key_averages()}
        k_var = sum(t for k, t in kt.items() if "postvar_" in k)
        k_all = sum(t for k, t in kt.items() if "Memcpy" not in k and "Memset" not in k)
        print("   variance kernels %.1f ms per call = %.2f %% of the unprofiled call with variance, %.2f %% of all kernel time; "
              "call with minus without variance: %.2f s" % (k_var, 100 * k_var / 1e3 / res[True], 100 * k_var / max(k_all, 1e-9), res[True] - res[False]),
              flush=True)
        keys = np.random.default_rng(1).choice(K, 100, replace=False)
        ms_pk, n_done = per_key_route(p, keys)
        print("   per-key route (session + upload + 9 x (fit_partition + posterior_variance)): %.2f ms per key over %d keys; "
              "batched call %.3f ms per key" % (ms_pk, n_done, res[True] * 1e3 / K), flush=True)
        del p
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
