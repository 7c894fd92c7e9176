"""Time the ADMM model's posterior at config 3's shape (4 partitions x 1M rows x 10k features, 100 entries a row, lambda in
{0.1, 1, 10}) after a 5-iteration job: the Hessian assembly per partition and K3's factorisation + inverse (kernel times from
torch.profiler), the whole call in full and diagonal mode, score_var over 1M rows with the dense Sigma and with the diagonal (a host
clock around calls that end in a device synchronise; warm-up, median of 5), and the existing atomic kernel of
mlease_posterior_variance on one partition for comparison.  Prints one JSON line with the card's name and power limit.
    python tools/time_admm_posterior.py [--rows 1000000] [--features 10000] [--parts 4]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "ml-ease_b200"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return q.strip().splitlines()[0] if q.strip() else "unknown"


def partition(rng, n, D, per_row):
    # per_row strata of D / per_row columns, one column from each: strictly increasing, per_row entries a row
    w = D // per_row
    cols = (np.arange(per_row, dtype=np.int32)[None, :] * w + rng.integers(0, w, (n, per_row), dtype=np.int32)).reshape(-1)
    vals = rng.normal(0, 1, n * per_row).astype(np.float32)
    rowptr = np.arange(n + 1, dtype=np.int64) * per_row
    y = (rng.random(n) < 0.3).astype(np.int32)
    return rowptr, cols, vals, y


def median_ms(fn, reps=5):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def kernel_ms(fn, names):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {k: [] for k in names}
    for e in prof.events():
        for k in names:
            if k in e.name and e.device_type.name == "CUDA":
                out[k].append(e.device_time_total / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1000000)
    ap.add_argument("--features", type=int, default=10000)
    ap.add_argument("--parts", type=int, default=4)
    ap.add_argument("--per-row", type=int, default=100)
    a = ap.parse_args()
    import torch
    import mlease_b200 as mb
    rng = np.random.default_rng(0)
    D, P = a.features, a.parts
    res = {"card": card(), "shape": "%d x %d x %d, %d a row" % (P, a.rows, D, a.per_row)}
    s = mb.AdmmSession(P, D, [0.1, 1.0, 10.0])
    parts = []
    for p in range(P):
        rp, ci, v, y = partition(rng, a.rows, D, a.per_row)
        s.add_partition_csr(p, rp, ci, v, y)
        if p == 0:
            parts.append((rp, ci, v))
    s.run(5)
    # kernel times of one full call: the Hessian assembly (one launch per partition) and K3
    k = kernel_ms(lambda: s.admm_posterior(1, full=True), ["postvar_hess_col_kernel", "chol", "trinv", "syrk", "dgemm", "hinv", "merge"])
    res["hessian_assembly_ms_per_partition"] = k.pop("postvar_hess_col_kernel")
    res["factor_and_inverse_ms_per_lambda"] = sum(sum(v) for v in k.values())
    res["call_full_ms"] = median_ms(lambda: s.admm_posterior(1, full=True))
    res["call_diag_ms"] = median_ms(lambda: s.admm_posterior(1, full=False))
    var, cov = s.admm_posterior(1, full=True, want_cov=True)
    z = s.z(1)
    rp, ci, v = parts[0]
    dev = [torch.from_numpy(x).cuda() for x in (rp, ci, v)]
    dcov, dvar, dz = torch.from_numpy(cov).cuda(), torch.from_numpy(var).cuda(), torch.from_numpy(z).cuda()
    res["score_var_dense_ms"] = median_ms(lambda: mb.score_var(*dev, dz, cov=dcov))
    res["score_var_diag_ms"] = median_ms(lambda: mb.score_var(*dev, dz, var=dvar))
    res["score_ms"] = median_ms(lambda: mb.score(dev[2], dz, rowptr=dev[0], colidx=dev[1], num_features=D))
    del dcov, cov
    # the existing atomic kernel (one partition, mlease_posterior_variance(full = 1)) at the same z and q
    q = np.full(D + 1, np.float64(np.float32(1.0)))
    q[D] = 0.0
    try:
        ka = kernel_ms(lambda: s.posterior_variance(0, z, q, full=True), ["postvar_hess_csr_kernel"])
        res["atomic_kernel_ms_one_partition"] = ka["postvar_hess_csr_kernel"]
    except Exception as e:   # noqa: BLE001
        res["atomic_kernel_ms_one_partition"] = "failed: %s" % e
    print(json.dumps(res))


if __name__ == "__main__":
    main()
