"""Time keyed multi-lambda scoring (mlease_score_keyed, ItemModelTest) with CUDA events on an H100, and the per-key route
through mlease_score for comparison.  Prints the card name and power limit first: the figures hold for that card only.

  A  NaiveTrain-like: 20 000 keys x 200 rows x 256 of 256 features, L = 1 and 3
  B  wide sparse:     10 000 keys x 500 rows x 100 of 10 000 features, L = 3 (several table chunks)

Algorithmic bytes = 8 nnz (column + value) + 16 n (rowptr, offset, pred at L = 1 ... counted once) + 4 L n (pred) + 8 model
entries (column + value); share = bytes / time over the 3.35 TB/s data-sheet HBM3 rate.  The table share is the time of the
table zero + scatter kernels over all kernels of one call (torch.profiler).  The call time includes the host's
model checks and the model upload."""
import subprocess
import sys
import os

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "ml-ease_b200"))
import mlease_b200 as mb  # noqa: E402

HBM = 3.35e12


def problem(rng, K, rows, nnz, D, L):
    g = torch.Generator(device="cuda").manual_seed(0)
    n = K * rows
    krs = torch.arange(K + 1, dtype=torch.int64, device="cuda") * rows
    rp = torch.arange(n + 1, dtype=torch.int64, device="cuda") * nnz
    if nnz == D:
        ci = torch.arange(D, dtype=torch.int32, device="cuda").repeat(n)
    else:
        ci = torch.randint(0, D, (n * nnz,), generator=g, dtype=torch.int32, device="cuda")
    v = torch.randn(n * nnz, generator=g, device="cuda")
    off = torch.zeros(n, dtype=torch.float32, device="cuda")
    per = min(D, 256) + 1   # a NaiveTrain model lists the features its rows list; here a 256-feature subset + intercept
    cols = np.concatenate([np.sort(rng.choice(D, per - 1, replace=False)), [D]]).astype(np.int32)
    mc = torch.from_numpy(np.tile(cols, L * K)).cuda()
    mv = torch.randn(L * K * per, generator=g, device="cuda") * 0.1
    mp = torch.arange(L * K + 1, dtype=torch.int64, device="cuda") * per
    return dict(krs=krs, rp=rp, ci=ci, v=v, off=off, mp=mp, mc=mc, mv=mv, D=D, K=K, L=L, n=n, nnz=n * nnz, nme=L * K * per)


def call(p, out):
    mb.score_keyed(p["v"], p["krs"], p["rp"], p["ci"], p["D"], p["mp"], p["mc"], p["mv"], offset=p["off"], out=out)


def timed(fn, reps):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print("card:", q.stdout.strip())
    rng = np.random.default_rng(0)
    for name, K, rows, nnz, D, L in (("A", 20000, 200, 256, 256, 1), ("A", 20000, 200, 256, 256, 3), ("B", 10000, 500, 100, 10000, 3)):
        p = problem(rng, K, rows, nnz, D, L)
        out = torch.empty((L, p["n"]), dtype=torch.float32, device="cuda")
        ms = timed(lambda: call(p, out), 5)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            call(p, out)
            torch.cuda.synchronize()
        kt = {e.key: e.device_time_total / 1e3 for e in prof.key_averages()}   # ms per kernel name
        k_score = sum(t for k, t in kt.items() if "score_keyed_kernel" in k)
        k_table = sum(t for k, t in kt.items() if "keyed_table_scatter" in k or "Memset" in k)
        by = 8 * p["nnz"] + 16 * p["n"] + 4 * L * p["n"] + 8 * p["nme"]
        print("%s L=%d: %d keys x %d rows x %d of %d: call %.2f ms, %.0f GB/s algorithmic = %.1f %% of 3.35 TB/s; kernels: scoring %.2f ms "
              "(%.1f %% of 3.35 TB/s), table zero + scatter %.2f ms (%.0f %% of kernel time)"
              % (name, L, K, rows, nnz, D, ms, by / ms / 1e6, 100 * by / ms / 1e-3 / HBM, k_score, 100 * by / k_score / 1e-3 / HBM, k_table,
                 100 * k_table / max(k_score + k_table, 1e-9)))
        if L == 1:   # today's route: one mlease_score call per key (first 1 000 keys)
            rp, ci, v = p["rp"], p["ci"], p["v"]
            krs, mp, mc, mv = p["krs"].cpu().numpy(), p["mp"].cpu().numpy(), p["mc"].cpu().long(), p["mv"].cpu().double()
            subs = []
            for k in range(1000):
                a, b = int(krs[k]), int(krs[k + 1])
                m = torch.zeros(D + 1, dtype=torch.float64)
                m[mc[mp[k]:mp[k + 1]]] = mv[mp[k]:mp[k + 1]]
                r0, r1 = int(rp[a]), int(rp[b])
                subs.append((v[r0:r1], m.cuda(), (rp[a:b + 1] - r0).contiguous(), ci[r0:r1], torch.empty(b - a, device="cuda")))
            ms_pk = timed(lambda: [mb.score(s[0], s[1], rowptr=s[2], colidx=s[3], num_features=D, out=s[4]) for s in subs], 2)
            print("   per-key mlease_score: %.3f ms per key (1 000 keys), keyed call %.4f ms per key" % (ms_pk / 1000, ms / K))


if __name__ == "__main__":
    main()
