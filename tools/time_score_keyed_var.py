"""Time keyed scoring with predictive variance (mlease_score_keyed_var, ItemModelGridTest) against plain keyed scoring
(mlease_score_keyed) on the same device data, with CUDA events on an H100, the two calls alternating.  Prints the card name and
power limit first: the figures hold for that card only.  Rows list sorted, unique columns, as mlease_score_keyed_var requires.

  A  NaiveTrain-like: 20 000 keys x 200 rows x 256 of 256 features, G = 1 and 4 grid points
  W  wide sparse:     10 000 keys x 200 rows x 100 of 10 000 features, G = 4 (the plain call's tables take two 1 GiB chunks, the
                      variance call's three)

Algorithmic bytes, as tools/time_score_keyed.py counts them: 8 nnz (column + value) + 16 n (rowptr, offset, pred) + 4 G n (pred) +
8 model entries; the variance call adds 4 G n (pred_var) + 8 variance entries + 4 G K (var_default).  Share = bytes / time over the
3.35 TB/s data-sheet HBM3 rate.  A call's time includes the host's model and variance checks and their upload; the kernel time
(torch.profiler) is the table fills and the scoring kernel."""
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "ml-ease_b200"))
import mlease_b200 as mb  # noqa: E402

HBM = 3.35e12


def problem(rng, K, rows, nnz, D, G):
    g = torch.Generator(device="cuda").manual_seed(0)
    n = K * rows
    krs = torch.arange(K + 1, dtype=torch.int64, device="cuda") * rows
    rp = torch.arange(n + 1, dtype=torch.int64, device="cuda") * nnz
    if nnz == D:
        ci = torch.arange(D, dtype=torch.int32, device="cuda").repeat(n)
    else:   # one column in each of nnz equal slices of [0, D): sorted and unique
        step = D // nnz
        ci = (torch.arange(nnz, dtype=torch.int32, device="cuda") * step).repeat(n)
        ci += torch.randint(0, step, (n * nnz,), generator=g, dtype=torch.int32, device="cuda")
    v = torch.randn(n * nnz, generator=g, device="cuda")
    off = torch.zeros(n, dtype=torch.float32, device="cuda")
    per = min(D, 256) + 1   # a model (and its variance list) lists a 256-feature subset + intercept
    cols = np.concatenate([np.sort(rng.choice(D, per - 1, replace=False)), [D]]).astype(np.int32)
    mc = torch.from_numpy(np.tile(cols, G * K)).cuda()
    mv = torch.randn(G * K * per, generator=g, device="cuda") * 0.1
    mp = torch.arange(G * K + 1, dtype=torch.int64, device="cuda") * per
    vv = torch.rand(G * K * per, generator=g, device="cuda")
    vd = torch.full((G * K,), 0.1, dtype=torch.float32, device="cuda")
    return dict(krs=krs, rp=rp, ci=ci, v=v, off=off, mp=mp, mc=mc, mv=mv, vv=vv, vd=vd, D=D, K=K, G=G, n=n, nnz=n * nnz, nme=G * K * per)


def plain(p, out):
    mb.score_keyed(p["v"], p["krs"], p["rp"], p["ci"], p["D"], p["mp"], p["mc"], p["mv"], offset=p["off"], out=out)


def with_var(p, out, out_var):
    mb.score_keyed_var(p["v"], p["krs"], p["rp"], p["ci"], p["D"], p["mp"], p["mc"], p["mv"], p["mp"], p["mc"], p["vv"], p["vd"], offset=p["off"],
                       out=out, out_var=out_var)


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def kernel_ms(fn):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    kt = {e.key: e.device_time_total / 1e3 for e in prof.key_averages()}
    return (sum(t for k, t in kt.items() if "score_keyed_kernel" in k),
            sum(t for k, t in kt.items() if "keyed_table_scatter" in k or "Memset" in k))


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print("card:", q.stdout.strip())
    rng = np.random.default_rng(0)
    for name, K, rows, nnz, D, G in (("A", 20000, 200, 256, 256, 1), ("A", 20000, 200, 256, 256, 4), ("W", 10000, 200, 100, 10000, 4)):
        p = problem(rng, K, rows, nnz, D, G)
        out = torch.empty((G, p["n"]), dtype=torch.float32, device="cuda")
        out_var = torch.empty_like(out)
        fp, fv = (lambda: plain(p, out)), (lambda: with_var(p, out, out_var))
        for f in (fp, fv, fp, fv):   # warm-up, and the two preds agree bitwise
            f()
        ref = out.clone()
        with_var(p, out, out_var)
        assert torch.equal(ref.view(torch.int32), out.view(torch.int32)), "pred of the variance call differs from mlease_score_keyed"
        ms_p, ms_v = [], []
        for _ in range(4):   # alternate, so both see the same host and clock state
            ms_p.append(timed(fp, 3))
            ms_v.append(timed(fv, 3))
        mp_, mv_ = float(np.median(ms_p)), float(np.median(ms_v))
        kp, tp = kernel_ms(fp)
        kv, tv = kernel_ms(fv)
        by_p = 8 * p["nnz"] + 16 * p["n"] + 4 * G * p["n"] + 8 * p["nme"]
        by_v = by_p + 4 * G * p["n"] + 8 * p["nme"] + 4 * G * K
        print("%s G=%d: %d keys x %d rows x %d of %d features" % (name, G, K, rows, nnz, D))
        for lab, ms, k, t, by in (("score_keyed    ", mp_, kp, tp, by_p), ("score_keyed_var", mv_, kv, tv, by_v)):
            print("   %s call %.2f ms (spread %.2f-%.2f), %.1f %% of 3.35 TB/s; scoring kernel %.3f ms = %.1f %% of 3.35 TB/s, table fill %.3f ms"
                  % (lab, ms, min(ms_p if by == by_p else ms_v), max(ms_p if by == by_p else ms_v), 100 * by / (ms * 1e-3) / HBM, k,
                     100 * by / (k * 1e-3) / HBM, t))
        print("   var / plain: call %.2fx, scoring kernel %.2fx, kernels incl. table fill %.2fx" % (mv_ / mp_, kv / kp, (kv + tv) / (kp + tp)))
        del p, out, out_var
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
