#!/usr/bin/env python
"""Times the Cholesky + inverse bucket at the bench shape (cfg3: 4 partitions x 10k features, lambdas 0.1 / 1 / 10): the cold
start of a run factorises the 4 partitions' leaders (ldh 10016) in one batch, the 8 followers parked.  Prints the card, its power
limit, the bucket's CUDA-event time (AdmmSession.profile) and a torch.profiler breakdown of the same bucket's kernels:
prep, diag/panel/in-panel update (the NB = 32 chain), trailing update, trinv leaves, TF32 merges, ysym.  With a look-ahead the
chain overlaps the trailing update, so the groups can add up to more than the bucket.  ROWS=n sets the rows per partition
(the factorisation does not depend on it), ONE=1 also times one factorisation through mlease_time_kernel, OUT=path writes JSON.
Scratch tool for kernel work on a GPU box, not part of the product."""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "ml-ease_b200"))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
import mlease_b200 as mb  # noqa: E402

GROUPS = (("prep", ("chol_prep_kernel",)),
          ("chain: diag", ("chol_diag_kernel",)),
          ("chain: panel", ("chol_panel_kernel",)),
          ("chain: in-panel update", ("chol_update_kernel",)),
          ("trailing update (DMMA)", ("dgemm_kernel<true, true>", "syrk_kernel")),
          ("trinv leaves", ("trinv_kernel",)),
          ("TF32 merges", ("merge_tf32_kernel",)),
          ("ysym", ("ysym_kernel",)),
          ("finish / share", ("chol_finish_kernel", "chol_share", "ysym_detach")))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def main():
    dev = torch.device("cuda:0")
    P, D, nnz, lambdas = 4, 10_000, 100, [0.1, 1.0, 10.0]
    n = int(os.environ.get("ROWS", 100_000))
    print("card (name, power limit, max SM clock):", card(), flush=True)
    beta = (np.random.default_rng(7).normal(size=D) / np.sqrt(nnz)).astype(np.float32)
    s = mb.AdmmSession(P, D, lambdas, device=0, epsilon=0.0)
    for p in range(P):
        rp, ci, vv, y = bench.gen_sparse(p, n, D, nnz, beta, dev)
        s.add_partition_csr(p, rp, ci, vv, y)
        del rp, ci, vv, y
    torch.cuda.empty_cache()
    s.run(1)                           # warm-up: module loads, allocations, one cold-start factorisation
    torch.cuda.synchronize()
    res = dict(card=card(), rows=n)
    s.profile(2)
    s.run(1)
    torch.cuda.synchronize()
    res["bucket_ms_events"] = [s.profile(0)["ms"]["cholesky"]]
    s.profile(2)
    s.run(1)
    torch.cuda.synchronize()
    res["bucket_ms_events"].append(s.profile(0)["ms"]["cholesky"])
    print("cholesky bucket (CUDA events, one cold start of 4 leaders): %s ms" % ", ".join("%.2f" % v for v in res["bucket_ms_events"]))

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        s.run(1)
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    groups = {g: [0.0, 0] for g, _ in GROUPS}
    first, last = None, None
    for e in ev:
        for g, keys in GROUPS:
            if any(k in e.name for k in keys):
                t0, t1 = e.time_range.start, e.time_range.end
                groups[g][0] += (t1 - t0) / 1e3
                groups[g][1] += 1
                first = t0 if first is None else min(first, t0)
                last = t1 if last is None else max(last, t1)
                break
    print("%-26s %10s %8s" % ("group", "kernel ms", "launches"))
    for g, (ms, cnt) in groups.items():
        print("%-26s %10.3f %8d" % (g, ms, cnt))
    span = (last - first) / 1e3 if first is not None else 0.0
    print("span first..last bucket kernel: %.3f ms (kernel sum %.3f ms)" % (span, sum(v[0] for v in groups.values())))
    res["groups_ms"] = {g: v[0] for g, v in groups.items()}
    res["groups_launches"] = {g: v[1] for g, v in groups.items()}
    res["span_ms"] = span
    if os.environ.get("ONE") == "1":
        one = s.time_kernel(0, "cholesky", reps=3)
        print("one factorisation + inverse (mlease_time_kernel): %.3f ms" % one)
        res["one_problem_ms"] = one
    s.close()
    if os.environ.get("OUT"):
        with open(os.environ["OUT"], "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
