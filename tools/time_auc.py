"""Time mlease_test_auc at the shape of a grid evaluation: 2^25 records x 12 sets (grid points), 100 000 item keys of Zipf-like
sizes (key k holds about n / ((k + 1) H_K) records), predictions, responses and weights resident on the device.  Reports the median
of 5 calls after one warm-up (CUDA events around each call), the bytes the kernels and sorts must move, and the time those bytes need
at the H100 SXM's 3.35 TB/s.  Prints one JSON line with the card's name and power limit.
    python tools/time_auc.py [--rows 33554432] [--sets 12] [--keys 100000]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "ml-ease_b200"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return q.strip().splitlines()[0] if q.strip() else "unknown"


def zipf_rowstart(n, K):
    h = 1.0 / np.arange(1, K + 1)
    sizes = np.floor(n * h / h.sum()).astype(np.int64)
    sizes[0] += n - sizes.sum()
    return np.r_[0, np.cumsum(sizes)].astype(np.int64)


def bytes_moved(n, S, K):
    """the bytes one call's kernels and radix sorts must move (onesweep: one histogram read of the keys, then per 8-bit pass a read
    and a write of keys and values); a gathered 4-byte value counts 4 bytes"""
    key_passes = max(1, -(-int(np.ceil(np.log2(max(K, 2)))) // 8))
    once = 8 * n + 8 * n + 2 * 4 * n                 # rows kernel: response, weight in; lw, kid out; the two weight passes
    per_set = (12 * n                                # pred in, orderable keys and row ids out
               + 4 * n + 4 * 16 * n                  # set sort: histogram, 4 passes of (4-byte key, 4-byte row)
               + 12 * n                              # set pass: keys, rows, gathered weights
               + 24 * n                              # pack: keys, rows, gathered key ids in; key ids, (key, row) pairs out
               + 4 * n + key_passes * 24 * n         # key sort: histogram, passes of (4-byte key id, 8-byte pair)
               + 12 * n)                             # key pass: pairs, gathered weights
    return once + S * per_set


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 25)
    ap.add_argument("--sets", type=int, default=12)
    ap.add_argument("--keys", type=int, default=100000)
    ap.add_argument("--profile", action="store_true", help="instead: one call under torch.profiler, device time per kernel name")
    a = ap.parse_args()
    import torch
    import mlease_b200 as mb
    n, S, K = a.rows, a.sets, a.keys
    g = torch.Generator(device="cuda").manual_seed(0)
    resp = (torch.rand(n, device="cuda", generator=g) < 0.05).to(torch.int32)
    pred = torch.randn((S, n), device="cuda", generator=g) + resp.float()
    w = torch.rand(n, device="cuda", generator=g) * 2
    krs = zipf_rowstart(n, K)
    times = []
    out = mb.test_auc(resp, pred, w, krs)   # warm-up
    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            mb.test_auc(resp, pred, w, krs)
            torch.cuda.synchronize()
        per = {}
        for e in prof.events():
            if e.device_type.name == "CUDA":
                k = e.name.split("(")[0].replace("(anonymous namespace)::", "")[:90]
                per[k] = per.get(k, 0.0) + (getattr(e, "device_time", None) or getattr(e, "cuda_time", 0.0)) / 1e3
        print(json.dumps({"card": card(), "kernel_ms": {k: round(v, 2) for k, v in sorted(per.items(), key=lambda x: -x[1])}}))
        return
    for _ in range(5):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        mb.test_auc(resp, pred, w, krs)
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    nb = bytes_moved(n, S, K)
    floor_ms = nb / 3.35e12 * 1e3
    ms = float(np.median(times))
    print(json.dumps({"card": card(), "rows": n, "sets": S, "keys": K, "largest_key": int(krs[1] - krs[0]), "median_ms": round(ms, 2),
                      "all_ms": [round(t, 2) for t in times], "bytes": nb, "floor_ms_at_3.35TBps": round(floor_ms, 2),
                      "x_floor": round(ms / floor_ms, 2), "auc": [round(float(x), 6) for x in out[0]]}))


if __name__ == "__main__":
    main()
