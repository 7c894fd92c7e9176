#!/usr/bin/env python
"""Times the fused multi-lambda CSR K1 (k1_csr_fused_kernel) at the bench's partition shape, 1M x 10k x 100 stored values per
row (bench.py's partition 0), for L = 3 lambdas (the 4-wide interleave, LP = 4) and L = 1 (LP = 1): gradient passes over a
one-partition ADMM batch through the solver's launcher (the mlease_internal_batch_grad hook), plus the Hv and Hessian-diagonal
passes of the matrix-free solver.  Kernel time = the summed CUDA time of the k1_csr_fused_kernel launches under torch.profiler.
Byte model of one pass (what the kernel moves for all lambdas together, per-row terms and the gpart_f partials left out):
phase A reads the CSR rows, COLBYTES (2 for 16-bit column ids, 4 for int32) + 4 B per stored value; phase B the segment list,
6 B per slot incl. its padding.  Scratch tool for kernel work on a GPU box, not part of the product."""
import os
import sys
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "ml-ease_b200"))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile
import mlease_b200 as mb
from mlease_b200 import _hooks
import bench

REPS = int(os.environ.get("REPS", 20))
COLBYTES = int(os.environ.get("COLBYTES", 2))
dev = torch.device("cuda:0")
n, D, nnz = int(os.environ.get("ROWS", 1000000)), 10000, 100
beta = (np.random.default_rng(7).normal(size=D) / np.sqrt(nnz)).astype(np.float32)
rp, ci, vv, y = bench.gen_sparse(0, n, D, nnz, beta, dev)
print(torch.cuda.get_device_name(0), flush=True)


def kernel_ms(fn, tag):
    """Mean CUDA time of the k1_csr_fused_kernel<LP, mode> launches (tag) of REPS calls of fn (after two warm-up calls)."""
    fn(); fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(REPS):
            fn()
        torch.cuda.synchronize()
    us, cnt = 0.0, 0
    for e in prof.key_averages():
        if tag in e.key:
            us += e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            cnt += e.count
    assert cnt == REPS, (cnt, REPS)
    return us / cnt / 1e3


hv = _hooks.bound().mlease_internal_batch_hv
for L in (3, 1):
    lambdas = [0.1, 1.0, 10.0][:L] if L == 3 else [1.0]
    for policy in (0, 2):
        with mb.AdmmSession(1, D, lambdas, device=0, hessian_policy=policy) as s:
            s.add_partition_csr(0, rp, ci, vv, y)
            s.begin()
            W = np.tile(np.append(beta, -1.0).astype(np.float64), (L, 1))
            info = _hooks.batch_grad(s, W)
            assert info["kind"] == "fused", info["kind"]
            LP = info["G"]
            S, rows = info["chunks"][0], info["RT"]
            # phase B slots: the segment lists hold every stored value plus the padding of each group to its longest column
            # (not known here; the byte model counts the stored values, i.e. it is a lower bound on what phase B reads)
            nbytes = (COLBYTES + 4.0) * n * nnz + 6.0 * n * nnz
            if policy == 0:
                ms = kernel_ms(lambda: _hooks.batch_grad(s, W), "k1_csr_fused_kernel<%d, 0>" % LP)
                print("gradient pass L=%d (LP=%d, %d segments x %d rows): %.3f ms, %.0f GB/s of the byte model" %
                      (L, LP, S, rows, ms, nbytes / ms / 1e6), flush=True)
            else:
                V = np.ones((L, D + 1))
                out = np.zeros((L, D + 1))
                for mode, name in ((1, "Hv"), (2, "diagonal")):
                    def call():
                        assert hv(s._h, mode, W.ctypes.data, V.ctypes.data, out.ctypes.data) == 0
                    ms = kernel_ms(call, "k1_csr_fused_kernel<%d, %d>" % (LP, mode))
                    print("%s pass L=%d (LP=%d): %.3f ms, %.0f GB/s of the byte model" % (name, L, LP, ms, nbytes / ms / 1e6), flush=True)
