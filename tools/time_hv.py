#!/usr/bin/env python
"""Times ONE Hv pass (the K1_HV mode of the CSR K1 kernels + its fixed-order reduction, what every CG step of a matrix-free
x-update runs) through mlease_time_kernel(which=4), at 1M x 10k x 1 % (the bench's partition 0) and 1M x 100k x 100 per row.
Byte model of one pass (what it must move at least): the CSR rows (8 B per stored value: column id + value, 8 B row pointer per
row) + sqrt(d) per row (4 B); the segment-list kernel also reads its column-major copy (6 B per stored value + padding), which
the model leaves out.  Scratch tool for kernel work on a GPU box, not part of the product."""
import os, sys
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "ml-ease_b200"))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np
import torch
import mlease_b200 as mb
import bench

dev = torch.device("cuda:0")
n, nnz = int(os.environ.get("ROWS", 1000000)), 100
for D in (10000, 100000):
    beta = (np.random.default_rng(7).normal(size=D) / np.sqrt(nnz)).astype(np.float32)
    rp, ci, vv, y = bench.gen_sparse(0, n, D, nnz, beta, dev)
    with mb.AdmmSession(1, D, [1.0], device=0, hessian_policy=2) as s:
        s.add_partition_csr(0, rp, ci, vv, y)
        ms = s.time_kernel(0, "hv", reps=10)
    nbytes = 8.0 * n * nnz + 8.0 * n + 4.0 * n
    print("Hv pass %d x %d x %d/row: %.3f ms, %.0f GB/s of the byte model" % (n, D, nnz, ms, nbytes / ms / 1e6))
    del rp, ci, vv, y
    torch.cuda.empty_cache()
