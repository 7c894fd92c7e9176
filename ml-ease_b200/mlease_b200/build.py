"""In-tree build of libmlease_b200.so (nvcc, sm_90a only).  `python -m mlease_b200.build`."""
from __future__ import annotations

import os
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)            # ml-ease_b200/
CSRC = os.path.join(ROOT, "csrc")
LIBDIR = os.path.join(ROOT, "lib")
SO = os.path.join(LIBDIR, "libmlease_b200.so")
SOURCES = ["session.cu", "batch.cu", "ingest.cu", "keyed_fit.cu", "keyed_cols.cu", "key_ranges.cu", "test_hooks.cu", "k1_score_grad.cu", "k1_csr_fused.cu", "newton.cu", "k2_gram.cu", "k3_cholesky.cu", "k4_consensus.cu", "k5_score.cu", "k6_postvar.cu", "k7_auc.cu", "comm.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC",
         "--expt-relaxed-constexpr", "-Xptxas", "-v"]


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(LIBDIR, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(os.path.dirname(ROOT), "include", "mlease_b200.h"))
    objs = []
    procs = []
    for src in SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(LIBDIR, src.replace(".cu", ".o"))
        objs.append(o)
        if force or _stale(o, [s] + headers):
            cmd = [NVCC] + FLAGS + ["-c", s, "-o", o]
            procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode != 0:
            sys.stderr.write("== %s ==\n%s\n" % (src, out))
        else:
            with open(os.path.join(LIBDIR, src + ".ptxas.log"), "w") as f:
                f.write(out)
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed")
    if force or procs or _stale(SO, objs):
        subprocess.check_call([NVCC, "-shared", "-o", SO] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-ldl"])
    build_host(force)
    return SO


HOST = os.path.join(ROOT, "host")
HOST_SO = os.path.join(LIBDIR, "libmlease_host.so")
HOST_CLI = os.path.join(LIBDIR, "mlease_regression")


def build_host(force: bool = False) -> str:
    """Host job layer (C++17, zlib): libmlease_host.so + the mlease_regression CLI, both linked to libmlease_b200.so."""
    srcs = [os.path.join(HOST, f) for f in ("avro_io.cpp", "regression_jobs.cpp", "item_model_jobs.cpp", "item_model_train_job.cpp",
                                                 "item_model_grid_test_job.cpp", "regression_posterior_job.cpp", "auc_jobs.cpp")]
    deps = srcs + [os.path.join(HOST, "avro_io.hpp"), os.path.join(HOST, "avro_walk.hpp"), os.path.join(HOST, "jobs_common.hpp"), os.path.join(os.path.dirname(ROOT), "include", "mlease_b200.h"),
                   os.path.join(os.path.dirname(ROOT), "include", "mlease_host.h"), SO]
    cxx = os.environ.get("CXX", "g++")
    common = ["-O2", "-std=c++17", "-fPIC", "-Wall", "-Wno-unused-function"]
    link = ["-L" + LIBDIR, "-lmlease_b200", "-lz", "-pthread", "-Wl,-rpath,$ORIGIN"]
    if force or _stale(HOST_SO, deps):
        subprocess.check_call([cxx] + common + ["-shared", "-o", HOST_SO] + srcs + link)
    main = os.path.join(HOST, "mlease_regression_main.cpp")
    if force or _stale(HOST_CLI, [main, HOST_SO]):
        subprocess.check_call([cxx] + common + ["-o", HOST_CLI, main, "-L" + LIBDIR, "-lmlease_host", "-lmlease_b200", "-lz", "-pthread", "-Wl,-rpath,$ORIGIN"])
    return HOST_SO


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
