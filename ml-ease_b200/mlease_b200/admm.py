"""Host-side mirror of the reference's ADMM train job for the accelerated path.

`AdmmSession` wraps the C ABI session = the body of RegressionAdmmTrain.run()
(jobs/RegressionAdmmTrain.java:278-501): partitions are uploaded once
(replacing AdmmReducer's per-iteration dataset rebuild, :677-690), `local_step` is the
reducer phase (:642-718) for all resident (partition, lambda) pairs, `consensus` is the
driver's z/u update (:362-404, :736-765).  Config keys keep the reference's names
(with '.' -> '_').
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._native import ALLREDUCE_FN, AdmmConfigC, MleaseError, StatsC, check, lib, ptr
# The test hooks' wrappers and layouts live in _hooks; code written against their former names here keeps working.
from ._hooks import (BFGS_M, CONSENSUS_CTRL, CONSENSUS_FVECS, CONSENSUS_INFO, CONSENSUS_STAGES, CONSENSUS_VECS, K1_KINDS,  # noqa: F401
                     STAGE_CTRL, STAGE_INTS, STAGE_REALS, STAGE_VECS, STAGES)
from ._hooks import batch_factor as _internal_batch_factor, batch_grad as _internal_batch_grad  # noqa: F401
from ._hooks import consensus as _internal_consensus, direction as _internal_direction  # noqa: F401
from ._hooks import keyed_last_call as _internal_keyed_last_call, set_keyed_budget as _internal_set_keyed_budget  # noqa: F401
from ._hooks import newton_stage as _internal_newton_stage, xupdate_trace as _internal_xupdate_trace  # noqa: F401


def _f32(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float32)


def _keep(a, dtype):
    """numpy/torch passthrough with dtype/contiguity enforcement; returns (object_to_keep_alive)."""
    if a is None:
        return None
    if hasattr(a, "data_ptr"):  # torch tensor
        import torch
        td = {np.float32: torch.float32, np.int32: torch.int32, np.int64: torch.int64, np.float64: torch.float64}[dtype]
        if a.dtype != td or not a.is_contiguous():
            a = a.to(td).contiguous()
        return a
    return np.ascontiguousarray(a, dtype=dtype)


class Comm:
    """One rank of the library's NCCL communicator (include/mlease_b200.h "Multi-GPU" (a)): rank 0 makes the id with
    Comm.unique_id(), ships the 128 bytes to the other processes (any transport), every rank builds Comm(id, rank, nranks, device)
    and attaches it to its AdmmSession with set_comm(); session.run(iters) then runs the whole loop in C with one
    ncclAllReduce per iteration."""

    def __init__(self, unique_id: bytes, rank: int, nranks: int, device: int = 0):
        self._h = None
        buf = (C.c_char * 128).from_buffer_copy(bytes(unique_id))
        h = C.c_void_p()
        check(lib().mlease_comm_create(buf, int(rank), int(nranks), int(device), C.byref(h)))
        self._h, self.rank, self.nranks = h, int(rank), int(nranks)

    @staticmethod
    def unique_id() -> bytes:
        buf = (C.c_char * 128)()
        check(lib().mlease_comm_unique_id(buf))
        return bytes(buf.raw)

    def nccl_version(self):
        v = C.c_int32(0)
        check(lib().mlease_comm_info(self._h, None, None, C.byref(v)))
        return v.value

    def close(self):
        if self._h is not None:
            lib().mlease_comm_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class AdmmSession:
    def __init__(self, num_blocks, num_features, lambdas, rhos=None, *, device=0, stream=None, regularizer=2,
                 penalize_intercept=False, epsilon=1e-4, rho_adapt_coefficient=0.0, aggressive_liblinear_epsilon_decay=False,
                 binary_feature=False, lambda_map=None, newton_xtol=0.0, max_newton=0, hessian_policy=0):
        self._h = None
        self.num_blocks, self.num_features = int(num_blocks), int(num_features)
        self.lambdas = _f32(np.atleast_1d(lambdas))
        self.L = len(self.lambdas)
        self.Dt = self.num_features + 1
        self.device = int(device)
        self._rhos = _f32(rhos)
        self._lmap = _f32(lambda_map)
        cfg = AdmmConfigC()
        cfg.device, cfg.num_blocks, cfg.num_features, cfg.num_lambdas = self.device, self.num_blocks, self.num_features, self.L
        cfg.lambdas = self.lambdas.ctypes.data_as(C.POINTER(C.c_float))
        cfg.rhos = None if self._rhos is None else self._rhos.ctypes.data_as(C.POINTER(C.c_float))
        cfg.lambda_map = None if self._lmap is None else self._lmap.ctypes.data_as(C.POINTER(C.c_float))
        cfg.regularizer, cfg.penalize_intercept = int(regularizer), int(bool(penalize_intercept))
        cfg.aggressive_decay, cfg.binary_feature = int(bool(aggressive_liblinear_epsilon_decay)), int(bool(binary_feature))
        cfg.epsilon, cfg.rho_adapt_coefficient = float(epsilon), float(rho_adapt_coefficient)
        cfg.newton_xtol, cfg.max_newton, cfg.hessian_policy = float(newton_xtol), int(max_newton), int(hessian_policy)
        cfg.stream = stream
        h = C.c_void_p()
        check(lib().mlease_session_create(C.byref(cfg), C.byref(h)))
        self._h = h
        self._cb = None

    def close(self):
        if self._h is not None:
            lib().mlease_session_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def set_comm(self, comm):
        """Attach (or detach with None) the NCCL communicator of a multi-process job; the session then holds only its own
        partitions (p % nranks == rank) and run()/iterate() all-reduce inside the library."""
        self._comm = comm
        check(lib().mlease_session_set_comm(self._h, None if comm is None else comm._h))

    # ---- data ----
    def add_partition_dense(self, partition_id, X, response, weight=None, offset=None):
        X = _keep(X, np.float32)
        n, d = X.shape
        ld = X.stride(0) if hasattr(X, "data_ptr") else d
        r, w, o = _keep(response, np.int32), _keep(weight, np.float32), _keep(offset, np.float32)
        check(lib().mlease_add_partition_dense(self._h, int(partition_id), n, ptr(X), ld, ptr(r), ptr(w), ptr(o)))

    def add_partition_csr(self, partition_id, rowptr, colidx, vals, response, weight=None, offset=None):
        rp, ci, v = _keep(rowptr, np.int64), _keep(colidx, np.int32), _keep(vals, np.float32)
        r, w, o = _keep(response, np.int32), _keep(weight, np.float32), _keep(offset, np.float32)
        check(lib().mlease_add_partition_csr(self._h, int(partition_id), len(r), ptr(rp), ptr(ci), ptr(v), ptr(r), ptr(w), ptr(o)))

    # ---- ADMM ----
    def begin(self, z0=None, boost_rate=0.0):
        """Cold start (z = {}), or -- initialize.boost.rate > 0 -- from z0 [L][D+1] with the reducers' rho scaled by boost_rate
        (jobs/RegressionAdmmTrain.java:236-266, 313-316)."""
        if z0 is None:
            check(lib().mlease_admm_begin(self._h))
        else:
            z = np.ascontiguousarray(z0, np.float64).reshape(self.L, self.Dt)
            check(lib().mlease_admm_begin_initialized(self._h, ptr(z), C.c_float(boost_rate)))

    def mean_naive_model(self, partition_ids, penalize_intercept=False):
        """z0 of initialize.boost.rate for a single-process job: per (partition, lambda) the RegressionNaiveTrain fit (prior
        variance 1/lambda, intercept variance 100000 unless penalised, prior mean 0, start 0: jobs/RegressionNaiveTrain.java:333-343,395),
        written as float and averaged by MeanLinearModelConsumer (cons/MeanLinearModelConsumer.java:44-70).  Multi-process jobs
        sum the per-rank partial means with one all-reduce of this array."""
        z0 = np.zeros((self.L, self.Dt), np.float64)
        nb = float(self.num_blocks)
        for li, lam in enumerate(self.lambdas):
            q = np.full(self.Dt, float(lam), np.float64)
            if not penalize_intercept:
                q[-1] = 1.0 / 100000.0
            for pid in partition_ids:
                x, _ = self.fit_partition(pid, np.zeros(self.Dt), np.zeros(self.Dt), q)
                z0[li] = 1.0 * z0[li] + (1.0 / nb) * x.astype(np.float32).astype(np.float64)
        return z0

    def local_step(self, exchange_dev_ptr):
        check(lib().mlease_admm_local_step(self._h, ptr(exchange_dev_ptr)))

    def consensus(self, exchange_sum_dev_ptr):
        md, stop = C.c_double(0), C.c_int32(0)
        check(lib().mlease_admm_consensus(self._h, ptr(exchange_sum_dev_ptr), C.byref(md), C.byref(stop)))
        return md.value, bool(stop.value)

    def iterate(self):
        """One iteration of a single-process job: local_step + consensus on the session's own exchange buffer."""
        md, stop = C.c_double(0), C.c_int32(0)
        check(lib().mlease_admm_iterate(self._h, C.byref(md), C.byref(stop)))
        return md.value, bool(stop.value)

    def run(self, num_iters, allreduce=None):
        """Single-process job (allreduce None) or with a Python all-reduce callable(buf_ptr, count, stream_ptr)."""
        done = C.c_int32(0)
        cb = None
        if allreduce is not None:
            def _cb(ctx, buf, count, stream):
                try:
                    allreduce(buf, count, stream)
                    return 0
                except Exception:  # pragma: no cover
                    import traceback
                    traceback.print_exc()
                    return 1
            cb = ALLREDUCE_FN(_cb)
            self._cb = cb
        check(lib().mlease_admm_run(self._h, int(num_iters), C.cast(cb, C.c_void_p) if cb else None, None, C.byref(done)))
        return done.value

    # ---- state ----
    def z(self, lambda_idx=0):
        out = np.zeros(self.Dt, np.float64)
        check(lib().mlease_get_z(self._h, lambda_idx, ptr(out)))
        return out

    def final_model(self, lambda_idx=0):
        out = np.zeros(self.Dt, np.float32)
        check(lib().mlease_get_final_model(self._h, lambda_idx, ptr(out)))
        return out

    def x(self, partition_id, lambda_idx=0):
        out = np.zeros(self.Dt, np.float64)
        check(lib().mlease_get_x(self._h, partition_id, lambda_idx, ptr(out)))
        return out

    def u(self, partition_id, lambda_idx=0):
        out = np.zeros(self.Dt, np.float32)
        check(lib().mlease_get_u(self._h, partition_id, lambda_idx, ptr(out)))
        return out

    def uplusx(self, partition_id, lambda_idx=0):
        out = np.zeros(self.Dt, np.float32)
        check(lib().mlease_get_uplusx(self._h, partition_id, lambda_idx, ptr(out)))
        return out

    def stats(self):
        s = StatsC()
        check(lib().mlease_get_stats(self._h, C.byref(s)))
        return {k: getattr(s, k) for k, _ in StatsC._fields_}

    # ---- function-level entry points ----
    def objective(self, partition_id, w, prior_mean, prior_precision, want_grad=True, want_hessian=False, tensor=True):
        w, m, q = (np.ascontiguousarray(a, np.float64) for a in (w, prior_mean, prior_precision))
        f = C.c_double(0)
        g = np.zeros(self.Dt, np.float64) if want_grad else None
        H = np.zeros((self.Dt, self.Dt), np.float64) if want_hessian else None
        check(lib().mlease_objective(self._h, partition_id, ptr(w), ptr(m), ptr(q), C.byref(f), ptr(g), ptr(H), int(tensor)))
        return f.value, g, H

    def fit_partition(self, partition_id, init, prior_mean, prior_precision):
        x = np.array(init, np.float64, copy=True)
        m, q = (np.ascontiguousarray(a, np.float64) for a in (prior_mean, prior_precision))
        steps = C.c_int32(0)
        check(lib().mlease_fit_partition(self._h, partition_id, ptr(x), ptr(m), ptr(q), C.byref(steps)))
        return x, steps.value

    def hessian_vector(self, partition_id, w, prior_precision, v):
        """LogisticRegressionL2.Hv (llf/LogisticRegressionL2.java:231-248) at w with prior precision q: X^T D(w) X v + q * v,
        computed by the Hv mode of the CSR K1 kernels (fp32 products, fp64 fixed-order reductions: bitwise repeatable)."""
        w, q, v = (np.ascontiguousarray(a, np.float64) for a in (w, prior_precision, v))
        out = np.zeros(self.Dt, np.float64)
        check(lib().mlease_hessian_vector(self._h, int(partition_id), ptr(w), ptr(q), ptr(v), ptr(out)))
        return out

    def posterior_variance(self, partition_id, w, prior_precision, full=False, want_cov=False):
        """LibLinear.train's computePosteriorVar tail (llf/LibLinear.java:315-334): diagonal (1 / hessianDiagonal) or full
        (diag of the inverse of the exact fp64 Hessian; want_cov also returns H^-1)."""
        w, q = (np.ascontiguousarray(a, np.float64) for a in (w, prior_precision))
        var = np.zeros(self.Dt, np.float64)
        cov = np.zeros((self.Dt, self.Dt), np.float64) if (full and want_cov) else None
        check(lib().mlease_posterior_variance(self._h, int(partition_id), ptr(w), ptr(q), int(bool(full)), ptr(var), ptr(cov)))
        return (var, cov) if want_cov else var

    def admm_posterior(self, lambda_idx=0, z=None, full=False, want_cov=False):
        """Posterior of the ADMM model at z (default: the consensus z of lambda_idx) over all partitions (and all ranks of an attached
        communicator: collective then).  -> var [Dt], or (var, cov [Dt, Dt]) with want_cov (full only)."""
        zz = None if z is None else np.ascontiguousarray(z, np.float64)
        var = np.zeros(self.Dt, np.float64)
        cov = np.zeros((self.Dt, self.Dt), np.float64) if want_cov else None
        check(lib().mlease_admm_posterior(self._h, int(lambda_idx), ptr(zz), int(bool(full)), ptr(var), ptr(cov)))
        return (var, cov) if want_cov else var

    def profile(self, enable=-1):
        """Per-kernel CUDA-event timing accumulators; enable: 1 on, 0 off, 2 on+reset, -1 read only."""
        ms = np.zeros(4, np.float64); cnt = np.zeros(4, np.int64)
        kb, eb, gf = C.c_double(0), C.c_double(0), C.c_double(0)
        check(lib().mlease_profile(self._h, int(enable), ptr(ms), ptr(cnt), C.byref(kb), C.byref(eb), C.byref(gf)))
        names = ("k1", "small", "gram", "cholesky")
        return dict(ms=dict(zip(names, ms.tolist())), launches=dict(zip(names, cnt.tolist())), k1_bytes=kb.value,
                    k1_emit_bytes=eb.value, gram_flops=gf.value)

    def time_kernel(self, partition_id, which, reps=5, emit_scaled=False):
        ms = C.c_float(0)
        check(lib().mlease_time_kernel(self._h, partition_id, {"k1": 1, "gram": 2, "cholesky": 3, "hv": 4}[which], reps, int(emit_scaled), C.byref(ms)))
        return ms.value


class World:
    """N GPUs of THIS process behind the session calls (include/mlease_b200.h "Multi-GPU" (b)): partitions go to GPU
    partition_id % ndev, one worker thread per GPU inside the library, NCCL all-reduce per iteration."""

    def __init__(self, devices, num_blocks, num_features, lambdas, rhos=None, *, regularizer=2, penalize_intercept=False, epsilon=1e-4,
                 rho_adapt_coefficient=0.0, aggressive_liblinear_epsilon_decay=False, binary_feature=False, lambda_map=None,
                 newton_xtol=0.0, max_newton=0, hessian_policy=0):
        self._h = None
        self.lambdas = _f32(np.atleast_1d(lambdas))
        self.L, self.Dt, self.num_blocks = len(self.lambdas), int(num_features) + 1, int(num_blocks)
        self._rhos, self._lmap = _f32(rhos), _f32(lambda_map)
        cfg = AdmmConfigC()
        cfg.device, cfg.num_blocks, cfg.num_features, cfg.num_lambdas = 0, self.num_blocks, int(num_features), self.L
        cfg.lambdas = self.lambdas.ctypes.data_as(C.POINTER(C.c_float))
        cfg.rhos = None if self._rhos is None else self._rhos.ctypes.data_as(C.POINTER(C.c_float))
        cfg.lambda_map = None if self._lmap is None else self._lmap.ctypes.data_as(C.POINTER(C.c_float))
        cfg.regularizer, cfg.penalize_intercept = int(regularizer), int(bool(penalize_intercept))
        cfg.aggressive_decay, cfg.binary_feature = int(bool(aggressive_liblinear_epsilon_decay)), int(bool(binary_feature))
        cfg.epsilon, cfg.rho_adapt_coefficient = float(epsilon), float(rho_adapt_coefficient)
        cfg.newton_xtol, cfg.max_newton, cfg.hessian_policy = float(newton_xtol), int(max_newton), int(hessian_policy)
        cfg.stream = None
        devs = np.ascontiguousarray(devices, np.int32)
        h = C.c_void_p()
        check(lib().mlease_world_create(C.byref(cfg), ptr(devs), len(devs), C.byref(h)))
        self._h, self.ndev = h, len(devs)

    def close(self):
        if self._h is not None:
            lib().mlease_world_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def add_partition_dense(self, partition_id, X, response, weight=None, offset=None):
        X = _keep(X, np.float32)
        n, d = X.shape
        ld = X.stride(0) if hasattr(X, "data_ptr") else d
        r, w, o = _keep(response, np.int32), _keep(weight, np.float32), _keep(offset, np.float32)
        check(lib().mlease_world_add_partition_dense(self._h, int(partition_id), n, ptr(X), ld, ptr(r), ptr(w), ptr(o)))

    def add_partition_csr(self, partition_id, rowptr, colidx, vals, response, weight=None, offset=None):
        rp, ci, v = _keep(rowptr, np.int64), _keep(colidx, np.int32), _keep(vals, np.float32)
        r, w, o = _keep(response, np.int32), _keep(weight, np.float32), _keep(offset, np.float32)
        check(lib().mlease_world_add_partition_csr(self._h, int(partition_id), len(r), ptr(rp), ptr(ci), ptr(v), ptr(r), ptr(w), ptr(o)))

    def begin(self, z0=None, boost_rate=0.0):
        if z0 is None:
            check(lib().mlease_world_begin(self._h))
        else:
            z = np.ascontiguousarray(z0, np.float64).reshape(self.L, self.Dt)
            check(lib().mlease_world_begin_initialized(self._h, ptr(z), C.c_float(boost_rate)))

    def iterate(self):
        md, stop = C.c_double(0), C.c_int32(0)
        check(lib().mlease_world_iterate(self._h, C.byref(md), C.byref(stop)))
        return md.value, bool(stop.value)

    def run(self, num_iters):
        done = C.c_int32(0)
        check(lib().mlease_world_run(self._h, int(num_iters), C.byref(done)))
        return done.value

    def z(self, lambda_idx=0):
        out = np.zeros(self.Dt, np.float64)
        check(lib().mlease_world_get_z(self._h, lambda_idx, ptr(out)))
        return out

    def _vec(self, fn, pid, l, dtype):
        out = np.zeros(self.Dt, dtype)
        check(fn(self._h, int(pid), int(l), ptr(out)))
        return out

    def x(self, partition_id, lambda_idx=0):
        return self._vec(lib().mlease_world_get_x, partition_id, lambda_idx, np.float64)

    def u(self, partition_id, lambda_idx=0):
        return self._vec(lib().mlease_world_get_u, partition_id, lambda_idx, np.float32)

    def uplusx(self, partition_id, lambda_idx=0):
        return self._vec(lib().mlease_world_get_uplusx, partition_id, lambda_idx, np.float32)

    def admm_posterior(self, lambda_idx=0, z=None, full=False, want_cov=False):
        """AdmmSession.admm_posterior over every device of the world."""
        zz = None if z is None else np.ascontiguousarray(z, np.float64)
        var = np.zeros(self.Dt, np.float64)
        cov = np.zeros((self.Dt, self.Dt), np.float64) if want_cov else None
        check(lib().mlease_world_admm_posterior(self._h, int(lambda_idx), ptr(zz), int(bool(full)), ptr(var), ptr(cov)))
        return (var, cov) if want_cov else var

    def stats(self):
        s = StatsC()
        check(lib().mlease_world_get_stats(self._h, C.byref(s)))
        return {k: getattr(s, k) for k, _ in StatsC._fields_}


def score(vals, model, *, rowptr=None, colidx=None, offset=None, num_features=None, device=0, stream=None,
          num_click_replicates=1, binary_feature=False, out=None):
    """RegressionTest scoring (models/LinearModel.java:241-257; jobs/RegressionTest.java:163). Dense if colidx is None."""
    model = _keep(model, np.float64)
    Dg = int(num_features if num_features is not None else len(model) - 1)
    if colidx is None:
        vals = _keep(vals, np.float32)
        n, ld = vals.shape[0], (vals.stride(0) if hasattr(vals, "data_ptr") else vals.shape[1])
        rp = ci = None
    else:
        rp, ci, vals = _keep(rowptr, np.int64), _keep(colidx, np.int32), _keep(vals, np.float32)
        n, ld = len(rp) - 1, 0
    o = _keep(offset, np.float32)
    pred = np.zeros(n, np.float32) if out is None else out
    check(lib().mlease_score(device, stream, Dg, n, ptr(rp), ptr(ci), ptr(vals), ld, ptr(o), ptr(model), int(num_click_replicates),
                             int(binary_feature), ptr(pred)))
    return pred


def score_var(rowptr, colidx, vals, model, *, var=None, cov=None, offset=None, num_features=None, device=0, stream=None,
              num_click_replicates=1, binary_feature=False):
    """score's pred (bit for bit) and each record's predictive variance float(g^T Sigma g) under var (diagonal Sigma, [Dt]) or cov
    (dense [Dt, Dt]; exactly one of the two).  CSR rows only, strictly ascending columns.  -> (pred, pred_var) float32."""
    model = _keep(model, np.float64)
    Dg = int(num_features) if num_features is not None else len(model) - 1
    rp, ci, v = _keep(rowptr, np.int64), _keep(colidx, np.int32), _keep(vals, np.float32)
    n = len(rp) - 1
    o = None if offset is None else _keep(offset, np.float32)
    va, cv = _keep(var, np.float64), _keep(cov, np.float64)
    pred = np.zeros(n, np.float32)
    pvar = np.zeros(n, np.float32)
    check(lib().mlease_score_var(device, stream, Dg, n, ptr(rp), ptr(ci), ptr(v), ptr(o), ptr(model), int(num_click_replicates),
                                 int(bool(binary_feature)), ptr(va), ptr(cv), ptr(pred), ptr(pvar)))
    return pred, pvar


def test_loglik(response, pred, weight=None, combiner_block=0, device=0, stream=None):
    """RegressionTestLoglik (jobs/RegressionTestLoglik.java:124-200) -> (float32 avg loglik, count)."""
    r, p, w = _keep(response, np.int32), _keep(pred, np.float32), _keep(weight, np.float32)
    ll, cnt = C.c_float(0), C.c_double(0)
    check(lib().mlease_test_loglik(device, stream, len(r), ptr(r), ptr(p), ptr(w), int(combiner_block), C.byref(ll), C.byref(cnt)))
    return np.float32(ll.value), cnt.value


test_loglik.__test__ = False


def score_keyed(vals, key_rowstart, rowptr, colidx, num_features, model_ptr, model_col, model_val, *, offset=None,
                binary_feature=False, device=0, stream=None, out=None):
    """ItemModelTest scoring (jobs/ItemModelTest.java:181-211): row i of key k (rows [key_rowstart[k], key_rowstart[k+1]) of the
    CSR) is scored with model l*K + k for every lambda l.  Models are a CSR over (lambda, key): entries
    [model_ptr[m], model_ptr[m+1]) of model_col (ascending, num_features = intercept) / model_val.  -> pred [L, nrows] float32."""
    krs, rp, ci, vals = _keep(key_rowstart, np.int64), _keep(rowptr, np.int64), _keep(colidx, np.int32), _keep(vals, np.float32)
    mp, mc, mv = _keep(model_ptr, np.int64), _keep(model_col, np.int32), _keep(model_val, np.float32)
    K = len(krs) - 1
    if K <= 0 or (len(mp) - 1) % K:
        raise ValueError("model_ptr must hold num_lambdas * num_keys + 1 entries")
    L = (len(mp) - 1) // K
    n = len(rp) - 1
    o = _keep(offset, np.float32)
    pred = np.zeros((L, n), np.float32) if out is None else out
    check(lib().mlease_score_keyed(device, stream, int(num_features), K, ptr(krs), ptr(rp), ptr(ci), ptr(vals), ptr(o), L, ptr(mp),
                                   ptr(mc), ptr(mv), int(bool(binary_feature)), ptr(pred)))
    return pred


def score_keyed_var(vals, key_rowstart, rowptr, colidx, num_features, model_ptr, model_col, model_val, var_ptr, var_col, var_val,
                    var_default, *, offset=None, binary_feature=False, device=0, stream=None, out=None, out_var=None):
    """score_keyed with each record's predictive variance under the diagonal posterior of its model (ItemModelTrain, compute.var).
    Rows must list strictly ascending columns.  Variance lists are a CSR over (grid point, key) like the models: entries
    [var_ptr[m], var_ptr[m+1]) of var_col (ascending, num_features = intercept) / var_val; var_default[m] for every unlisted
    column.  -> (pred [G, nrows] float32, pred_var [G, nrows] float32); an empty variance list gives NaN."""
    krs, rp, ci, vals = _keep(key_rowstart, np.int64), _keep(rowptr, np.int64), _keep(colidx, np.int32), _keep(vals, np.float32)
    mp, mc, mv = _keep(model_ptr, np.int64), _keep(model_col, np.int32), _keep(model_val, np.float32)
    vp, vc, vv, vd = _keep(var_ptr, np.int64), _keep(var_col, np.int32), _keep(var_val, np.float32), _keep(var_default, np.float32)
    K = len(krs) - 1
    if K <= 0 or (len(mp) - 1) % K or len(vp) != len(mp) or len(vd) != len(mp) - 1:
        raise ValueError("model_ptr and var_ptr must hold G * num_keys + 1 entries, var_default G * num_keys")
    G = (len(mp) - 1) // K
    n = len(rp) - 1
    o = _keep(offset, np.float32)
    pred = np.zeros((G, n), np.float32) if out is None else out
    pred_var = np.zeros((G, n), np.float32) if out_var is None else out_var
    check(lib().mlease_score_keyed_var(device, stream, int(num_features), K, ptr(krs), ptr(rp), ptr(ci), ptr(vals), ptr(o), G, ptr(mp),
                                       ptr(mc), ptr(mv), ptr(vp), ptr(vc), ptr(vv), ptr(vd), int(bool(binary_feature)), ptr(pred),
                                       ptr(pred_var)))
    return pred, pred_var


def score_keyed_cov(vals, key_rowstart, rowptr, colidx, num_features, model_ptr, model_col, model_val, cov_ptr, cov_val, var_default, *,
                    lambda_map=None, offset=None, binary_feature=False, device=0, stream=None, out=None, out_var=None):
    """score_keyed with each record's predictive variance under the full posterior of its model (mlease_score_keyed_cov): model m's
    covariance is cov_val[cov_ptr[m]:cov_ptr[m+1]], the packed lower triangle of Sigma over its model_col list (keyed_cov_for_scoring
    orders item_model_train_cov's blocks so), or empty (NaN pred_var).  Unlisted columns: 1 / lambda_map[c] where > 0, else
    var_default[m].  Rows must list strictly ascending columns.  -> (pred [G, nrows] float32, pred_var [G, nrows] float32)."""
    krs, rp, ci, vals = _keep(key_rowstart, np.int64), _keep(rowptr, np.int64), _keep(colidx, np.int32), _keep(vals, np.float32)
    mp, mc, mv = _keep(model_ptr, np.int64), _keep(model_col, np.int32), _keep(model_val, np.float32)
    cp, cv, vd, lm = _keep(cov_ptr, np.int64), _keep(cov_val, np.float64), _keep(var_default, np.float32), _keep(lambda_map, np.float32)
    K = len(krs) - 1
    if K <= 0 or (len(mp) - 1) % K or len(cp) != len(mp) or len(vd) != len(mp) - 1:
        raise ValueError("model_ptr and cov_ptr must hold G * num_keys + 1 entries, var_default G * num_keys")
    G = (len(mp) - 1) // K
    n = len(rp) - 1
    o = _keep(offset, np.float32)
    pred = np.zeros((G, n), np.float32) if out is None else out
    pred_var = np.zeros((G, n), np.float32) if out_var is None else out_var
    check(lib().mlease_score_keyed_cov(device, stream, int(num_features), K, ptr(krs), ptr(rp), ptr(ci), ptr(vals), ptr(o), G, ptr(mp),
                                       ptr(mc), ptr(mv), ptr(cp), ptr(cv), ptr(lm), ptr(vd), int(bool(binary_feature)), ptr(pred),
                                       ptr(pred_var)))
    return pred, pred_var


def test_loglik_keyed(entry_key, entry_group, response, pred, num_keys, weight=None, device=0, stream=None):
    """ItemModelTestLoglik (jobs/ItemModelTestLoglik.java:60-142): one entry per (record, pred-map key), combiner group per entry
    (non-decreasing) -> (float32 loglik [num_keys], float64 count [num_keys])."""
    k, g, r = _keep(entry_key, np.int32), _keep(entry_group, np.int32), _keep(response, np.int32)
    p, w = _keep(pred, np.float32), _keep(weight, np.float32)
    ll = np.zeros(int(num_keys), np.float32)
    cnt = np.zeros(int(num_keys), np.float64)
    check(lib().mlease_test_loglik_keyed(device, stream, len(r), ptr(k), ptr(g), ptr(r), ptr(w), ptr(p), int(num_keys), ptr(ll), ptr(cnt)))
    return ll, cnt


test_loglik_keyed.__test__ = False


def test_auc(response, pred, weight=None, key_rowstart=None, device=0, stream=None):
    """Weighted ROC AUC (Mann-Whitney U, ties 1/2) of pred [S, n] (1-D: S = 1) against response (1 positive; 0, -1 negative) ->
    (auc [S], weight [2] = positive and negative weight of all rows, key_auc [S, K] or None, key_weight [K, 2] or None); keys own
    rows [key_rowstart[k], key_rowstart[k+1]).  pred, response and weight may be CUDA tensors."""
    p = _keep(pred, np.float32)
    S = 1 if len(p.shape) == 1 else int(p.shape[0])
    n = int(p.shape[-1])
    r, w = _keep(response, np.int32), _keep(weight, np.float32)
    krs = None if key_rowstart is None else np.ascontiguousarray(key_rowstart, np.int64)
    K = 0 if krs is None else len(krs) - 1
    auc = np.zeros(S, np.float64)
    wt = np.zeros(2, np.float64)
    kauc = np.zeros((S, K), np.float64) if krs is not None else None
    kw = np.zeros((K, 2), np.float64) if krs is not None else None
    check(lib().mlease_test_auc(device, stream, n, S, ptr(p), ptr(r), ptr(w), K, ptr(krs), ptr(auc), ptr(wt), ptr(kauc), ptr(kw)))
    return auc, wt, kauc, kw


test_auc.__test__ = False


def naive_train_dense(X, key_rowstart, response, lam, weight=None, offset=None, lambda_map=None, prior_mean=0.0,
                      penalize_intercept=False, has_intercept=True, data_size_threshold=0, device=0, stream=None):
    """RegressionNaiveTrain reducer for K keys (jobs/RegressionNaiveTrain.java:302-415) -> (models [K,D+1], skipped[K])."""
    X = _keep(X, np.float32)
    krs = np.ascontiguousarray(key_rowstart, np.int64)
    K, D = len(krs) - 1, X.shape[1]
    ld = X.stride(0) if hasattr(X, "data_ptr") else D
    r, w, o, lm = _keep(response, np.int32), _keep(weight, np.float32), _keep(offset, np.float32), _keep(lambda_map, np.float32)
    out = np.zeros((K, D + 1), np.float64)
    skipped = np.zeros(K, np.int32)
    check(lib().mlease_naive_train_dense(device, stream, K, D, ptr(krs), ptr(X), ld, ptr(r), ptr(w), ptr(o), float(lam), ptr(lm),
                                         float(prior_mean), int(penalize_intercept), int(has_intercept), int(data_size_threshold),
                                         ptr(out), ptr(skipped)))
    return out, skipped.astype(bool)


def naive_train(vals, key_rowstart, response, lambdas, *, rowptr=None, colidx=None, num_features=None, weight=None, offset=None,
                lambda_map=None, prior_mean=0.0, penalize_intercept=False, has_intercept=True, data_size_threshold=0,
                binary_feature=False, device=0, stream=None):
    """RegressionNaiveTrain reducers for K keys x L lambdas on one upload (jobs/RegressionNaiveTrain.java:228-241, 302-415).
    CSR when rowptr/colidx are given (vals = stored values), dense otherwise (vals = X [rows, D]).
    -> (models [L, K, D+1] float64, skipped [K] bool)."""
    krs = np.ascontiguousarray(key_rowstart, np.int64)
    K = len(krs) - 1
    lam = _f32(np.atleast_1d(lambdas))
    L = len(lam)
    if colidx is None:
        vals = _keep(vals, np.float32)
        D = vals.shape[1]
        ld = vals.stride(0) if hasattr(vals, "data_ptr") else D
        rp = ci = None
    else:
        rp, ci, vals = _keep(rowptr, np.int64), _keep(colidx, np.int32), _keep(vals, np.float32)
        D, ld = int(num_features), 0
    r, w, o, lm = _keep(response, np.int32), _keep(weight, np.float32), _keep(offset, np.float32), _keep(lambda_map, np.float32)
    out = np.zeros((L, K, D + 1), np.float64)
    skipped = np.zeros(K, np.int32)
    check(lib().mlease_naive_train(device, stream, K, D, ptr(krs), ptr(rp), ptr(ci), ptr(vals), ld, ptr(r), ptr(w), ptr(o), L, ptr(lam), ptr(lm),
                                   float(prior_mean), int(penalize_intercept), int(has_intercept), int(data_size_threshold),
                                   int(bool(binary_feature)), ptr(out), ptr(skipped)))
    return out, skipped.astype(bool)


def item_model_train(vals, key_rowstart, response, intercept_lambdas, default_lambdas, *, rowptr, colidx, num_features,
                     intercept_prior_mean=None, weight=None, offset=None, lambda_map=None, binary_feature=False, compute_var=False,
                     device=0, stream=None):
    """ItemModelTrain reducers (jobs/ItemModelTrain.java:226-276) for K keys on one CSR upload: one fit per (intercept lambda, default
    lambda), in list order.  intercept_prior_mean [K] float64 (None = 0).
    -> (models [IL, DL, K, D+1] float64, posterior variance of the same shape or None)."""
    krs = np.ascontiguousarray(key_rowstart, np.int64)
    K, D = len(krs) - 1, int(num_features)
    il, dl = _f32(np.atleast_1d(intercept_lambdas)), _f32(np.atleast_1d(default_lambdas))
    rp, ci, vals = _keep(rowptr, np.int64), _keep(colidx, np.int32), _keep(vals, np.float32)
    r, w, o, lm = _keep(response, np.int32), _keep(weight, np.float32), _keep(offset, np.float32), _keep(lambda_map, np.float32)
    im = np.zeros(K, np.float64) if intercept_prior_mean is None else np.ascontiguousarray(intercept_prior_mean, np.float64)
    if len(im) != K:
        raise ValueError("intercept_prior_mean must hold one entry per key")
    out = np.zeros((len(il), len(dl), K, D + 1), np.float64)
    var = np.zeros_like(out) if compute_var else None
    check(lib().mlease_item_model_train(device, stream, K, D, ptr(krs), ptr(rp), ptr(ci), ptr(vals), ptr(r), ptr(w), ptr(o), ptr(im),
                                        len(il), ptr(il), len(dl), ptr(dl), ptr(lm), int(bool(binary_feature)), int(bool(compute_var)),
                                        ptr(out), ptr(var)))
    return out, var


def _host(a, dtype):
    """numpy copy of a host array or torch tensor (any device)"""
    if hasattr(a, "data_ptr"):
        a = a.detach().cpu().numpy()
    return np.ascontiguousarray(a, dtype=dtype)


def _list_capacity(key_rowstart, rowptr, num_features, fitted, intercept):
    """entries the keys' lists may need: sum over fitted keys of min(stored entries, num_features) (+ 1 for the intercept), from
    rowptr at the key boundaries alone"""
    krs = _host(key_rowstart, np.int64)
    if hasattr(rowptr, "data_ptr"):
        import torch
        at = _host(rowptr[torch.as_tensor(krs, device=rowptr.device)], np.int64)
    else:
        at = np.asarray(rowptr, np.int64)[krs]
    nnz = np.diff(at)
    return int((np.minimum(nnz, int(num_features))[fitted] + (1 if intercept else 0)).sum())


def naive_train_sparse(vals, key_rowstart, response, lambdas, *, rowptr, colidx, num_features, weight=None, offset=None, lambda_map=None,
                       prior_mean=0.0, penalize_intercept=False, has_intercept=True, data_size_threshold=0, binary_feature=False, device=0,
                       stream=None, capacity=None):
    """naive_train on CSR keys with each key's model returned as the columns its rows list (mlease_naive_train_sparse): key k's list
    is cols[key_ptr[k]:key_ptr[k+1]] (ascending, then num_features for the intercept when has_intercept), its values for lambda l
    models[l, key_ptr[k]:key_ptr[k+1]], the dense call's fit at those columns; an unlisted feature's coefficient is 0.  Skipped
    keys and keys without rows have empty lists.  capacity (None: the bound from rowptr at the key boundaries) is the room allocated.
    -> (key_ptr [K+1] int64, cols [n] int32, models [L, n] float64, skipped [K] bool)."""
    krs = np.ascontiguousarray(key_rowstart, np.int64)
    K, D = len(krs) - 1, int(num_features)
    lam = _f32(np.atleast_1d(lambdas))
    L = len(lam)
    rp, ci, vals = _keep(rowptr, np.int64), _keep(colidx, np.int32), _keep(vals, np.float32)
    r, w, o, lm = _keep(response, np.int32), _keep(weight, np.float32), _keep(offset, np.float32), _keep(lambda_map, np.float32)
    rows = np.diff(krs)
    cap = _list_capacity(krs, rp, D, (rows > 0) & (rows >= int(data_size_threshold)), has_intercept) if capacity is None else int(capacity)
    key_ptr = np.zeros(K + 1, np.int64)
    cols = np.zeros(max(cap, 1), np.int32)
    models = np.zeros((L, max(cap, 1)), np.float64)
    skipped = np.zeros(K, np.int32)
    check(lib().mlease_naive_train_sparse(device, stream, K, D, ptr(krs), ptr(rp), ptr(ci), ptr(vals), ptr(r), ptr(w), ptr(o), L, ptr(lam),
                                          ptr(lm), float(prior_mean), int(penalize_intercept), int(has_intercept), int(data_size_threshold),
                                          int(bool(binary_feature)), cap, ptr(key_ptr), ptr(cols), ptr(models), ptr(skipped)))
    n = int(key_ptr[K])
    return key_ptr, cols[:n].copy(), models[:, :n].copy(), skipped.astype(bool)


def item_model_train_sparse(vals, key_rowstart, response, intercept_lambdas, default_lambdas, *, rowptr, colidx, num_features,
                            intercept_prior_mean=None, weight=None, offset=None, lambda_map=None, binary_feature=False, compute_var=False,
                            device=0, stream=None, capacity=None):
    """item_model_train with each key's model (and posterior variance) returned as the columns its rows list, then the intercept
    (mlease_item_model_train_sparse); values the dense call's fit at those columns, an unlisted feature's coefficient 0 and
    variance 1/q.  -> (key_ptr [K+1] int64, cols [n] int32, models [IL, DL, n] float64, var [IL, DL, n] float64 or None)."""
    krs = np.ascontiguousarray(key_rowstart, np.int64)
    K, D = len(krs) - 1, int(num_features)
    il, dl = _f32(np.atleast_1d(intercept_lambdas)), _f32(np.atleast_1d(default_lambdas))
    rp, ci, vals = _keep(rowptr, np.int64), _keep(colidx, np.int32), _keep(vals, np.float32)
    r, w, o, lm = _keep(response, np.int32), _keep(weight, np.float32), _keep(offset, np.float32), _keep(lambda_map, np.float32)
    im = np.zeros(K, np.float64) if intercept_prior_mean is None else np.ascontiguousarray(intercept_prior_mean, np.float64)
    if len(im) != K:
        raise ValueError("intercept_prior_mean must hold one entry per key")
    cap = _list_capacity(krs, rp, D, np.diff(krs) > 0, True) if capacity is None else int(capacity)
    G = len(il) * len(dl)
    key_ptr = np.zeros(K + 1, np.int64)
    cols = np.zeros(max(cap, 1), np.int32)
    models = np.zeros((G, max(cap, 1)), np.float64)
    var = np.zeros_like(models) if compute_var else None
    check(lib().mlease_item_model_train_sparse(device, stream, K, D, ptr(krs), ptr(rp), ptr(ci), ptr(vals), ptr(r), ptr(w), ptr(o), ptr(im),
                                               len(il), ptr(il), len(dl), ptr(dl), ptr(lm), int(bool(binary_feature)), int(bool(compute_var)),
                                               cap, ptr(key_ptr), ptr(cols), ptr(models), ptr(var)))
    n = int(key_ptr[K])
    shape = (len(il), len(dl), n)
    return (key_ptr, cols[:n].copy(), models[:, :n].reshape(shape).copy(),
            None if var is None else var[:, :n].reshape(shape).copy())


def _list_lengths(key_rowstart, rowptr, colidx, num_features):
    """each key's list length on the host: its distinct columns + 1 for the intercept, 0 for a key without rows"""
    krs, rp, ci = _host(key_rowstart, np.int64), _host(rowptr, np.int64), _host(colidx, np.int64)
    K = len(krs) - 1
    rows = np.diff(krs)
    row_key = np.repeat(np.arange(K, dtype=np.int64), rows)
    entry_key = np.repeat(row_key, np.diff(rp[krs[0]:krs[-1] + 1]))
    pairs = np.unique(entry_key * (int(num_features) + 1) + ci[rp[krs[0]]:rp[krs[-1]]])
    distinct = np.bincount(pairs // (int(num_features) + 1), minlength=K)
    return np.where(rows > 0, distinct + 1, 0).astype(np.int64)


def item_model_train_cov(vals, key_rowstart, response, intercept_lambdas, default_lambdas, *, rowptr, colidx, num_features,
                         intercept_prior_mean=None, weight=None, offset=None, lambda_map=None, binary_feature=False, want_cov=True,
                         device=0, stream=None, capacity=None, cov_capacity=None):
    """item_model_train_sparse with the full posterior of every fit (mlease_item_model_train_cov): var is diag(Sigma), Sigma the
    inverse of the key's exact Hessian at its fit, over its list; key k's covariance block is cov[..., cov_ptr[k]:cov_ptr[k+1]], the
    lower triangle of Sigma over the list's order, row-major (entry (a, b), a >= b, at cov_ptr[k] + a(a+1)/2 + b).  Rows must list
    strictly ascending columns.  The blocks are allocated at their exact sizes, from each key's distinct columns (cov_capacity
    overrides that).  want_cov = False: the variances only (cov_ptr and cov None).
    -> (key_ptr [K+1] int64, cols [n] int32, models [IL, DL, n], var [IL, DL, n], cov_ptr [K+1] int64, cov [IL, DL, m] float64)."""
    krs = np.ascontiguousarray(key_rowstart, np.int64)
    K, D = len(krs) - 1, int(num_features)
    il, dl = _f32(np.atleast_1d(intercept_lambdas)), _f32(np.atleast_1d(default_lambdas))
    rp, ci, vals = _keep(rowptr, np.int64), _keep(colidx, np.int32), _keep(vals, np.float32)
    r, w, o, lm = _keep(response, np.int32), _keep(weight, np.float32), _keep(offset, np.float32), _keep(lambda_map, np.float32)
    im = np.zeros(K, np.float64) if intercept_prior_mean is None else np.ascontiguousarray(intercept_prior_mean, np.float64)
    if len(im) != K:
        raise ValueError("intercept_prior_mean must hold one entry per key")
    cap = _list_capacity(krs, rp, D, np.diff(krs) > 0, True) if capacity is None else int(capacity)
    if want_cov and cov_capacity is None:
        n_k = _list_lengths(krs, rp, ci, D)
        cov_capacity = int((n_k * (n_k + 1) // 2).sum())
    ccap = int(cov_capacity) if want_cov else 0
    G = len(il) * len(dl)
    key_ptr = np.zeros(K + 1, np.int64)
    cols = np.zeros(max(cap, 1), np.int32)
    models = np.zeros((G, max(cap, 1)), np.float64)
    var = np.zeros_like(models)
    cov_ptr = np.zeros(K + 1, np.int64) if want_cov else None
    cov = np.zeros((G, max(ccap, 1)), np.float64) if want_cov else None
    check(lib().mlease_item_model_train_cov(device, stream, K, D, ptr(krs), ptr(rp), ptr(ci), ptr(vals), ptr(r), ptr(w), ptr(o), ptr(im),
                                            len(il), ptr(il), len(dl), ptr(dl), ptr(lm), int(bool(binary_feature)), cap, ptr(key_ptr),
                                            ptr(cols), ptr(models), ptr(var), ccap, ptr(cov_ptr), ptr(cov)))
    n = int(key_ptr[K])
    shape = (len(il), len(dl), n)
    out = (key_ptr, cols[:n].copy(), models[:, :n].reshape(shape).copy(), var[:, :n].reshape(shape).copy())
    if not want_cov:
        return out + (None, None)
    m = int(cov_ptr[K])
    cov = cov.reshape((len(il), len(dl), -1))   # a view; the blocks can be gigabytes, so trim by copying only when over-allocated
    return out + (cov_ptr, cov if cov.shape[-1] == m else cov[..., :m].copy())


def keyed_cov_for_scoring(key_ptr, cov_ptr, cov):
    """item_model_train_cov's blocks in the (prior, key) order score_keyed_cov takes them, the order keyed_models_for_scoring gives
    the models: model m = p * K + k is key k's block with prior p's values (cov [..., m_total], the priors flattened in order).
    -> (cov_ptr [P*K+1] int64, cov_val float64)."""
    cp = np.ascontiguousarray(cov_ptr, np.int64)
    m = int(cp[-1])
    cov = np.asarray(cov, np.float64)
    P = int(np.prod(cov.shape[:-1]))
    ptrs = np.concatenate([[0], (cp[1:][None, :] + m * np.arange(P, dtype=np.int64)[:, None]).reshape(-1)]).astype(np.int64)
    return ptrs, np.ascontiguousarray(cov.reshape(P, m)).reshape(-1)


def keyed_models_for_scoring(key_ptr, cols, models):
    """The sparse fits' lists as score_keyed's models: model m = p * K + k (prior p, key k) is key k's list with prior p's values
    (models [..., n], the priors flattened in order).  -> (model_ptr [P*K+1] int64, model_col int32, model_val float32)."""
    kp = np.ascontiguousarray(key_ptr, np.int64)
    n = int(kp[-1])
    models = np.asarray(models, np.float64)
    P = int(np.prod(models.shape[:-1]))
    vals = models.reshape(P, n)
    model_ptr = np.concatenate([[0], (kp[1:][None, :] + n * np.arange(P, dtype=np.int64)[:, None]).reshape(-1)]).astype(np.int64)
    return model_ptr, np.tile(np.ascontiguousarray(cols, np.int32)[:n], P), vals.astype(np.float32).reshape(-1)
