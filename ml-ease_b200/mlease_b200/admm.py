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


def _internal_set_keyed_budget(nbytes):
    """Test hook (not part of the C ABI): caps, process-wide, the device bytes the keyed calls plan with (0 = free memory only),
    so that small inputs stream through many chunks."""
    fn = lib().mlease_internal_set_keyed_budget
    fn.argtypes, fn.restype = [C.c_int64], C.c_int
    check(fn(int(nbytes)))


K1_KINDS = {1: "dense", 2: "fx", 3: "fx_window", 4: "csr", 5: "fused"}


def _internal_batch_grad(session, w, active=None, rows=None, want_sd=False, want_xt=False):
    """Test hook (not part of the C ABI): one K1 gradient pass over the ADMM batch of `session` (after begin()), problem b =
    partition * L + lambda at float(w[b]) when active[b] (default: all).  rows: the row count of each partition (needed for
    want_sd / want_xt).  Consumes the batch's x-update state.
    -> dict(f [nprob], g [nprob, Dt] (data term, no prior; NaN for inactive problems), sd (list of [n] float32 or None),
    xt (list of [n, Dp] uint16 bf16 bits or None), kind, G (dense G / fused LP / beta in shared memory), dyn, grid, RT (dense rows
    per thread / fused segment rows / column window), nsl, chunks [nprob])."""
    nprob, Dt = session.num_blocks * session.L, session.Dt
    w = np.ascontiguousarray(w, np.float64).reshape(nprob, Dt)
    act = np.ones(nprob, np.int32) if active is None else np.ascontiguousarray(active, np.int32)
    if len(act) != nprob:
        raise ValueError("active must hold one entry per problem")
    Dp = ((Dt + 3) // 4 * 4 + 127) // 128 * 128
    n_b = [int(rows[b // session.L]) for b in range(nprob)] if (want_sd or want_xt) else None
    f = np.zeros(nprob, np.float64)
    g = np.zeros((nprob, Dt), np.float64)
    sd = np.zeros(sum(n_b), np.float32) if want_sd else None
    xt = np.zeros(sum(n_b) * Dp, np.uint16) if want_xt else None
    info = np.zeros(8 + nprob, np.int32)
    fn = lib().mlease_internal_batch_grad
    fn.argtypes, fn.restype = [C.c_void_p] * 8, C.c_int
    check(fn(session._h, act.ctypes.data, w.ctypes.data, f.ctypes.data, g.ctypes.data, ptr(sd), ptr(xt), info.ctypes.data))
    split = np.cumsum([0] + (n_b or []))
    return dict(f=f, g=g, sd=[sd[split[b]:split[b + 1]] for b in range(nprob)] if want_sd else None,
                xt=[xt[split[b] * Dp:split[b + 1] * Dp].reshape(-1, Dp) for b in range(nprob)] if want_xt else None,
                kind=K1_KINDS[int(info[0])], G=int(info[1]), dyn=int(info[2]), grid=int(info[3]), RT=int(info[4]), nsl=int(info[5]),
                chunks=info[8:].copy())


def _internal_batch_factor(session, mode, H=None, G=None, q=None, order=None, share=0, share_factor=False):
    """Test hook (not part of the C ABI): one factorisation of the ADMM batch of `session` (after begin(), ldh <= 2048) through
    the solver's rebuild code.  mode[b]: 0 = done (untouched), 1 = factorise H[b] (Dt x Dt fp64), 2 = factorise the fp32 Gram G[b]
    plus diag(q[b]) through chol_prep_kernel.  order: launch order (a permutation or subset of the problems; default: batch
    order).  share / share_factor: the cold start of a rebuild slot (see mlease_internal_batch_factor).  Consumes the batch's
    x-update state.  -> dict(L [nprob, Dt, Dt], Y, Hinv [nprob, ldh, ldh], Ldinv [nprob, ldh, 32],
    fail, done, hess_valid, tot_hess [nprob]); buffers no kernel wrote hold the all-ones NaN sentinel."""
    nprob, Dt = session.num_blocks * session.L, session.Dt
    ldh = (Dt + 31) // 32 * 32
    md = np.ascontiguousarray(mode, np.int32)
    if md.shape != (nprob,):
        raise ValueError("mode must hold one entry per problem")
    Hc = None if H is None else np.ascontiguousarray(H, np.float64).reshape(nprob, Dt, Dt)
    Gc = None if G is None else np.ascontiguousarray(G, np.float32).reshape(nprob, Dt, Dt)
    qc = None if q is None else np.ascontiguousarray(q, np.float64).reshape(nprob, Dt)
    oc = None if order is None else np.ascontiguousarray(order, np.int32)
    out = dict(L=np.empty((nprob, Dt, Dt)), Y=np.empty((nprob, ldh, ldh)), Hinv=np.empty((nprob, ldh, ldh)),
               Ldinv=np.empty((nprob, ldh, 32)))
    ctrl = np.zeros((nprob, 4), np.int32)
    fn = lib().mlease_internal_batch_factor
    vp = C.c_void_p
    fn.argtypes, fn.restype = [vp] * 6 + [C.c_int32] * 3 + [vp] * 5, C.c_int
    check(fn(session._h, md.ctypes.data, ptr(Hc), ptr(Gc), ptr(qc), ptr(oc), 0 if oc is None else len(oc), int(share),
             int(bool(share_factor)), out["L"].ctypes.data, out["Y"].ctypes.data, out["Hinv"].ctypes.data, out["Ldinv"].ctypes.data,
             ctrl.ctypes.data))
    out.update(fail=ctrl[:, 0].copy(), done=ctrl[:, 1].copy(), hess_valid=ctrl[:, 2].copy(), tot_hess=ctrl[:, 3].copy())
    return out


BFGS_M = 6   # secant pairs kept per problem (common.cuh)


def _internal_direction(session, active, g, S, Y, rho, count, h0, beta):
    """Test hook (not part of the C ABI): the quasi-Newton direction on the explicit inverse H^-1 (ldh <= 2048) of the active
    problems of the ADMM batch, through the kernels of a chord slot, after _internal_batch_factor.  Per problem: g [Dt] data-term
    gradient, S, Y [BFGS_M, Dt] secant ring (slot-major), rho [BFGS_M], count (bfgs_count), h0 (h0_scale), beta [Dt] point.
    Consumes the batch's x-update state.  -> dict(dir [nprob, Dt], phi0, dirnorm [nprob], beta_t [nprob, Dt]); NaN where inactive."""
    nprob, Dt = session.num_blocks * session.L, session.Dt
    act = np.ascontiguousarray(active, np.int32)
    g, beta = (np.ascontiguousarray(a, np.float64).reshape(nprob, Dt) for a in (g, beta))
    S, Y = (np.ascontiguousarray(a, np.float64).reshape(nprob, BFGS_M, Dt) for a in (S, Y))
    rho = np.ascontiguousarray(rho, np.float64).reshape(nprob, BFGS_M)
    cnt = np.ascontiguousarray(count, np.int32).reshape(nprob)
    h0 = np.ascontiguousarray(h0, np.float64).reshape(nprob)
    out = dict(dir=np.empty((nprob, Dt)), phi0=np.empty(nprob), dirnorm=np.empty(nprob), beta_t=np.empty((nprob, Dt)))
    fn = lib().mlease_internal_direction
    fn.argtypes, fn.restype = [C.c_void_p] * 13, C.c_int
    check(fn(session._h, act.ctypes.data, g.ctypes.data, S.ctypes.data, Y.ctypes.data, rho.ctypes.data, cnt.ctypes.data, h0.ctypes.data,
             beta.ctypes.data, out["dir"].ctypes.data, out["phi0"].ctypes.data, out["dirnorm"].ctypes.data, out["beta_t"].ctypes.data))
    return out


STAGE_INTS = ("done", "have_dir", "need_solve", "need_hess", "emit", "hess_valid", "fail", "newton_steps", "evals", "rejects",
              "hess_builds", "stall", "bfgs_count", "k1_chunks", "refresh_next", "skip_eval", "warm_used", "build_step", "max_newton",
              "hess_policy", "rebuild_is_expensive", "cg_active", "cg_iter", "pad_")
STAGE_REALS = ("h0_scale", "worst_ratio", "alpha", "phi0", "f_acc", "f_t", "gnorm", "gnorm_prev", "dirnorm", "dirnorm_prev", "xtol",
               "cg_rz", "cg_g2", "hv_vinf", "tot_evals", "tot_newton", "tot_rejects", "tot_hess")
STAGE_CTRL = np.dtype([(k, np.int32) for k in STAGE_INTS] + [(k, np.float64) for k in STAGE_REALS])   # StageCtrl of test_hooks.cu
STAGE_VECS = ("beta", "beta_t", "m", "q", "g_t", "g_acc", "dir", "cg_r", "cg_p", "cg_z", "cg_Hp", "cg_diag")
STAGES = dict(begin=1, decide=2, solve=4, finish=8, cg_begin=16, cg_init=32, cg_step=64, cg_poll=128)


def _internal_newton_stage(session, stages=(), ctrl=None, vec=None, ring=None, fvec=None, gpart=None, fpart=None, spec=0, begin_args=None):
    """Test hook (not part of the C ABI): inject an x-update state into every problem of the ADMM batch (after begin()), run the
    kernels named in `stages` (keys of STAGES) once through the solver's launchers, read the state back.  ctrl [nprob] STAGE_CTRL;
    vec [nprob, 12, ldx] (STAGE_VECS); ring [nprob, 2 BFGS_M ldx + 2 BFGS_M] (S, Y, rho, alpha); fvec [nprob, 3, ldx] float32
    (beta_tf, qf = hv_vf, tf); gpart [nprob, nct, ldx], fpart [nprob, nct] or None; begin_args (xtol, max_newton, policy,
    invalidate, expensive).  Without stages: info only.  Consumes the batch's x-update state.
    -> dict(info=dict(nprob, Dt, ldx, ldh, part_rows, fused, matrix_free, ysym, expensive, group_L), ctrl, vec, ring, fvec, cg_any)."""
    mask = 0
    for k in stages:
        mask |= STAGES[k]
    info = np.zeros(12, np.int32)
    cg_any = C.c_int32(-1)
    fn = lib().mlease_internal_newton_stage
    vp = C.c_void_p
    fn.argtypes, fn.restype = [vp, C.c_int32, C.c_int32] + [vp] * 7 + [C.c_int32, vp, C.POINTER(C.c_int32)], C.c_int
    out = {}
    nct = 0
    if mask:
        out["ctrl"] = np.array(ctrl, STAGE_CTRL, copy=True)
        out["vec"] = np.array(vec, np.float64, copy=True, order="C")
        out["ring"] = np.array(ring, np.float64, copy=True, order="C")
        out["fvec"] = np.array(fvec, np.float32, copy=True, order="C")
        gpart = None if gpart is None else np.ascontiguousarray(gpart, np.float64)
        fpart = None if fpart is None else np.ascontiguousarray(fpart, np.float64)
        nct = 0 if fpart is None else fpart.shape[1]
        begin_args = None if begin_args is None else np.ascontiguousarray(begin_args, np.float64)
    check(fn(session._h, mask, int(spec), ptr(begin_args) if mask else None, ptr(out.get("ctrl")), ptr(out.get("vec")),
             ptr(out.get("ring")), ptr(out.get("fvec")), ptr(gpart) if mask else None, ptr(fpart) if mask else None, nct,
             info.ctypes.data, C.byref(cg_any)))
    out["info"] = dict(zip(("nprob", "Dt", "ldx", "ldh", "part_rows", "fused", "matrix_free", "ysym", "expensive", "group_L"),
                           (int(x) for x in info)))
    out["cg_any"] = cg_any.value
    return out


def _internal_xupdate_trace(session, policy=0, invalidate=0, spec=(), max_slots=60, xtol=0.0, max_newton=0):
    """Test hook (not part of the C ABI): one real x-update of the ADMM batch, slot by slot through the solver's own slot code.
    spec: slot indices asked to run speculatively (policy 0 only, never slot 0).  xtol / max_newton 0: the session's.
    -> dict(nslots, spec [nslots], with_hess [nslots], ctrl [nslots + 1, nprob] STAGE_CTRL, vec [nslots + 1, nprob, 12, ldx],
    ring [nslots + 1, nprob, 2 BFGS_M ldx + 2 BFGS_M], fvec [nslots + 1, nprob, 3, ldx]); entry 0 is the state newton_begin left,
    entry i + 1 the state after slot i."""
    info = _internal_newton_stage(session)["info"]
    nprob, ldx = info["nprob"], info["ldx"]
    sp = np.zeros(max_slots, np.int32)
    for i in spec:
        if i < max_slots:
            sp[i] = 1
    ctrl = np.zeros((max_slots + 1, nprob), STAGE_CTRL)
    vec = np.zeros((max_slots + 1, nprob, 12, ldx))
    ring = np.zeros((max_slots + 1, nprob, 2 * BFGS_M * ldx + 2 * BFGS_M))
    fvec = np.zeros((max_slots + 1, nprob, 3, ldx), np.float32)
    sinfo = np.zeros((max_slots, 2), np.int32)
    n = C.c_int32(0)
    args = np.array([xtol, max_newton, policy, invalidate], np.float64)
    fn = lib().mlease_internal_xupdate_trace
    vp = C.c_void_p
    fn.argtypes, fn.restype = [vp, vp, vp, C.c_int32, vp, vp, vp, vp, vp, C.POINTER(C.c_int32)], C.c_int
    check(fn(session._h, args.ctypes.data, sp.ctypes.data, int(max_slots), ctrl.ctypes.data, vec.ctypes.data, ring.ctypes.data,
             fvec.ctypes.data, sinfo.ctypes.data, C.byref(n)))
    k = n.value
    return dict(nslots=k, spec=sinfo[:k, 0].copy(), with_hess=sinfo[:k, 1].copy(), ctrl=ctrl[:k + 1], vec=vec[:k + 1], ring=ring[:k + 1],
                fvec=fvec[:k + 1], info=info)


CONSENSUS_VECS = ("beta", "m", "q", "g_t", "x_d")
CONSENSUS_FVECS = ("u_f", "uplusx_f", "x_f")
CONSENSUS_CTRL = ("hess_valid", "skip_eval", "k1_chunks")
CONSENSUS_STAGES = dict(reset=1, init=2, pack=4, consensus=8)
CONSENSUS_INFO = ("nprob", "Dt", "ldx", "L", "P", "nlocal", "csr", "fused", "matrix_free", "regularizer", "k1_grid", "ctrl_bytes")


def _internal_consensus(session, stages=(), state=None, iter=1, liblinear_eps=0.01, read=True):
    """Test hook (not part of the C ABI): inject a K4 state into the begun ADMM batch, run the stages named in `stages` (keys of
    CONSENSUS_STAGES, run in the order reset, init, pack, consensus) through the solver's own code, read everything back.  state:
    dict(vec [nprob, 5, ldx] (CONSENSUS_VECS), fvec [nprob, 3, ldx] float32 (CONSENSUS_FVECS), z [L, ldx], exch [L Dt + 1],
    diff [L], ctrl [nprob, 3] int32 (CONSENSUS_CTRL)), whole vectors with their padding.  The consensus stage runs with the session's
    iteration counter at `iter` and its liblinear epsilon at `liblinear_eps`.  Without stages nothing is injected: the state is read
    (read=False: info only).  With stages the batch's x-update state is consumed: begin() again before iterating.
    -> dict(info, the state's keys after the last stage, ctrl_raw [2, nprob, ctrl_bytes] uint8 (before / after, the three ctrl
    fields zeroed), wz [L, ldx], l1thr [L] or None, rho [L], maxdiff, mindiff, stop)."""
    mask = stages if isinstance(stages, int) else 0   # (a raw mask: lets a test pass one the hook must refuse)
    for k in ([] if isinstance(stages, int) else stages):
        mask |= CONSENSUS_STAGES[k]
    info = np.zeros(12, np.int32)
    fn = lib().mlease_internal_consensus
    vp = C.c_void_p
    fn.argtypes, fn.restype = [vp, C.c_int32] + [vp] * 13, C.c_int
    check(fn(session._h, 0, None, None, None, None, None, None, None, None, None, None, None, None, info.ctypes.data))
    inf = dict(zip(CONSENSUS_INFO, (int(x) for x in info)))
    if not mask and not read:
        return dict(info=inf)
    nprob, L, Dt, ldx = inf["nprob"], inf["L"], inf["Dt"], inf["ldx"]
    if mask:
        out = dict(vec=np.array(state["vec"], np.float64, copy=True, order="C"), fvec=np.array(state["fvec"], np.float32, copy=True, order="C"),
                   z=np.array(state["z"], np.float64, copy=True, order="C"), exch=np.array(state["exch"], np.float64, copy=True, order="C"),
                   diff=np.array(state["diff"], np.float64, copy=True, order="C"), ctrl=np.array(state["ctrl"], np.int32, copy=True, order="C"))
        if out["vec"].shape != (nprob, 5, ldx) or out["fvec"].shape != (nprob, 3, ldx) or out["z"].shape != (L, ldx) or \
                out["exch"].shape != (L * Dt + 1,) or out["diff"].shape != (L,) or out["ctrl"].shape != (nprob, 3):
            raise ValueError("state arrays do not match the batch")
    else:
        out = dict(vec=np.zeros((nprob, 5, ldx)), fvec=np.zeros((nprob, 3, ldx), np.float32), z=np.zeros((L, ldx)),
                   exch=np.zeros(L * Dt + 1), diff=np.zeros(L), ctrl=np.zeros((nprob, 3), np.int32))
    out.update(ctrl_raw=np.zeros((2, nprob, inf["ctrl_bytes"]), np.uint8), wz=np.zeros((L, ldx)),
               l1thr=np.zeros(L) if inf["regularizer"] == 1 else None, rho=np.zeros(L))
    res = np.zeros(3)
    args = np.array([iter, liblinear_eps], np.float64)
    check(fn(session._h, mask, args.ctypes.data, out["vec"].ctypes.data, out["fvec"].ctypes.data, out["z"].ctypes.data,
             out["exch"].ctypes.data, out["diff"].ctypes.data, out["ctrl"].ctypes.data, out["ctrl_raw"].ctypes.data, out["wz"].ctypes.data,
             ptr(out["l1thr"]), out["rho"].ctypes.data, res.ctypes.data, info.ctypes.data))
    out.update(info=inf, maxdiff=float(res[0]), mindiff=float(res[1]), stop=int(res[2]))
    return out


def _internal_keyed_last_call():
    """Test hook: the most recent keyed call of the process -> (key boundaries of its chunks, streamed, stage ms, wait ms)."""
    fn = lib().mlease_internal_keyed_last_call
    fn.argtypes, fn.restype = [C.c_void_p, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_double),
                               C.POINTER(C.c_double)], C.c_int
    n, s, a, b = C.c_int32(), C.c_int32(), C.c_double(), C.c_double()
    check(fn(None, 0, C.byref(n), None, None, None))
    bounds = np.zeros(max(n.value, 1), np.int64)
    check(fn(bounds.ctypes.data, n.value, C.byref(n), C.byref(s), C.byref(a), C.byref(b)))
    return bounds[:n.value], bool(s.value), a.value, b.value
