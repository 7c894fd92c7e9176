"""ctypes binding of the test hooks of libmlease_b200.so (csrc/mlease_internal.h): entry points for the tests and tools that drive
single kernels of a session's batches, not part of the C ABI.  SIG is applied once, by bound(); the wrappers below call it.

A hook that runs kernels on the ADMM batch consumes its x-update state (mlease_internal.h says what it leaves behind): begin()
again before iterating, or the library refuses the iteration.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._native import check, lib, ptr

_vp, _i32, _i64, _pi32, _pf64 = C.c_void_p, C.c_int32, C.c_int64, C.POINTER(C.c_int32), C.POINTER(C.c_double)
SIG = {
    "mlease_internal_set_keyed_budget": [_i64],
    "mlease_internal_keyed_last_call": [_vp, _i32, _pi32, _pi32, _pf64, _pf64],
    "mlease_internal_batch_hv": [_vp, _i32, _vp, _vp, _vp],
    "mlease_internal_batch_grad": [_vp] * 8,
    "mlease_internal_batch_factor": [_vp] * 6 + [_i32] * 3 + [_vp] * 5,
    "mlease_internal_direction": [_vp] * 13,
    "mlease_internal_newton_stage": [_vp, _i32, _i32] + [_vp] * 7 + [_i32, _vp, _pi32],
    "mlease_internal_xupdate_trace": [_vp, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _pi32],
    "mlease_internal_factor": [_vp, _i32, _vp, _vp, _vp, _vp],
    "mlease_internal_factored_direction": [_vp] * 5,
    "mlease_internal_ysym": [_vp, _i32, _vp, _pi32, _pi32],
    "mlease_internal_request_refresh": [_vp, _i32],
    "mlease_internal_set_csr_gram": [_vp, _i32],
    "mlease_internal_csr_gram": [_vp, _pi32, _pi32],
    "mlease_internal_dmma_shapes": [_vp, _vp, _i32, _i32, _vp, _vp],
    "mlease_internal_consensus": [_vp, _i32] + [_vp] * 13,
    "mlease_internal_partition_info": [_vp, _i32, _vp],
    "mlease_internal_partition_data": [_vp, _i32, _vp, _vp, _vp, _vp],
}

_bound = None


def bound():
    """The library with every hook of SIG typed (argtypes, restype int)."""
    global _bound
    if _bound is None:
        L = lib()
        for name, args in SIG.items():
            fn = getattr(L, name)
            fn.argtypes, fn.restype = args, C.c_int
        _bound = L
    return _bound


BFGS_M = 6   # secant pairs kept per problem (common.cuh)


def set_keyed_budget(nbytes):
    """Caps, process-wide, the device bytes the keyed calls plan with (0 = free memory only), so that small inputs stream through
    many chunks."""
    check(bound().mlease_internal_set_keyed_budget(int(nbytes)))


def keyed_last_call():
    """The most recent keyed call of the process -> (key boundaries of its chunks, streamed, stage ms, wait ms)."""
    fn = bound().mlease_internal_keyed_last_call
    n, s, a, b = C.c_int32(), C.c_int32(), C.c_double(), C.c_double()
    check(fn(None, 0, C.byref(n), None, None, None))
    bounds = np.zeros(max(n.value, 1), np.int64)
    check(fn(bounds.ctypes.data, n.value, C.byref(n), C.byref(s), C.byref(a), C.byref(b)))
    return bounds[:n.value], bool(s.value), a.value, b.value


PARTITION_INFO = ("n", "nnz", "csr", "ldx", "wmax", "vmax", "rowl1", "gram_pairs", "csr_unique", "block_major", "gram_col_index",
                  "k1_segments", "sg_S")


def partition_info(session, pid):
    """Partition pid as uploaded, after its deferred CSR checks and lists: dict of PARTITION_INFO (wmax, vmax, rowl1 float32, flags
    bool, the rest int)."""
    out = np.zeros(len(PARTITION_INFO), np.float64)
    check(bound().mlease_internal_partition_info(session._h, int(pid), out.ctypes.data))
    info = dict(zip(PARTITION_INFO, out))
    for k in PARTITION_INFO:
        info[k] = np.float32(info[k]) if k in ("wmax", "vmax", "rowl1") else \
            bool(info[k]) if k in ("csr", "csr_unique", "block_major", "gram_col_index", "k1_segments") else int(info[k])
    return info


def partition_data(session, pid, info=None):
    """The session's device copies of partition pid -> dict(y int8 [n], w, o float32 [n], X float32 [n, ldx] (dense) or vals float32
    [nnz] (CSR, as binary.feature left them))."""
    info = info or partition_info(session, pid)
    n = info["n"]
    y = np.zeros(n, np.int8)
    w, o = np.zeros(n, np.float32), np.zeros(n, np.float32)
    xv = np.zeros(info["nnz"] if info["csr"] else (n, info["ldx"]), np.float32)
    check(bound().mlease_internal_partition_data(session._h, int(pid), y.ctypes.data, w.ctypes.data, o.ctypes.data, xv.ctypes.data))
    return dict(y=y, w=w, o=o, **{"vals" if info["csr"] else "X": xv})


K1_KINDS = {1: "dense", 2: "fx", 3: "fx_window", 4: "csr", 5: "fused"}


def batch_grad(session, w, active=None, rows=None, want_sd=False, want_xt=False):
    """One K1 gradient pass over the ADMM batch of `session` (after begin()), problem b = partition * L + lambda at float(w[b])
    when active[b] (default: all).  rows: the row count of each partition (needed for want_sd / want_xt).  Consumes the batch's
    x-update state.
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
    check(bound().mlease_internal_batch_grad(session._h, act.ctypes.data, w.ctypes.data, f.ctypes.data, g.ctypes.data, ptr(sd), ptr(xt),
                                             info.ctypes.data))
    split = np.cumsum([0] + (n_b or []))
    return dict(f=f, g=g, sd=[sd[split[b]:split[b + 1]] for b in range(nprob)] if want_sd else None,
                xt=[xt[split[b] * Dp:split[b + 1] * Dp].reshape(-1, Dp) for b in range(nprob)] if want_xt else None,
                kind=K1_KINDS[int(info[0])], G=int(info[1]), dyn=int(info[2]), grid=int(info[3]), RT=int(info[4]), nsl=int(info[5]),
                chunks=info[8:].copy())


def batch_factor(session, mode, H=None, G=None, q=None, order=None, share=0, share_factor=False):
    """One factorisation of the ADMM batch of `session` (after begin(), ldh <= 2048) through the solver's rebuild code.  mode[b]:
    0 = done (untouched), 1 = factorise H[b] (Dt x Dt fp64), 2 = factorise the fp32 Gram G[b] plus diag(q[b]) through
    chol_prep_kernel.  order: launch order (a permutation or subset of the problems; default: batch order).  share / share_factor:
    the cold start of a rebuild slot (see mlease_internal_batch_factor).  Consumes the batch's x-update state.
    -> dict(L [nprob, Dt, Dt], Y, Hinv [nprob, ldh, ldh], Ldinv [nprob, ldh, 32], fail, done, hess_valid, tot_hess [nprob]);
    buffers no kernel wrote hold the all-ones NaN sentinel."""
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
    check(bound().mlease_internal_batch_factor(session._h, md.ctypes.data, ptr(Hc), ptr(Gc), ptr(qc), ptr(oc), 0 if oc is None else len(oc),
                                               int(share), int(bool(share_factor)), out["L"].ctypes.data, out["Y"].ctypes.data,
                                               out["Hinv"].ctypes.data, out["Ldinv"].ctypes.data, ctrl.ctypes.data))
    out.update(fail=ctrl[:, 0].copy(), done=ctrl[:, 1].copy(), hess_valid=ctrl[:, 2].copy(), tot_hess=ctrl[:, 3].copy())
    return out


def direction(session, active, g, S, Y, rho, count, h0, beta):
    """The quasi-Newton direction on the explicit inverse H^-1 (ldh <= 2048) of the active problems of the ADMM batch, through the
    kernels of a chord slot, after batch_factor.  Per problem: g [Dt] data-term gradient, S, Y [BFGS_M, Dt] secant ring
    (slot-major), rho [BFGS_M], count (bfgs_count), h0 (h0_scale), beta [Dt] point.  Consumes the batch's x-update state.
    -> dict(dir [nprob, Dt], phi0, dirnorm [nprob], beta_t [nprob, Dt]); NaN where inactive."""
    nprob, Dt = session.num_blocks * session.L, session.Dt
    act = np.ascontiguousarray(active, np.int32)
    g, beta = (np.ascontiguousarray(a, np.float64).reshape(nprob, Dt) for a in (g, beta))
    S, Y = (np.ascontiguousarray(a, np.float64).reshape(nprob, BFGS_M, Dt) for a in (S, Y))
    rho = np.ascontiguousarray(rho, np.float64).reshape(nprob, BFGS_M)
    cnt = np.ascontiguousarray(count, np.int32).reshape(nprob)
    h0 = np.ascontiguousarray(h0, np.float64).reshape(nprob)
    out = dict(dir=np.empty((nprob, Dt)), phi0=np.empty(nprob), dirnorm=np.empty(nprob), beta_t=np.empty((nprob, Dt)))
    check(bound().mlease_internal_direction(session._h, act.ctypes.data, g.ctypes.data, S.ctypes.data, Y.ctypes.data, rho.ctypes.data,
                                            cnt.ctypes.data, h0.ctypes.data, beta.ctypes.data, out["dir"].ctypes.data,
                                            out["phi0"].ctypes.data, out["dirnorm"].ctypes.data, out["beta_t"].ctypes.data))
    return out


STAGE_INTS = ("done", "have_dir", "need_solve", "need_hess", "emit", "hess_valid", "fail", "newton_steps", "evals", "rejects",
              "hess_builds", "stall", "bfgs_count", "k1_chunks", "refresh_next", "skip_eval", "warm_used", "build_step", "max_newton",
              "hess_policy", "rebuild_is_expensive", "cg_active", "cg_iter", "pad_")
STAGE_REALS = ("h0_scale", "worst_ratio", "alpha", "phi0", "f_acc", "f_t", "gnorm", "gnorm_prev", "dirnorm", "dirnorm_prev", "xtol",
               "cg_rz", "cg_g2", "hv_vinf", "tot_evals", "tot_newton", "tot_rejects", "tot_hess")
STAGE_CTRL = np.dtype([(k, np.int32) for k in STAGE_INTS] + [(k, np.float64) for k in STAGE_REALS])   # StageCtrl of mlease_internal.h
STAGE_VECS = ("beta", "beta_t", "m", "q", "g_t", "g_acc", "dir", "cg_r", "cg_p", "cg_z", "cg_Hp", "cg_diag")
STAGES = dict(begin=1, decide=2, solve=4, finish=8, cg_begin=16, cg_init=32, cg_step=64, cg_poll=128)


def newton_stage(session, stages=(), ctrl=None, vec=None, ring=None, fvec=None, gpart=None, fpart=None, spec=0, begin_args=None):
    """Inject an x-update state into every problem of the ADMM batch (after begin()), run the kernels named in `stages` (keys of
    STAGES) once through the solver's launchers, read the state back.  ctrl [nprob] STAGE_CTRL; vec [nprob, 12, ldx] (STAGE_VECS);
    ring [nprob, 2 BFGS_M ldx + 2 BFGS_M] (S, Y, rho, alpha); fvec [nprob, 3, ldx] float32 (beta_tf, qf = hv_vf, tf); gpart
    [nprob, nct, ldx], fpart [nprob, nct] or None; begin_args (xtol, max_newton, policy, invalidate, expensive).  Without stages:
    info only.  Consumes the batch's x-update state.
    -> dict(info=dict(nprob, Dt, ldx, ldh, part_rows, fused, matrix_free, ysym, expensive, group_L), ctrl, vec, ring, fvec, cg_any)."""
    mask = 0
    for k in stages:
        mask |= STAGES[k]
    info = np.zeros(12, np.int32)
    cg_any = C.c_int32(-1)
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
    check(bound().mlease_internal_newton_stage(session._h, mask, int(spec), ptr(begin_args) if mask else None, ptr(out.get("ctrl")),
                                               ptr(out.get("vec")), ptr(out.get("ring")), ptr(out.get("fvec")),
                                               ptr(gpart) if mask else None, ptr(fpart) if mask else None, nct, info.ctypes.data,
                                               C.byref(cg_any)))
    out["info"] = dict(zip(("nprob", "Dt", "ldx", "ldh", "part_rows", "fused", "matrix_free", "ysym", "expensive", "group_L"),
                           (int(x) for x in info)))
    out["cg_any"] = cg_any.value
    return out


def xupdate_trace(session, policy=0, invalidate=0, spec=(), max_slots=60, xtol=0.0, max_newton=0):
    """One real x-update of the ADMM batch, slot by slot through the solver's own slot code.  spec: slot indices asked to run
    speculatively (policy 0 only, never slot 0).  xtol / max_newton 0: the session's.
    -> dict(nslots, spec [nslots], with_hess [nslots], ctrl [nslots + 1, nprob] STAGE_CTRL, vec [nslots + 1, nprob, 12, ldx],
    ring [nslots + 1, nprob, 2 BFGS_M ldx + 2 BFGS_M], fvec [nslots + 1, nprob, 3, ldx]); entry 0 is the state newton_begin left,
    entry i + 1 the state after slot i."""
    info = newton_stage(session)["info"]
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
    check(bound().mlease_internal_xupdate_trace(session._h, args.ctypes.data, sp.ctypes.data, int(max_slots), ctrl.ctypes.data,
                                                vec.ctypes.data, ring.ctypes.data, fvec.ctypes.data, sinfo.ctypes.data, C.byref(n)))
    k = n.value
    return dict(nslots=k, spec=sinfo[:k, 0].copy(), with_hess=sinfo[:k, 1].copy(), ctrl=ctrl[:k + 1], vec=vec[:k + 1], ring=ring[:k + 1],
                fvec=fvec[:k + 1], info=info)


CONSENSUS_VECS = ("beta", "m", "q", "g_t", "x_d")
CONSENSUS_FVECS = ("u_f", "uplusx_f", "x_f")
CONSENSUS_CTRL = ("hess_valid", "skip_eval", "k1_chunks")
CONSENSUS_STAGES = dict(reset=1, init=2, pack=4, consensus=8)
CONSENSUS_INFO = ("nprob", "Dt", "ldx", "L", "P", "nlocal", "csr", "fused", "matrix_free", "regularizer", "k1_grid", "ctrl_bytes")


def consensus(session, stages=(), state=None, iter=1, liblinear_eps=0.01, read=True):
    """Inject a K4 state into the begun ADMM batch, run the stages named in `stages` (keys of CONSENSUS_STAGES, run in the order
    reset, init, pack, consensus) through the solver's own code, read everything back.  state: dict(vec [nprob, 5, ldx]
    (CONSENSUS_VECS), fvec [nprob, 3, ldx] float32 (CONSENSUS_FVECS), z [L, ldx], exch [L Dt + 1], diff [L], ctrl [nprob, 3] int32
    (CONSENSUS_CTRL)), whole vectors with their padding.  The consensus stage runs with the session's iteration counter at `iter`
    and its liblinear epsilon at `liblinear_eps`.  Without stages nothing is injected: the state is read (read=False: info only).
    With stages, consumes the batch's x-update state.
    -> dict(info, the state's keys after the last stage, ctrl_raw [2, nprob, ctrl_bytes] uint8 (before / after, the three ctrl
    fields zeroed), wz [L, ldx], l1thr [L] or None, rho [L], maxdiff, mindiff, stop)."""
    mask = stages if isinstance(stages, int) else 0   # (a raw mask: lets a test pass one the hook must refuse)
    for k in ([] if isinstance(stages, int) else stages):
        mask |= CONSENSUS_STAGES[k]
    info = np.zeros(12, np.int32)
    fn = bound().mlease_internal_consensus
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
