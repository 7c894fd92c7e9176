"""fp64 replica of the device-side Newton x-update state machine (csrc/newton.cu), in plain numpy.

Each function restates one kernel from its formulas: begin (newton_begin_kernel), reduce_partials (k1_partial_reduce_kernel),
decide (k1_reduce_decide_kernel), solve (newton_solve_kernel, given r = H0^-1 q), cg_init / cg_step (cg_init_kernel,
cg_step_kernel).  A state is a dict: the x-update fields of Ctrl (common.cuh) plus the vectors beta, beta_t, m, q, g_t, g_acc,
dir (Dt long), the secant ring bfgs_S, bfgs_Y [BFGS_M, Dt], bfgs_rho, bfgs_alpha [BFGS_M], the fp32 copies beta_tf and qf, and
for the matrix-free path cg_r, cg_p, cg_z, cg_Hp, cg_diag, hv_vf.  state["wide"] says whether the batch keeps the bf16 Ysym
(the decide kernel then writes qf).  Every function returns a new state; state["branch"] is the set of branch names the call took,
so a test can assert which branches its cases reach (BRANCHES lists them all).

Every threshold of the state machine is a constant below and is used nowhere else: a deliberate change of one in newton.cu is a
one-line change here.

What can be compared by bits with the kernels: everything, when the data make every sum exact (dyadic values: small integers
times powers of two), because each scalar formula is evaluated in the kernel's order with IEEE operations.  The expressions
whose operands are not exact on such data -- the rejected step's trial point beta + alpha dir with alpha = 0.1 or 0.6 of the old
one, and the updates of the two loops with the new pair's rho = 1 / s.y -- are fused multiply-adds on the device and are computed
here with one rounding (fma).  On generic data the block reductions run in
another order than numpy's sums: scalars agree to a few ulp x Dt and discrete outcomes wherever the deciding quantity is not
within a relative margin of its threshold (near())."""
import copy
from fractions import Fraction

import numpy as np

BFGS_M = 6
CG_MAX_STEPS = 64
CG_ETA = 0.1
ACCEPT_FRAC = 0.5                 # accept while phi'(alpha) <= ACCEPT_FRAC |phi'(0)|
SHRINK_LO, SHRINK_HI = 0.1, 0.6   # clamp of the secant root, as fractions of alpha
MAX_REJECTS = 40                  # the line search gives up (fail 2) at reject MAX_REJECTS + 1
SY_REL = 1e-10                    # a pair is kept when s.y > SY_REL sqrt(s.s y.y)
TAU_LO, TAU_HI = 0.5, 2.0         # clamp of one self-scaling factor
H0_LO, H0_HI = 0.25, 16.0         # clamp of h0_scale
POOR_RATIO = 0.25                 # cheap rebuilds: refresh when |g| contracted by less than 4x
STUCK_RATIO, STUCK_STEPS = 0.5, 12  # expensive rebuilds: less than 2x after a dozen steps on one factor
MIN_EXACT_EVALS = 2               # contraction is judged between exact gradients
BETA_FLOOR = 1e-2                 # the stop tests scale with max(|beta|_inf, BETA_FLOOR)
STALL_TOL, STALL_RATIO, STALL_COUNT, STALL_MIN_STEPS = 1e-5, 0.5, 2, 2
REFRESH_STEPS_CHEAP, REFRESH_STEPS_EXPENSIVE = 6, 16

INT_FIELDS = ("done", "have_dir", "need_solve", "need_hess", "emit", "hess_valid", "fail", "newton_steps", "evals", "rejects",
              "hess_builds", "stall", "bfgs_count", "k1_chunks", "refresh_next", "skip_eval", "warm_used", "build_step",
              "max_newton", "hess_policy", "rebuild_is_expensive", "cg_active", "cg_iter")
REAL_FIELDS = ("h0_scale", "worst_ratio", "alpha", "phi0", "f_acc", "f_t", "gnorm", "gnorm_prev", "dirnorm", "dirnorm_prev", "xtol",
               "cg_rz", "cg_g2", "hv_vinf")
TOTALS = ("tot_evals", "tot_newton", "tot_rejects", "tot_hess")
VECTORS = ("beta", "beta_t", "m", "q", "g_t", "g_acc", "dir")
CG_VECTORS = ("cg_r", "cg_p", "cg_z", "cg_Hp", "cg_diag")

BRANCHES = (
    "decide:done", "accept:no_dir", "accept:curvature", "accept:first_exact", "reject:unclamped", "reject:clamp_lo", "reject:clamp_hi",
    "reject:nan", "reject:give_up", "eval:counted", "eval:skipped", "stop:zero_gradient", "stop:max_newton",
    "pair:stored", "pair:refused_sy_nonpositive", "pair:refused_sy_small", "pair:refused_rebuild", "pair:none_matrix_free",
    "h0:tau_lo", "h0:tau_hi", "h0:tau_free", "h0:clamp_lo", "h0:clamp_hi", "h0:cheap_unchanged",
    "emit:always", "emit:never", "emit:poor", "emit:stuck", "emit:invalid", "emit:deferred", "emit:none", "need_hess", "spec:no_rebuild",
    "solve:idle", "solve:fail_phi0", "solve:fail_nan", "solve:xtol", "solve:xtol_before_exact", "solve:stall_counted", "solve:stall_stop",
    "solve:stall_reset", "solve:refresh_next", "solve:h0_scaled", "solve:floor",
    "begin:emit", "begin:no_emit", "begin:h0_repaired", "begin:skip_eval_cleared", "begin:skip_eval_kept",
    "cg_init:idle", "cg_init:unit_diagonal", "cg_step:idle", "cg_step:curvature", "cg_step:forcing", "cg_step:cap", "cg_step:go",
)


def new_state(Dt, wide=False, matrix_free=False):
    st = {k: 0 for k in INT_FIELDS + TOTALS}
    st.update({k: 0.0 for k in REAL_FIELDS})
    st.update(h0_scale=1.0, alpha=1.0, xtol=1e-8, max_newton=50, wide=bool(wide), branch=set())
    for k in VECTORS:
        st[k] = np.zeros(Dt)
    st["q"] = np.ones(Dt)
    st["bfgs_S"], st["bfgs_Y"] = np.zeros((BFGS_M, Dt)), np.zeros((BFGS_M, Dt))
    st["bfgs_rho"], st["bfgs_alpha"] = np.zeros(BFGS_M), np.zeros(BFGS_M)
    st["beta_tf"], st["qf"] = np.zeros(Dt, np.float32), np.zeros(Dt, np.float32)
    if matrix_free:
        for k in CG_VECTORS:
            st[k] = np.zeros(Dt)
        st["hv_vf"] = np.zeros(Dt, np.float32)
    return st


def _next(st):
    s = copy.deepcopy(st)
    s["branch"] = set()
    return s


def _max_abs(v):
    """max |v| as the kernels take it: fmax from 0, which skips NaN."""
    return float(np.fmax.reduce(np.abs(np.asarray(v, np.float64)), initial=0.0))


def fma(a, x, y):
    """fl(a x + y) with one rounding, as the device's fused multiply-add (a scalar; x, y vectors or scalars)."""
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        out = np.asarray(float(a) * x + y, np.float64).copy()
    if np.isfinite(float(a)):
        fa = Fraction(float(a))
        xs, ys, os_ = x.reshape(-1), y.reshape(-1), out.reshape(-1)
        for k in np.flatnonzero((xs != 0.0) & np.isfinite(xs) & np.isfinite(ys)):
            os_[k] = float(fa * Fraction(float(xs[k])) + Fraction(float(ys[k])))
    return out if out.ndim else float(out)


def near(value, threshold, rel=1e-12):
    """Whether a deciding quantity is within the relative margin of its threshold (the outcome may then differ from the device's)."""
    return abs(value - threshold) <= rel * max(abs(value), abs(threshold))


def begin(st, xtol, max_newton, policy, invalidate, expensive):
    s = _next(st)
    bf = s["beta"].astype(np.float32)
    s["beta"], s["beta_t"], s["beta_tf"] = bf.astype(np.float64), bf.astype(np.float64), bf
    s["dir"] = np.zeros_like(s["beta"])
    if invalidate:
        s["hess_valid"] = 0
    if not s["h0_scale"] > 0.0:
        s["h0_scale"] = 1.0
        s["branch"].add("begin:h0_repaired")
    for k in ("done", "have_dir", "need_solve", "need_hess", "fail", "newton_steps", "evals", "rejects", "hess_builds", "stall",
              "build_step", "warm_used"):
        s[k] = 0
    for k in ("phi0", "f_acc", "f_t", "gnorm", "gnorm_prev", "dirnorm", "dirnorm_prev", "worst_ratio"):
        s[k] = 0.0
    s.update(alpha=1.0, xtol=float(xtol), max_newton=int(max_newton), hess_policy=int(policy), rebuild_is_expensive=int(expensive))
    if not expensive:
        s["h0_scale"] = 1.0
    s["emit"] = 1 if (policy != 2 and (policy == 1 or not s["hess_valid"] or s["refresh_next"])) else 0
    s["cg_active"] = 0
    s["refresh_next"] = 0
    if s["emit"]:
        if s["skip_eval"]:
            s["branch"].add("begin:skip_eval_cleared")
        s["skip_eval"] = 0
    elif s["skip_eval"]:
        s["branch"].add("begin:skip_eval_kept")
    s["branch"].add("begin:emit" if s["emit"] else "begin:no_emit")
    return s


def reduce_partials(parts, nct, fp32=False):
    """Column sums of parts[:nct] in the kernel's fixed order: 8 strided groups (rows grp, grp + 8, ...), then the group sums in order."""
    parts = np.asarray(parts, np.float32 if fp32 else np.float64)
    a = np.zeros(parts.shape[1])
    for grp in range(8):
        sg = np.zeros(parts.shape[1])
        for t in range(grp, nct, 8):
            sg = sg + parts[t].astype(np.float64)
        a = a + sg
    return a


def decide(st, loss_parts, spec=0):
    """k1_reduce_decide_kernel on a state whose g_t holds the reduced data-term gradient of beta_t."""
    s = _next(st)
    br = s["branch"]
    if s["done"]:
        br.add("decide:done")
        return s
    have_dir = s["have_dir"] != 0
    dlt = s["beta_t"] - s["m"]
    g = s["g_t"] + s["q"] * dlt
    s["g_t"] = g
    prior2 = float(np.sum(s["q"] * dlt * dlt))
    ginf = _max_abs(g)
    phi = float(np.sum(g * s["dir"])) if have_dir else 0.0
    lossp = float(np.sum(np.asarray(loss_parts, np.float64)[:s["k1_chunks"]]))
    sy = ss = yy = 0.0
    if have_dir:
        sk, yk = s["beta_t"] - s["beta"], g - s["g_acc"]
        sy, ss, yy = float(np.sum(sk * yk)), float(np.sum(sk * sk)), float(np.sum(yk * yk))
    s["scalars"] = dict(phi=phi, sy=sy, ss=ss, yy=yy, ginf=ginf, prior2=prior2, lossp=lossp)
    s["f_t"] = f_t = lossp + 0.5 * prior2
    if not s["skip_eval"]:
        s["evals"] += 1
        s["tot_evals"] += 1
        br.add("eval:counted")
    else:
        s["warm_used"] = 1
        br.add("eval:skipped")
    s["skip_eval"] = 0
    first_exact = have_dir and s["warm_used"] and s["evals"] == 1
    action, alpha = 1, s["alpha"]
    s["decide_margin"] = None   # (value, threshold) of the accept test, for near()
    if have_dir and not first_exact:
        a0 = abs(s["phi0"])
        s["decide_margin"] = (phi, ACCEPT_FRAC * a0)
        if not phi <= ACCEPT_FRAC * a0:
            action = 0
            an = alpha * a0 / (phi + a0)
            lo, hi = SHRINK_LO * alpha, SHRINK_HI * alpha
            clamped = float(np.fmin(np.fmax(an, lo), hi))
            br.add("reject:nan" if phi != phi else "reject:clamp_lo" if clamped == lo and an != lo else
                   "reject:clamp_hi" if clamped == hi and an != hi else "reject:unclamped")
            alpha = clamped
            s["rejects"] += 1
            s["tot_rejects"] += 1
            if s["rejects"] > MAX_REJECTS or phi != phi:
                s["fail"], s["done"] = 2, 1
                if phi == phi:
                    br.add("reject:give_up")
        else:
            br.add("accept:curvature")
    else:
        br.add("accept:first_exact" if first_exact else "accept:no_dir")
    if action == 1:
        s["gnorm_prev"] = s["gnorm"]
        s["gnorm"] = ginf
        s["f_acc"] = f_t
        if have_dir:
            s["newton_steps"] += 1
            s["tot_newton"] += 1
            if s["gnorm_prev"] > 0.0 and s["evals"] >= MIN_EXACT_EVALS:
                s["worst_ratio"] = float(np.fmax(s["worst_ratio"], ginf / s["gnorm_prev"]))
        if ginf == 0.0:
            s.update(done=1, need_solve=0, need_hess=0)
            br.add("stop:zero_gradient")
        elif s["newton_steps"] >= s["max_newton"]:
            s.update(done=1, fail=3, need_solve=0, need_hess=0)
            br.add("stop:max_newton")
        else:
            s["need_solve"] = 1
            deferred = bool(spec and s["emit"])
            s["need_hess"] = 1 if (s["emit"] and not spec) else 0
            if s["need_hess"]:
                br.add("need_hess")
            if spec and not s["emit"]:
                br.add("spec:no_rebuild")
            if s["hess_policy"] == 1:
                s["emit"] = 1
                br.add("emit:always")
            elif s["hess_policy"] == 2:
                s["emit"] = 0
                br.add("emit:never")
            else:
                exp = bool(s["rebuild_is_expensive"])
                stuck = exp and have_dir and s["gnorm_prev"] > 0.0 and ginf > STUCK_RATIO * s["gnorm_prev"] and \
                    s["newton_steps"] - s["build_step"] >= STUCK_STEPS
                poor = stuck or (not exp and have_dir and s["evals"] >= MIN_EXACT_EVALS and s["gnorm_prev"] > 0.0 and
                                 ginf > POOR_RATIO * s["gnorm_prev"])
                s["emit"] = 1 if (poor and not s["need_hess"]) else 0
                why = "emit:none"
                if s["emit"]:
                    why = "emit:stuck" if stuck else "emit:poor"
                if not s["need_hess"] and not s["hess_valid"]:
                    s["emit"] = 1
                    why = "emit:invalid" if why == "emit:none" else why
                if deferred:
                    s["emit"] = 1
                    why = "emit:deferred"
                br.add(why)
    else:
        s["need_solve"] = s["need_hess"] = 0
    s["alpha"] = alpha
    slot = -1
    if action == 1 and s["need_hess"]:
        s["bfgs_count"] = 0
    if action == 1 and have_dir:
        if s["need_hess"]:
            br.add("pair:refused_rebuild")
        elif s["hess_policy"] == 2:
            br.add("pair:none_matrix_free")
        elif not sy > 0.0:
            br.add("pair:refused_sy_nonpositive")
        elif not sy > SY_REL * np.sqrt(ss * yy):
            br.add("pair:refused_sy_small")
        else:
            br.add("pair:stored")
            slot = s["bfgs_count"] % BFGS_M
            s["bfgs_rho"][slot] = 1.0 / sy
            s["bfgs_count"] += 1
            if s["rebuild_is_expensive"]:
                raw = -(alpha * s["phi0"]) / sy
                tau = float(np.fmin(np.fmax(raw, TAU_LO), TAU_HI))
                br.add("h0:tau_lo" if raw < TAU_LO else "h0:tau_hi" if raw > TAU_HI else "h0:tau_free")
                prod = s["h0_scale"] * tau
                if prod < H0_LO:
                    br.add("h0:clamp_lo")
                if prod > H0_HI:
                    br.add("h0:clamp_hi")
                s["h0_scale"] = float(np.fmin(np.fmax(prod, H0_LO), H0_HI))
            else:
                br.add("h0:cheap_unchanged")
    s["stored_slot"] = slot
    if action == 1:
        if slot >= 0:
            s["bfgs_S"][slot] = s["beta_t"] - s["beta"]
            s["bfgs_Y"][slot] = g - s["g_acc"]
        s["beta"] = s["beta_t"].copy()
        s["g_acc"] = g.copy()
    else:
        btf = fma(alpha, s["dir"], s["beta"]).astype(np.float32)
        s["beta_t"], s["beta_tf"] = btf.astype(np.float64), btf
    s["action"] = action
    if s["done"] or not s["need_solve"]:
        return s
    # the first loop of the two-loop recursion, newest pair first: q -> g_t
    q = s["g_acc"].copy()
    for j in range(min(s["bfgs_count"], BFGS_M)):
        sl = (s["bfgs_count"] - 1 - j) % BFGS_M
        a = s["bfgs_rho"][sl] * float(np.sum(s["bfgs_S"][sl] * q))
        s["bfgs_alpha"][sl] = a
        q = fma(-a, s["bfgs_Y"][sl], q)
    s["g_t"] = q
    if s["wide"]:
        s["qf"] = q.astype(np.float32)
    return s


def solve(st, r):
    """newton_solve_kernel given r = H0^-1 q (what the GEMV leaves in dir; q = state["g_t"] after decide)."""
    s = _next(st)
    br = s["branch"]
    if s["done"] or not s["need_solve"]:
        br.add("solve:idle")
        return s
    rhs = np.asarray(r, np.float64).copy()
    if s["h0_scale"] != 1.0:
        rhs = rhs * s["h0_scale"]
        br.add("solve:h0_scaled")
    npairs = min(s["bfgs_count"], BFGS_M)
    for j in range(npairs - 1, -1, -1):
        sl = (s["bfgs_count"] - 1 - j) % BFGS_M
        coef = fma(-s["bfgs_rho"][sl], float(np.sum(s["bfgs_Y"][sl] * rhs)), s["bfgs_alpha"][sl])
        rhs = fma(coef, s["bfgs_S"][sl], rhs)
    rhs = -rhs
    s["dir"] = rhs
    dinf, binf = _max_abs(rhs), _max_abs(s["beta"])
    phi0 = float(np.sum(rhs * s["g_acc"]))
    s["dirnorm_prev"] = s["dirnorm"]
    s.update(dirnorm=dinf, phi0=phi0, alpha=1.0, have_dir=1, need_solve=0, rejects=0)
    scale = float(np.fmax(binf, BETA_FLOOR))
    if binf < BETA_FLOOR:
        br.add("solve:floor")
    fin = 0
    s["solve_margins"] = [(dinf, s["xtol"] * scale), (dinf, STALL_TOL * scale), (dinf, STALL_RATIO * s["dirnorm_prev"])]
    # (the kernel also tests dinf != dinf; fmax skips NaN, so dinf is never NaN and a NaN direction shows in phi0 alone)
    if not phi0 < 0.0:
        s.update(fail=1, done=1)
        fin = 2
        br.add("solve:fail_nan" if phi0 != phi0 else "solve:fail_phi0")
    elif dinf <= s["xtol"] * scale and s["evals"] > 0:
        s["done"] = 1
        fin = 1
        br.add("solve:xtol")
    elif s["newton_steps"] >= STALL_MIN_STEPS and dinf <= STALL_TOL * scale and dinf > STALL_RATIO * s["dirnorm_prev"]:
        if dinf <= s["xtol"] * scale:
            br.add("solve:xtol_before_exact")
        s["stall"] += 1
        br.add("solve:stall_counted")
        if s["stall"] >= STALL_COUNT:
            s["done"] = 1
            fin = 1
            br.add("solve:stall_stop")
    else:
        if dinf <= s["xtol"] * scale:
            br.add("solve:xtol_before_exact")
        if s["stall"]:
            br.add("solve:stall_reset")
        s["stall"] = 0
    s["need_hess"] = 0
    if fin and s["hess_policy"] == 0 and s["hess_builds"] == 0 and \
            s["newton_steps"] >= (REFRESH_STEPS_EXPENSIVE if s["rebuild_is_expensive"] else REFRESH_STEPS_CHEAP):
        s["refresh_next"] = 1
        br.add("solve:refresh_next")
    s["fin"] = fin
    if fin == 2:
        return s
    bt = s["beta"] + rhs
    s["beta_tf"] = bt.astype(np.float32)
    s["beta_t"] = s["beta_tf"].astype(np.float64)
    if fin:
        s["beta"] = bt
    return s


def cg_begin(st):
    s = _next(st)
    s["cg_active"] = 1 if (not s["done"] and s["need_solve"]) else 0
    s["cg_iter"] = 0
    return s


def cg_init(st):
    """cg_init_kernel: cg_diag holds the data term of diag(H) on entry."""
    s = _next(st)
    if not s["cg_active"]:
        s["branch"].add("cg_init:idle")
        return s
    m = s["cg_diag"] + s["q"]
    bad = ~(m > 0.0)
    if bad.any():
        s["branch"].add("cg_init:unit_diagonal")
    m = np.where(bad, 1.0, m)
    r = s["g_acc"].copy()
    z = r / m
    s.update(cg_diag=m, cg_r=r, cg_z=z, cg_p=z.copy(), hv_vf=z.astype(np.float32), dir=np.zeros_like(r))
    s["cg_rz"], s["cg_g2"] = float(np.sum(r * z)), float(np.sum(r * r))
    s["hv_vinf"] = float(np.float32(_max_abs(s["hv_vf"])))
    return s


def cg_step(st):
    """cg_step_kernel: cg_Hp holds the data term X^T D X p on entry.  The updates dir += alpha p, r -= alpha Hp, p = z + beta p are
    fused multiply-adds on the device and plain multiply-adds here: bit-comparable only when alpha and beta are powers of two (or
    the products are otherwise exact), as the dyadic CG cases of the GPU test arrange."""
    s = _next(st)
    br = s["branch"]
    if not s["cg_active"]:
        br.add("cg_step:idle")
        return s
    hp = s["cg_Hp"] + s["q"] * s["cg_p"]
    s["cg_Hp"] = hp
    php = float(np.sum(s["cg_p"] * hp))
    rr = 0.0
    if php > 0.0:
        alpha = s["cg_rz"] / php
        s["dir"] = s["dir"] + alpha * s["cg_p"]
        s["cg_r"] = s["cg_r"] - alpha * hp
        rr = float(np.sum(s["cg_r"] * s["cg_r"]))
    s["cg_margin"] = (rr, CG_ETA * CG_ETA * s["cg_g2"])
    if not php > 0.0:
        s.update(fail=1, done=1, cg_active=0)
        br.add("cg_step:curvature")
        return s
    s["cg_iter"] += 1
    if s["cg_iter"] >= CG_MAX_STEPS:
        s["cg_active"] = 0
        br.add("cg_step:cap")
        return s
    if rr <= CG_ETA * CG_ETA * s["cg_g2"]:
        s["cg_active"] = 0
        br.add("cg_step:forcing")
        return s
    br.add("cg_step:go")
    z = s["cg_r"] / s["cg_diag"]
    rz = float(np.sum(s["cg_r"] * z))
    beta = rz / s["cg_rz"]
    p = z + beta * s["cg_p"]
    s.update(cg_z=z, cg_p=p, hv_vf=p.astype(np.float32), cg_rz=rz)
    s["hv_vinf"] = float(np.float32(_max_abs(s["hv_vf"])))
    return s


def rebuilt(st):
    """The control fields a factorisation leaves (the tail of the Cholesky kernels): call after decide set need_hess."""
    s = _next(st)
    s.update(hess_valid=1, bfgs_count=0, h0_scale=1.0, build_step=s["newton_steps"])
    s["hess_builds"] += 1
    s["tot_hess"] += 1
    return s
