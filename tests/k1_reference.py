"""fp64 reference of the K1 gradient pass, per-column error bounds derived from the kernels' arithmetic, and a numpy fp32 emulation
of each kernel's order of operations (CPU only).

One partition is held as CSR over the Dg feature columns (dense data: every column of every row); the intercept is column Dt - 1
and is not stored.  At the fp32 point beta = float(w):

    s_i = x_i . beta + beta_bias + o_i,  t_i = y_i s_i,  p_i = sigma(t_i),  q_i = sigma(-t_i)
    loss = sum_i w_i (log1p(exp(-|t_i|)) + max(-t_i, 0)),  r_i = -w_i y_i q_i,  g_c = sum_i x_ic r_i,  sqrt(d_i) = sqrt(w_i p_i q_i)

Bounds (first order in the unit roundoffs; u = 2^-24, gamma_m = m u / (1 - m u)):
  * s_i is an fp32 dot product: |ds_i| <= gamma_m (sum_j |x_ij beta_j| + |beta_bias| + |o_i|), m the most roundings a term goes
    through in the kernel's order (dot_depth: the lane chains, the shuffle levels, the bias and the offset).
  * e = __expf(-|t|) has a documented error of 2 + floor(1.173 |t|) ulp (relative 2^-23 per ulp); below 2^-126 the result is
    flushed to 0 (relative error 1).  __frcp_rn and the fp32 products are correctly rounded.  This bounds the relative error
    eps_q of q (and of r = -w y q with its product rounding), and |dr_i| <= w_i (p_i q_i |ds_i| + q_i eps_q) e^|ds_i|.
  * Column sums: |g_c - g_ref,c| <= sum_i |x_ic| |dr_i| + sum over fp32 runs of gamma_m sum_run |x_ic r_i| + fp64 terms, with m the
    fp32 run length of the kernel before each fp64 add: RT rows (dense), the column's depth in a segment (fused), the column's
    float-atomic count in a CTA's rows + 1 (general CSR), one product (fixed point) plus, per contribution, the fixed-point
    resolution 2^-(kbits + e_hi + 1) of the CTA (k1_csr_fx_kernel: e_hi from the bound per * wmax * max(vmax, 1), kbits from per).
  * The loss adds the documented absolute error 2^-21.41 of __logf on [0.5, 1] per row; sqrt(d) its own propagated error.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np

U = 2.0 ** -24          # fp32 unit roundoff
U64 = 2.0 ** -53
BF16_U = 2.0 ** -8      # bf16 round-to-nearest: 8 significant bits
LOGF_ABS = 2.0 ** -21.41
EXP_FLUSH_T = 87.0      # __expf(-|t|) flushes to 0 once 2^(-|t| log2 e) < 2^-126 (|t| > 87.34); from 87 on it is counted as lost


def gamma(m, u=U):
    m = np.asarray(m, np.float64)
    return m * u / (1.0 - m * u)


@dataclass
class Part:
    """One partition: CSR rows over Dg features (bias not stored), labels y in {+1, -1}, weights, offsets.  dense_ldx > 0 marks a
    dense partition (all Dg columns listed in every row; the kernel's row dot has ldx terms)."""
    rowptr: np.ndarray
    colidx: np.ndarray
    vals: np.ndarray
    y: np.ndarray
    w: np.ndarray
    o: np.ndarray
    Dg: int
    dense_ldx: int = 0

    @property
    def n(self):
        return len(self.y)

    @property
    def Dt(self):
        return self.Dg + 1

    @property
    def rows(self):
        return np.repeat(np.arange(self.n), np.diff(self.rowptr))

    @staticmethod
    def from_dense(X, response, weight, offset):
        X = np.ascontiguousarray(X, np.float32)
        n, Dg = X.shape
        rp = np.arange(n + 1, dtype=np.int64) * Dg
        return Part(rp, np.tile(np.arange(Dg, dtype=np.int32), n), X.reshape(-1).copy(), labels(response), np.asarray(weight, np.float32),
                    np.asarray(offset, np.float32), Dg, dense_ldx=(Dg + 1 + 3) // 4 * 4)

    @staticmethod
    def from_csr(rowptr, colidx, vals, response, weight, offset, Dg, binary=False):
        v = np.asarray(vals, np.float32).copy()
        if binary:
            v[:] = 1.0
        return Part(np.asarray(rowptr, np.int64), np.asarray(colidx, np.int32), v, labels(response), np.asarray(weight, np.float32),
                    np.asarray(offset, np.float32), int(Dg))


def labels(response):
    """Responses {1, 0, -1} -> y {+1, -1, -1}."""
    return np.where(np.asarray(response) > 0, 1, -1).astype(np.int8)


@dataclass
class Ref:
    s: np.ndarray
    t: np.ndarray
    p: np.ndarray
    q: np.ndarray
    r: np.ndarray
    g: np.ndarray
    f: float
    sd: np.ndarray
    loss_rows: np.ndarray
    absdot: np.ndarray   # sum_j |x_ij beta_j| + |beta_bias| + |o_i|
    nterms: np.ndarray   # terms of the kernel's row sum (+ bias + offset)


def reference(part: Part, beta) -> Ref:
    b = np.asarray(beta, np.float32).astype(np.float64)
    assert len(b) == part.Dt
    rows = part.rows
    x = part.vals.astype(np.float64)
    xb = x * b[part.colidx]
    s = np.bincount(rows, xb, part.n) + b[-1] + part.o.astype(np.float64)
    y = part.y.astype(np.float64)
    w = part.w.astype(np.float64)
    t = y * s
    e = np.exp(-np.abs(t))
    p = np.where(t >= 0, 1.0 / (1.0 + e), e / (1.0 + e))
    q = np.where(t >= 0, e / (1.0 + e), 1.0 / (1.0 + e))
    r = -w * y * q
    lr = w * (np.log1p(e) + np.maximum(-t, 0.0))
    g = np.bincount(part.colidx, x * r[rows], part.Dt).astype(np.float64)   # (int64 when the partition stores no value)
    g[-1] = r.sum()
    absdot = np.bincount(rows, np.abs(xb), part.n) + abs(b[-1]) + np.abs(part.o.astype(np.float64))
    return Ref(s, t, p, q, r, g, float(lr.sum()), np.sqrt(w * p * q), lr, absdot, ref_nterms(part))


# ---------------------------------------------------------------------------------------------------------------------------------
# per-row errors
# ---------------------------------------------------------------------------------------------------------------------------------
@dataclass
class RowErr:
    ds: np.ndarray
    dr: np.ndarray
    dl: np.ndarray
    eps_sd: np.ndarray   # relative error of the emitted sqrt(d)
    grow: np.ndarray


def dense_shape(ldx):
    """G, RT, nsl of the dense K1 tile plan (k1_plan) for a row width ldx."""
    ncg = ldx // 4
    G = -(-ncg // 256)
    G = 4 if G == 3 else G
    return G, (4 if G == 4 else 8), (min(16, max(1, 256 // ncg)) if G == 1 else 1)


def dot_depth(part: Part, plan: "Plan | None"):
    """Most fp32 roundings any term of s_i = x_i . beta + beta_bias + o_i goes through in the kernel's summation order (+ 1 for the
    product, which the kernels fuse into an FMA): a sum whose terms each pass through at most m roundings is within gamma_m of the
    sum of their magnitudes.  Dense: 4 G chained FMAs per thread, 5 butterfly levels, 8 warp partials in sequence (one row slice),
    or 4 FMAs, ceil(ncg / 32) lane-strided adds and 5 levels (several slices); + the offset.  CSR: ceil(len / 16) chained FMAs per
    lane of a half-warp and 4 levels (fixed point, fused), ceil(len / 32) and 5 levels (general CSR); + bias + offset.  Without a
    plan: the row's terms in any order."""
    lens = np.diff(part.rowptr)
    if plan is None:
        return ref_nterms(part)
    if part.dense_ldx:
        G, RT, nsl = dense_shape(part.dense_ldx)
        ncg = part.dense_ldx // 4
        d = 4 * G + 5 + 8 + 1 if nsl == 1 else 4 + -(-ncg // 32) + 5 + 1
        return np.full(part.n, d + 1)
    if plan.kind == "csr":
        return -(-lens // 32) + 5 + 2 + 1
    return -(-lens // 16) + 4 + 2 + 1


def ref_nterms(part: Part):
    cnt = np.diff(part.rowptr) if not part.dense_ldx else np.full(part.n, part.dense_ldx)
    return cnt + 2


def row_errors(part: Part, ref: Ref, plan: "Plan | None" = None) -> RowErr:
    at = np.abs(ref.t)
    ds = gamma(dot_depth(part, plan)) * ref.absdot
    grow = np.exp(ds)   # p q and q change by at most this factor over [t - ds, t + ds]
    flushed = at >= EXP_FLUSH_T
    eps_e = np.where(flushed, 1.0, (2.0 + np.floor(1.173 * (at + ds))) * 2.0 ** -23)
    frac = np.exp(-at) / (1.0 + np.exp(-at))
    eps_inv = eps_e * frac + 2 * U                                    # (1 + e) rounded, then a correctly rounded reciprocal
    eps_big = eps_e + eps_inv + U                                    # e * inv
    pos = ref.t >= 0
    eps_q = np.where(pos, eps_big, eps_inv) + U                      # + the rounding of -w y * q
    eps_p = np.where(pos, eps_inv, eps_big)
    w = part.w.astype(np.float64)
    dr = w * (ref.p * ref.q * ds + ref.q * eps_q) * grow
    # loss row: w (max(-t, 0) - __logf(inv)): q |ds| from the margin, the absolute error of __logf on [0.5, 1], inv's relative
    # error, and the roundings of the subtraction and of the product with w
    dl = w * (ref.q * ds * grow + LOGF_ABS + eps_inv + 2 * U * (np.maximum(-ref.t, 0.0) + np.log1p(np.exp(-at)))) * (1 + 4 * U)
    eps_sd = 0.5 * (eps_p + eps_q + 2 * U) + U + 0.5 * ds * grow
    eps_sd = np.where(flushed, 1.0, eps_sd)
    return RowErr(ds, dr, dl, eps_sd, grow)


# ---------------------------------------------------------------------------------------------------------------------------------
# accumulation plans: how each kernel adds the per-row contributions of a column
# ---------------------------------------------------------------------------------------------------------------------------------
@dataclass
class Plan:
    """kind: 'dense' (RT), 'fused' (seg_rows), 'fx' / 'fx_window' (chunks, wmax, vmax), 'csr' (chunks)."""
    kind: str
    RT: int = 8
    seg_rows: int = 0
    chunks: int = 1

    def per(self, n):
        return (n + self.chunks - 1) // self.chunks


def plan_from_info(info, b, n):
    """The Plan of problem b from mlease_b200._hooks.batch_grad's result."""
    k = info["kind"]
    if k == "dense":
        return Plan("dense", RT=info["RT"], chunks=int(info["chunks"][b]))
    if k == "fused":
        return Plan("fused", seg_rows=info["RT"], chunks=int(info["chunks"][b]))
    return Plan(k, chunks=int(info["chunks"][b]))


def fx_scales(part: Part, per):
    """e_hi and kbits of k1_csr_fx_kernel (gradient mode, with intercept) for a CTA of `per` rows: bound, computed in fp32 as the
    kernel does, and the fixed-point resolution 0.5 2^-(kbits + e_hi) of one contribution."""
    wmax = np.float32(part.w.max()) if part.n else np.float32(0)
    vmax = np.float32(np.abs(part.vals).max()) if len(part.vals) else np.float32(0)
    bound = np.float32(np.float32(per) * wmax) * np.float32(max(vmax, np.float32(1)))
    if not (bound > 0 and bound < np.float32(3.0e38)):
        bound = np.float32(1)
    e_hi = 29 - (math.frexp(float(bound))[1] - 1 + 1)
    kbits = max(0, min(30 - int(per).bit_length() if per > 0 else 30 - 1, 24))
    return e_hi, kbits, 0.5 * 2.0 ** (-kbits - e_hi)


def _chunk_of_rows(part: Part, plan: Plan):
    if plan.kind == "fused":
        return np.arange(part.n) // plan.seg_rows
    if plan.kind == "dense":
        return np.arange(part.n) // plan.RT
    return np.arange(part.n) // max(1, plan.per(part.n))


def grad_bound(part: Part, ref: Ref, plan: Plan, err: RowErr | None = None):
    """Per-column bound on |g_kernel - g_ref| (Dt entries), and its parts (prop, fp32, fixed point) for reporting."""
    err = err or row_errors(part, ref, plan)
    rows = part.rows
    Dt = part.Dt
    x = np.abs(part.vals.astype(np.float64))
    xr = x * np.abs(ref.r[rows])
    absr = np.abs(ref.r)
    prop = np.bincount(part.colidx, x * err.dr[rows], Dt).astype(np.float64)
    prop[-1] = err.dr.sum()
    ch = _chunk_of_rows(part, plan)
    nch = int(ch.max()) + 1 if part.n else 1
    key = ch[rows].astype(np.int64) * Dt + part.colidx
    cnt = np.bincount(key, minlength=nch * Dt)
    sxr = np.bincount(key, xr, nch * Dt)
    rows_in = np.bincount(ch, minlength=nch)
    sr = np.bincount(ch, absr, nch)
    fx = np.zeros(Dt)
    if plan.kind == "dense":
        acc = gamma(plan.RT) * np.bincount(part.colidx, xr, Dt)
        acc[-1] = gamma(plan.RT) * absr.sum()   # the physical bias column is summed like the others
    elif plan.kind == "fused":
        acc = np.bincount(np.arange(nch * Dt) % Dt, gamma(cnt) * sxr, Dt)
        acc[-1] = gamma(-(-plan.seg_rows // 48) + 2) * absr.sum()   # per-lane fp32 sums, the pair add and the fp32 segment partial
    elif plan.kind == "csr":
        acc = np.bincount(np.arange(nch * Dt) % Dt, gamma(cnt + 1) * sxr, Dt)
        acc[-1] = (gamma(rows_in) * sr).sum()
    else:   # fixed point: one product rounding, then exact integer sums at the CTA's resolution
        acc = gamma(1) * np.bincount(part.colidx, xr, Dt)
        acc[-1] = 0.0
        res = fx_scales(part, plan.per(part.n))[2]
        fx = np.bincount(part.colidx, minlength=Dt) * res
        fx[-1] = part.n * res
    ccount = np.bincount(part.colidx, minlength=Dt).astype(np.float64)
    ccount[-1] = part.n
    f64 = (ccount + plan.chunks + 16) * U64 * np.append(np.bincount(part.colidx, xr, Dt)[:-1], absr.sum())
    return prop + acc + fx + f64, dict(prop=prop, fp32=acc, fx=fx)


def loss_bound(part: Part, ref: Ref, plan: Plan, err: RowErr | None = None):
    err = err or row_errors(part, ref, plan)
    m = (-(-plan.seg_rows // 48) + 1) if plan.kind == "fused" else 0   # the fused kernel sums a lane's rows in fp32
    return float(err.dl.sum() + gamma(m) * ref.loss_rows.sum() + (part.n + plan.chunks + 16) * U64 * ref.loss_rows.sum())


def sd_bound(ref: Ref, err: RowErr):
    return ref.sd * err.eps_sd * (1 + 4 * U) + 2.0 ** -126


def xt_check(part: Part, ref: Ref, err: RowErr, xt_bits: np.ndarray):
    """Checks the bf16 Xt rows (n x Dp bits) against x_ic sqrt(d_i): within half a bf16 ulp (one per duplicate of a column in a
    row) plus the propagated sqrt(d) error; positions no row lists (and the padding) exactly 0.  Returns the worst ratio."""
    n, Dp = xt_bits.shape
    xt = (xt_bits.astype(np.uint32) << 16).view(np.float32).astype(np.float64)
    rows = part.rows
    key = rows.astype(np.int64) * Dp + part.colidx
    ref_sum = np.bincount(key, part.vals.astype(np.float64), n * Dp)
    abs_sum = np.bincount(key, np.abs(part.vals.astype(np.float64)), n * Dp)
    kdup = np.bincount(key, minlength=n * Dp).astype(np.float64)
    bias = np.arange(n) * Dp + part.Dt - 1
    ref_sum[bias] += 1.0; abs_sum[bias] += 1.0; kdup[bias] += 1
    sd = np.repeat(ref.sd, Dp)
    dsd = np.repeat(sd_bound(ref, err), Dp)
    want = ref_sum * sd
    bnd = abs_sum * dsd + kdup * (BF16_U + U) * (1 + BF16_U) ** kdup * abs_sum * (sd + dsd) + 2.0 ** -133
    got = xt.reshape(-1)
    listed = kdup > 0
    assert np.all(got[~listed] == 0.0), "Xt has values outside the rows' patterns"
    d = np.abs(got - want)[listed]
    assert np.all(np.isfinite(got[listed]))
    ratio = d / bnd[listed]
    assert np.all(ratio <= 1.0), ("Xt", int(np.argmax(ratio)), float(ratio.max()))
    return float(ratio.max()) if ratio.size else 0.0


# ---------------------------------------------------------------------------------------------------------------------------------
# fp32 emulation of the kernels' order of operations
# ---------------------------------------------------------------------------------------------------------------------------------
def seq_sum32(keys, vals, nkeys):
    """fp32 sums of vals per key, each key's values added one after the other in the given order."""
    keys = np.asarray(keys, np.int64)
    vals = np.asarray(vals, np.float32)
    acc = np.zeros(nkeys, np.float32)
    if len(keys) == 0:
        return acc
    order = np.argsort(keys, kind="stable")
    k = keys[order]
    v = vals[order]
    rank = np.arange(len(k)) - np.searchsorted(k, k, side="left")
    o2 = np.argsort(rank, kind="stable")
    bounds = np.searchsorted(rank[o2], np.arange(rank.max() + 2))
    for r in range(rank.max() + 1):
        sel = o2[bounds[r]:bounds[r + 1]]
        acc[k[sel]] = acc[k[sel]] + v[sel]
    return acc


def _butterfly32(v):
    """xor-shuffle tree over the last axis (a power of two) in fp32: the value every lane holds at the end."""
    v = v.astype(np.float32)
    m = v.shape[-1] // 2
    while m >= 1:
        v = (v + v[..., np.arange(v.shape[-1]) ^ m]).astype(np.float32)
        m //= 2
    return v[..., 0]


def _dot32(part: Part, b, plan: Plan, with_bias=True):
    """s_i + o_i in the kernel's fp32 order (see dot_depth)."""
    f32 = np.float32
    n = part.n
    if part.dense_ldx:
        ldx = part.dense_ldx
        G, RT, nsl = dense_shape(ldx)
        ncg = ldx // 4
        Xf = np.zeros((n, ldx), f32)
        Xf[:, :part.Dg] = part.vals.reshape(n, part.Dg)
        Xf[:, part.Dt - 1] = 1.0 if with_bias else 0.0
        bf = np.zeros(ldx, f32)
        bf[:part.Dt] = b
        prod = (Xf * bf).astype(f32).reshape(n, ncg, 4)
        if nsl == 1:   # thread t: column groups t + 256 g, chained; warp butterflies; 8 warp partials in sequence
            th = np.zeros((n, 256), f32)
            for g in range(G):
                for k in range(4):
                    cg = np.arange(256) + 256 * g
                    ok = cg < ncg
                    th[:, ok] = (th[:, ok] + prod[:, cg[ok], k]).astype(f32)
            wv = _butterfly32(th.reshape(n, 8, 32))
            sc = np.zeros(n, f32)
            for wq in range(8):
                sc = (sc + wv[:, wq]).astype(f32)
        else:          # thread cg: 4 chained products; lane-strided sums over the ncg partials; warp butterfly
            th = np.zeros((n, ncg), f32)
            for k in range(4):
                th = (th + prod[:, :, k]).astype(f32)
            lanes = np.zeros((n, 32), f32)
            for c in range(ncg):
                lanes[:, c % 32] = (lanes[:, c % 32] + th[:, c]).astype(f32)
            sc = _butterfly32(lanes)
        return (sc + part.o).astype(f32)
    Wl = 32 if plan.kind == "csr" else 16
    rows = part.rows
    pos = np.arange(len(rows)) - part.rowptr[rows]
    prod = (part.vals * b[part.colidx]).astype(f32)
    lanes = seq_sum32(rows * Wl + pos % Wl, prod, n * Wl).reshape(n, Wl)
    sc = _butterfly32(lanes)
    if with_bias:
        sc = (sc + b[-1]).astype(f32)
    return (sc + part.o).astype(f32)


DEFECTS = ("drop_last_row", "dup_row", "move_entry", "lose_bias_partial", "q_one_minus_p", "no_bias")


def emulate(part: Part, beta, plan: Plan, defect: str | None = None):
    """-> (g [Dt] float64, f, sd [n] float32) as the kernel of `plan` computes them, with an optional seeded defect."""
    f32 = np.float32
    b = np.asarray(beta, np.float32)
    rows = part.rows
    Dt, n = part.Dt, part.n
    s = _dot32(part, b, plan, with_bias=defect != "no_bias")
    y = part.y.astype(f32)
    w = part.w
    t = (y * s).astype(f32)
    with np.errstate(under="ignore", over="ignore"):
        e = np.exp(-np.abs(t)).astype(f32)
    e[e < f32(2.0 ** -126)] = 0   # ex2.approx.ftz
    inv = (f32(1) / (f32(1) + e)).astype(f32)
    ei = (e * inv).astype(f32)
    pos = t >= 0
    p = np.where(pos, inv, ei)
    q = np.where(pos, ei, inv)
    if defect == "q_one_minus_p":
        q = np.where(pos, (f32(1) - p).astype(f32), q)
    r = ((-w * y).astype(f32) * q).astype(f32)
    lrow = (w * (np.where(pos, f32(0), -t) - np.log(inv)).astype(f32)).astype(f32)
    sd = np.sqrt(((w * p).astype(f32) * q).astype(f32)).astype(f32)
    # gradient contributions (row, column, value, product) in CSR order; the bias as one more entry of every row
    ent_row, ent_col, ent_val = rows, part.colidx.astype(np.int64), part.vals
    ch = _chunk_of_rows(part, plan)
    nch = int(ch.max()) + 1
    rmask = np.ones(n, f32)
    bias_rows = np.ones(n, f32)
    if defect == "drop_last_row":
        last = np.flatnonzero(ch == 0)[-1]
        rmask[last] = 0
    if defect == "lose_bias_partial":
        bias_rows[ch == 0] = 0
    if defect == "dup_row":
        sel = rows == 0
        ent_row = np.concatenate([ent_row, rows[sel]]); ent_col = np.concatenate([ent_col, ent_col[sel]])
        ent_val = np.concatenate([ent_val, part.vals[sel]])
    if defect == "move_entry":
        ent_col = ent_col.copy()
        c0 = ent_col[0]
        ent_col[0] = c0 + 1 if c0 + 1 < Dt - 1 else c0 - 1
    rr = (r * rmask).astype(f32)
    g = np.zeros(Dt)
    if plan.kind == "dense":   # RT-row runs of fp32 products (bias column physical), fp64 over runs
        ent_row = np.concatenate([ent_row, np.arange(n)]); ent_col = np.concatenate([ent_col, np.full(n, Dt - 1)])
        ent_val = np.concatenate([ent_val, bias_rows])
        key = ch[ent_row].astype(np.int64) * Dt + ent_col
        acc = seq_sum32(key, (ent_val * rr[ent_row]).astype(f32), nch * Dt)
        g = np.bincount(np.arange(nch * Dt) % Dt, acc.astype(np.float64), Dt)
    elif plan.kind == "fused":   # per segment: each column's entries in row order in fp32; the bias from per-lane fp32 sums
        key = ch[ent_row].astype(np.int64) * Dt + ent_col
        acc = seq_sum32(key, (ent_val * rr[ent_row]).astype(f32), nch * Dt)
        g = np.bincount(np.arange(nch * Dt) % Dt, acc.astype(np.float64), Dt)
        loc = np.arange(n) - ch * plan.seg_rows
        lane = ch * 48 + loc % 48
        lsum = seq_sum32(lane, (rr * bias_rows).astype(f32), nch * 48).reshape(nch, 24, 2)
        wsum = (lsum[:, :, 0] + lsum[:, :, 1]).astype(f32)
        seg = wsum.astype(np.float64).sum(1).astype(f32).astype(np.float64)
        g[-1] = seg.sum()
        llane = seq_sum32(lane, lrow, nch * 48).reshape(nch, 24, 2)
        lw = (llane[:, :, 0] + llane[:, :, 1]).astype(f32)
        return g, float(lw.astype(np.float64).sum()), sd
    elif plan.kind == "csr":   # float atomics per CTA (emulated in CSR order), the bias after each row
        ent_row = np.concatenate([ent_row, np.arange(n)]); ent_col = np.concatenate([ent_col, np.full(n, Dt - 1)])
        ent_val = np.concatenate([ent_val, bias_rows])
        o = np.argsort(ent_row, kind="stable")
        ent_row, ent_col, ent_val = ent_row[o], ent_col[o], ent_val[o]
        key = ch[ent_row].astype(np.int64) * Dt + ent_col
        acc = seq_sum32(key, (ent_val * rr[ent_row]).astype(f32), nch * Dt)
        g = np.bincount(np.arange(nch * Dt) % Dt, acc.astype(np.float64), Dt)
    else:   # fixed point per CTA: hi = rint(c S), lo = rint((c S - hi) 2^k), exact integer sums
        e_hi, kbits, _ = fx_scales(part, plan.per(n))
        s_hi, s_k = f32(2.0 ** e_hi), f32(2.0 ** kbits)
        rs = (rr * s_hi).astype(f32)
        ent_row = np.concatenate([ent_row, np.arange(n)]); ent_col = np.concatenate([ent_col, np.full(n, Dt - 1)])
        ent_val = np.concatenate([ent_val, bias_rows])
        ts = (ent_val * rs[ent_row]).astype(f32)
        h = np.rint(ts)
        lo = np.rint(((ts - h).astype(f32) * s_k).astype(f32))
        key = ch[ent_row].astype(np.int64) * Dt + ent_col
        hi_s = np.bincount(key, h.astype(np.float64), nch * Dt)
        lo_s = np.bincount(key, lo.astype(np.float64), nch * Dt)
        part_g = (hi_s + lo_s * 2.0 ** -kbits) * 2.0 ** -e_hi
        g = np.bincount(np.arange(nch * Dt) % Dt, part_g, Dt)
    return g, float(lrow.astype(np.float64).sum()), sd


# ---------------------------------------------------------------------------------------------------------------------------------
# Hv / diagonal modes
# ---------------------------------------------------------------------------------------------------------------------------------
def hv_reference_and_bound(part: Part, beta, v, mode, plan: Plan, rowl1=None, vinf=None):
    """fp64 data term of the Hv (mode 1: sum_i x_ic d_i (x_i . v + v_bias)) or diagonal (mode 2: sum_i x_ic^2 d_i) pass at
    beta = float(w), v = float(v), with d_i = w_i p_i q_i, and the per-column bound of the kernels: d_i is read back as the square
    of the emitted fp32 sqrt(d_i) (relative error 2 eps_sd + u), x_i . v is an fp32 dot product, t_i = d_i a_i one more rounding;
    the column sums are accumulated as in the gradient mode, with the fixed-point bound of k1_fx_mode_bound.
    -> (reference [Dt], bound [Dt])."""
    ref = reference(part, beta)
    err = row_errors(part, ref, plan)
    vf = np.asarray(v, np.float32).astype(np.float64)
    rows = part.rows
    Dt, n = part.Dt, part.n
    x = part.vals.astype(np.float64)
    d = ref.sd ** 2
    dd = d * (2 * err.eps_sd + err.eps_sd ** 2 + 2 * U)
    if mode == 1:
        a = np.bincount(rows, x * vf[part.colidx], n) + vf[-1]
        absa = np.bincount(rows, np.abs(x * vf[part.colidx]), n) + abs(vf[-1])
        da = gamma(-(-np.diff(part.rowptr) // 16) + 4 + 1 + 1) * absa   # half-warp lane chains, 4 levels, v_bias (as dot_depth)
        tr = d * a
        dt_row = dd * np.abs(a) + (d + dd) * da + U * (d + dd) * (np.abs(a) + da)
        xe = x
    else:
        tr = d
        dt_row = dd + U * (d + dd)
        xe = x * x
    out = np.bincount(part.colidx, xe * tr[rows], Dt)
    out[-1] = tr.sum()
    axe = np.abs(xe) * (1 + 2 * U)   # x^2 of the diagonal is one more fp32 product
    prop = np.bincount(part.colidx, axe * dt_row[rows], Dt)
    prop[-1] = dt_row.sum()
    xt = np.abs(xe) * (np.abs(tr) + dt_row)[rows]
    at = np.abs(tr) + dt_row
    ch = _chunk_of_rows(part, plan)
    nch = int(ch.max()) + 1
    key = ch[rows].astype(np.int64) * Dt + part.colidx
    cnt = np.bincount(key, minlength=nch * Dt)
    sxt = np.bincount(key, xt, nch * Dt)
    fx = np.zeros(Dt)
    if plan.kind == "fused":
        acc = np.bincount(np.arange(nch * Dt) % Dt, gamma(cnt + 1) * sxt, Dt)
        acc[-1] = gamma(-(-plan.seg_rows // 48) + 2) * at.sum()
    else:
        acc = gamma(2) * np.bincount(part.colidx, xt, Dt)
        acc[-1] = 0.0
        per = plan.per(n)
        wmax = np.float32(part.w.max())
        vmax = np.float32(np.abs(part.vals).max())
        if mode == 1:
            bound = np.float32(np.float32(np.float32(np.float32(np.float32(per) * np.float32(0.25)) * wmax) * np.float32(np.float32(rowl1) + np.float32(1)))
                               * np.float32(vinf)) * np.float32(max(vmax, np.float32(1)))
        else:
            bound = np.float32(np.float32(np.float32(per) * np.float32(0.25)) * wmax) * np.float32(max(np.float32(vmax * vmax), np.float32(1)))
        if not (bound > 0 and bound < np.float32(3.0e38)):
            bound = np.float32(1)
        e_hi = 29 - math.frexp(float(bound))[1]
        kbits = max(0, min(30 - int(per).bit_length(), 24))
        res = 0.5 * 2.0 ** (-kbits - e_hi)
        fx = np.bincount(part.colidx, minlength=Dt) * res
        fx[-1] = n * res
    f64 = (np.append(np.bincount(part.colidx, minlength=Dt)[:-1], n) + plan.chunks + 16) * U64 * np.append(
        np.bincount(part.colidx, xt, Dt)[:-1], at.sum())
    return out, prop + acc + fx + f64


# ---------------------------------------------------------------------------------------------------------------------------------
# test data
# ---------------------------------------------------------------------------------------------------------------------------------
def synth(seed, n, Dg, dense=False, nnz=8, edge=False, dup=False, binary=False, empty_rows=False):
    """One partition's arrays (dict: X or rowptr/colidx/vals, response, weight, offset) and its Part.

    Every case has 'hot' rows (~2 %): offset 15 y, so t ~ +15 and q ~ 3e-7, and they alone list the last feature (dense: the
    column is 0 elsewhere); a q formed as 1 - p in fp32 is wrong there by ~10 %.  CSR rows list 1 .. 2 nnz sorted unique columns
    of the first Dg - 2 (every 7th never: columns absent from the partition); the first 40 rows also list feature Dg - 2.  edge adds weights 0, responses -1 / 0 / 1, offsets
    up to +-30, rows with |t| up to ~100 (feature 0 at +-70 / scale: the betas of make_betas give feature 0 the weight scale),
    column scales 2^-12 .. 2^12; dup (CSR) repeats one column in some rows and shuffles rows; empty_rows leaves some rows empty."""
    rng = np.random.default_rng(seed)
    scale = np.exp2(rng.integers(-12, 13, Dg)).astype(np.float32) if edge else np.ones(Dg, np.float32)
    scale[0] = 1.0
    hot = rng.random(n) < 0.02
    hot[min(5, n - 1)] = True
    huge = (rng.random(n) < 0.02) & ~hot if edge else np.zeros(n, bool)
    response = (rng.random(n) < 0.5).astype(np.int32)
    if edge:
        response = rng.integers(-1, 2, n).astype(np.int32)
    y = np.where(response > 0, 1.0, -1.0)
    weight = rng.uniform(0.5, 2.0, n).astype(np.float32)
    offset = rng.normal(0, 0.1, n).astype(np.float32)
    if edge:
        weight[rng.random(n) < 0.05] = 0.0
        big = rng.random(n) < 0.05
        offset[big] = rng.uniform(-30, 30, big.sum())
        offset[huge] = 30.0 * np.sign(rng.normal(size=huge.sum()))
    offset[hot] = 15.0 * y[hot]
    out = dict(response=response, weight=weight, offset=offset)
    if dense:
        X = (rng.normal(size=(n, Dg)) * scale).astype(np.float32)
        X[:, -1] = 0.0
        X[hot, -1] = rng.uniform(0.5, 1.5, hot.sum()) * scale[-1]
        X[huge, 0] = 70.0 * np.sign(rng.normal(size=huge.sum()))
        out["X"] = X
        return out, Part.from_dense(X, response, weight, offset)
    avail = np.array([c for c in range(Dg - 2) if c % 7 != 3] or [0])
    rowptr = [0]; cols = []; vals = []
    for i in range(n):
        k = int(rng.integers(1, 2 * nnz + 1))
        if empty_rows and rng.random() < 0.03:
            k = 0
        c = np.sort(rng.choice(avail, size=min(k, len(avail)), replace=False)).astype(np.int64)
        if huge[i] and 0 not in c:
            c = np.sort(np.append(c, 0))
        if i < 40 and Dg > 2:
            c = np.append(c, Dg - 2)   # a column of the first rows only (one segment of the fused kernel)
        if hot[i] and Dg - 1 > 0:
            c = np.append(c, Dg - 1)
        v = (rng.normal(size=len(c)) * scale[c]).astype(np.float32)
        if huge[i]:
            v[c == 0] = 70.0 * np.sign(rng.normal())
        if dup and len(c) and rng.random() < 0.3:
            j = int(rng.integers(len(c)))
            c = np.append(c, c[j]); v = np.append(v, np.float32(rng.normal() * scale[c[j]]))
        if dup:
            o = rng.permutation(len(c)); c = c[o]; v = v[o]
        cols.append(c); vals.append(v); rowptr.append(rowptr[-1] + len(c))
    out.update(rowptr=np.array(rowptr, np.int64), colidx=np.concatenate(cols).astype(np.int32), vals=np.concatenate(vals).astype(np.float32))
    return out, Part.from_csr(out["rowptr"], out["colidx"], out["vals"], response, weight, offset, Dg, binary=binary)


def make_betas(Dg, count, seed, nnz=8, edge_seed=None):
    """count fp32 points (Dt entries): beta_c ~ N(0, 0.5 / sqrt(nnz)) / scale_c (the scales of synth(edge_seed, ..., edge=True),
    else 1), beta_0 = 1 / scale_0, a different intercept per point, each point a different multiple of the first."""
    rng = np.random.default_rng(seed)
    scale = np.ones(Dg)
    if edge_seed is not None:
        scale = np.exp2(np.random.default_rng(edge_seed).integers(-12, 13, Dg)).astype(np.float64)
        scale[0] = 1.0
    base = rng.normal(0, 0.5 / math.sqrt(nnz), Dg) / scale
    base[0] = 1.0
    out = []
    for l in range(count):
        b = np.append(base * (1.0 + 0.25 * l) + rng.normal(0, 0.01 / math.sqrt(nnz), Dg) / scale, 0.3 * (l + 1) - 0.5)
        b[0] = 1.0
        out.append(b.astype(np.float32).astype(np.float64))
    return out


def ratio(diff, bound):
    """|error| / bound per entry: 0 where both are 0 (columns no row lists must be exactly 0), inf where only the bound is."""
    diff = np.abs(np.asarray(diff, np.float64))
    bound = np.asarray(bound, np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(bound > 0, diff / np.where(bound > 0, bound, 1.0), np.where(diff > 0, np.inf, 0.0))
