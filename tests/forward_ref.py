"""Row-by-row reference of the layer's forward on the GPU's own similarities, for the forward row tests.

The inputs are one rank's S (npair_debug_read(0), or that of a materialised twin context in row-block mode, whose S is the same bits),
the labels of its rows and of the database columns, each row's self column by position (-1: none), the mining, and the GPU's
thresholds (npair_debug_read 1 and 2, which the L2 parity holds bit for bit against the oracle).  From them:

  statistics   min_within, max_within, max_between, max_all (fp32) and the same-label count, exactly.  A row with no same-label
               column keeps the reset values (reset_row_stats): min_within = FLT_MAX, max_within = -FLT_MAX, count 0; with no
               diff-label column max_between = -FLT_MAX; max_all of a row with no other column is -FLT_MAX.
  sums         A64, T64: fp64 sums of exp(s - max_all) over the selected same-label (A) and all selected (T) pairs whose exponent the
               row pass keeps.  The row pass evaluates ex2.approx.ftz(fmaf(s, LOG2E, -m2)), m2 = max_all * LOG2E in fp32: a term whose
               fp32 argument lies below -126 is 0 (the flush, DESIGN 5), and the reference drops exactly those terms.  The GPU's fp32
               sum must satisfy |A - A64| <= tau A64 + n_edge 2^-126, where n_edge counts terms whose argument lies within rounding
               of -126 (ex2.approx may flush or keep them) and tau (tau_rows) models the ex2.approx error, the argument's rounding,
               which grows with |m2| and |s - max_all|, and fp32 summation over a lane's ceil(N / (32 wpr)) terms, the warp tree and
               the row's segments.
  records      m2 = max_all * LOG2E - j, the transformed thresholds and the label bit for bit; j as lse_rows_kernel picks it from the
               GPU's A and T; m2c, cA and cT against fp64 of m2 + log2 T + log2 world - k, 2^(k-j) (1/T - 1/A) and 2^(k-j) / T of the
               GPU's own A and T; every field finite except m2c = +inf on a row with T = 0.
  log term     log(A / T) against fp64 log(A64 / T64) within the bound that A's and T's bounds imply; 0 where A64 or T64 is 0.
  tops         tops[0] = (fp64 sum of the GPU's per-row log values) / -Q within one float ulp; tops[1..3] = hits / Q exactly.
  retrieval    in the S domain: c_i = #{non-self j : s_j >= max_within_i} (every column when expf(max_within - max_all) underflows to
               0), hit_k <=> count > 0 and c_i <= min(k, N - 2).  A row is ambiguous when a column below max_within has
               expf(s_j - max_all) within 2 ulp of p* = expf(max_within - max_all) (CUDA's expf error) and counting it changes a
               decision; every other row must agree exactly.

Largest ratios |A - A64| / (tau A64) and |T - T64| / (tau T64) measured on an H100 80GB HBM3 (700 W) over test_gpu_forward_rows.py,
in 2^-24 units of A64 / T64 (the bound tau of that row in brackets):
  unit-norm rows, every case up to Q = N = 8192 and the memory rows at N = 8448: A 3.1 (52), T 3.0 (140)
  rows 60 .. 110 nats from their maximum (test_dynamic_range, |m2| ~ 185): A 94.5 (320), T 78.0 (284)
and no ambiguous retrieval row in any case but the planted dynamic-range rows' own."""
from __future__ import annotations

import math

import numpy as np

FLT_MAX = np.float32(3.4028234663852886e38)
LOG2E = np.float32(1.4426950408889634)
U24 = 2.0 ** -24
FLUSH = -126.0                # ex2.approx.ftz returns 0 below 2^-126
EDGE = 2.0 ** -14             # |argument + 126| within which ex2.approx's own error may flush or keep a term
HARD, EASY, RAND, RELATIVE_HARD, RELATIVE_EASY = 0, 1, 2, 3, 4
KLIST = (1, 5, 10)

# ------------------------------------------------------------------------------------------------------------------ selection
def _next_below(t):
    with np.errstate(over="ignore"):
        return np.nextafter(np.float32(t), np.float32(-np.inf)).astype(np.float32)


def selection(S, same, diff, posi, nega, margin_ident=0.0, margin_diff=0.0, ap_method=RAND, an_method=RAND, **_):
    """The oracle's selection rule (.cu:69-122, npair_oracle_np.forward) on the given per-row thresholds."""
    tp = (np.asarray(posi, np.float32) + np.float32(margin_ident)).astype(np.float32)[:, None]
    tn = (np.asarray(nega, np.float32) + np.float32(margin_diff)).astype(np.float32)[:, None]
    ap = {HARD: S < tp, EASY: S >= tp, RAND: np.ones_like(same), RELATIVE_HARD: S <= tp, RELATIVE_EASY: S >= tp}[ap_method]
    an = {HARD: S > tn, EASY: S <= tn, RAND: np.ones_like(same), RELATIVE_HARD: S >= tn, RELATIVE_EASY: S <= tn}[an_method]
    return (same & ap) | (diff & an)


def transformed_thresholds(posi, nega, margin_ident=0.0, margin_diff=0.0, ap_method=RAND, an_method=RAND, **_):
    """thr_p, thr_n of the row record (ap_thr / an_thr, kernels.cuh): each rule as one compare sgn * s <= thr'."""
    tp = (np.asarray(posi, np.float32) + np.float32(margin_ident)).astype(np.float32)
    tn = (np.asarray(nega, np.float32) + np.float32(margin_diff)).astype(np.float32)
    inf = np.full_like(tp, np.inf)
    thr_p = {HARD: _next_below(tp), EASY: -tp, RAND: inf, RELATIVE_HARD: tp, RELATIVE_EASY: -tp}[ap_method]
    thr_n = {HARD: _next_below(-tn), EASY: tn, RAND: inf, RELATIVE_HARD: -tn, RELATIVE_EASY: tn}[an_method]
    return thr_p.astype(np.float32), thr_n.astype(np.float32)


# ------------------------------------------------------------------------------------------------------------------ the reference
def reference(S, lab_rows, lab_cols, self_cols, posi, nega, mining, wpr=1):
    """The per-row reference of one rank (module docstring).  S: Q x N fp32, self_cols: [Q] column of each row's self pair (-1: none),
    wpr: warps per row of the row pass (its summation length per lane)."""
    S = np.ascontiguousarray(S, dtype=np.float32)
    Q, N = S.shape
    lab_rows = np.asarray(lab_rows, np.float32)
    lab_cols = np.asarray(lab_cols, np.float32)
    cols = np.arange(N)[None, :]
    notself = cols != np.asarray(self_cols)[:, None]
    eq = lab_rows[:, None] == lab_cols[None, :]
    same, diff = notself & eq, notself & ~eq
    st = dict(
        min_within=np.where(same, S, FLT_MAX).min(axis=1).astype(np.float32),
        max_within=np.where(same, S, -FLT_MAX).max(axis=1).astype(np.float32),
        max_between=np.where(diff, S, -FLT_MAX).max(axis=1).astype(np.float32),
        max_all=np.where(notself, S, -FLT_MAX).max(axis=1).astype(np.float32),
        cnt_same=same.sum(axis=1).astype(np.int64))
    sel = selection(S, same, diff, posi, nega, **mining)
    max_all = st["max_all"]
    m2 = (max_all * LOG2E).astype(np.float32)
    # the row pass's fp32 argument fmaf(s, LOG2E, -m2): s * LOG2E is exact in fp64, so one rounding to fp32 follows the FMA
    arg64 = S.astype(np.float64) * np.float64(LOG2E) - m2.astype(np.float64)[:, None]
    arg32 = arg64.astype(np.float32).astype(np.float64)
    kept = sel & (arg32 >= FLUSH)
    edge = sel & (np.abs(arg32 - FLUSH) <= EDGE)
    with np.errstate(over="ignore", under="ignore"):
        E64 = np.exp(S.astype(np.float64) - max_all.astype(np.float64)[:, None])
    A64 = np.where(kept & same, E64, 0.0).sum(axis=1)
    T64 = np.where(kept, E64, 0.0).sum(axis=1)
    st.update(same=same, diff=diff, notself=notself, sel=sel, kept=kept, A64=A64, T64=T64, m2=m2,
              n_edge_A=(edge & same).sum(axis=1), n_edge_T=edge.sum(axis=1),
              tau=tau_rows(N, wpr, m2, np.where(kept, np.abs(arg32), 0.0).max(axis=1)))
    return st


def tau_rows(N, wpr, m2, max_arg):
    """Per-row relative bound on A and T: ex2.approx (2^-22), the argument's error (|m2| + 2 |arg|) 2^-24 in log2 units (m2's rounding
    and the FMA's), i.e. ln 2 times that relative, and the fp32 sums: ceil(N / (32 wpr)) terms per lane, 5 levels of warp tree,
    wpr segments."""
    n_lane = -(-N // (32 * wpr))
    units = 4.0 + math.log(2.0) * (np.abs(m2.astype(np.float64)) + 2.0 * max_arg) + n_lane + 5 + wpr
    return units * U24


# ------------------------------------------------------------------------------------------------------------------ the checks
def check_stats(ref, gpu):
    """gpu: dict of the GPU's min_within, max_within, max_between, max_all, cnt_same (debug 3, 9, 4, 5, 8).  Returns the failures."""
    bad = []
    for k in ("min_within", "max_within", "max_between", "max_all"):
        g = np.asarray(gpu[k], np.float32)
        diff = g.view(np.uint32) != ref[k].view(np.uint32)
        if diff.any():
            i = int(np.argmax(diff))
            bad.append(f"{k}: {int(diff.sum())} rows, row {i} gpu {g[i]!r} ref {ref[k][i]!r}")
    c = np.asarray(gpu["cnt_same"]).astype(np.int64)
    if (c != ref["cnt_same"]).any():
        i = int(np.argmax(c != ref["cnt_same"]))
        bad.append(f"cnt_same: {int((c != ref['cnt_same']).sum())} rows, row {i} gpu {c[i]} ref {ref['cnt_same'][i]}")
    return bad


def _sum_ratio(g, r64, tau, n_edge):
    """|g - r64| over its allowance tau r64 + n_edge 2^-126, and over r64 in 2^-24 units (0 where both are 0)."""
    g = np.asarray(g, np.float64)
    err = np.abs(g - r64)
    allow = tau * r64 + n_edge * 2.0 ** -126
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.where(err == 0, 0.0, err / allow)
        units = np.where(err == 0, 0.0, err / r64 / U24)
    return ratio, units


def check_sums(ref, A, T):
    """The GPU's A and T (debug 6, 7) against A64 and T64.  Returns (failures, measured: worst error in 2^-24 units and its row's tau)."""
    bad, meas = [], {}
    for name, g, r64, ne in (("A", A, ref["A64"], ref["n_edge_A"]), ("T", T, ref["T64"], ref["n_edge_T"])):
        g = np.asarray(g, np.float32)
        if not np.isfinite(g).all():
            bad.append(f"{name}: non-finite")
        ratio, units = _sum_ratio(g, r64, ref["tau"], ne)
        over = ~(ratio <= 1.0)
        if over.any():
            i = int(np.argmax(np.where(over, np.nan_to_num(ratio, nan=np.inf), -1.0)))
            bad.append(f"{name}: {int(over.sum())} rows outside tau, row {i} gpu {float(g[i])!r} fp64 {r64[i]!r} "
                       f"({units[i]:.1f} x 2^-24, tau {ref['tau'][i] / U24:.1f})")
        i = int(np.nanargmax(units)) if units.size else 0
        meas[name] = (float(units[i]) if units.size else 0.0, float(ref["tau"][i] / U24) if units.size else 0.0)
    return bad, meas


def log_bound(ref):
    """Bound on |log(A/T) - log(A64/T64)|: the relative bounds of A and T (edge terms included), the fp32 division and logf."""
    with np.errstate(divide="ignore", invalid="ignore"):
        da = ref["tau"] + np.where(ref["A64"] > 0, ref["n_edge_A"] * 2.0 ** -126 / ref["A64"], 0.0)
        dt = ref["tau"] + np.where(ref["T64"] > 0, ref["n_edge_T"] * 2.0 ** -126 / ref["T64"], 0.0)
        L64 = np.where((ref["A64"] > 0) & (ref["T64"] > 0), np.log(ref["A64"] / ref["T64"]), 0.0)
    return L64, 1.01 * (da + dt) + 2 * U24 + 2 * U24 * np.abs(L64) + 1e-30


def check_log(ref, logv, A, T):
    """The GPU's log(A/T) (debug 11) against fp64; exactly 0 where the GPU's A or T is 0, and A is 0 exactly where A64 is."""
    bad = []
    logv = np.asarray(logv, np.float32)
    A = np.asarray(A, np.float32)
    T = np.asarray(T, np.float32)
    if not np.isfinite(logv).all():
        bad.append("log(A/T): non-finite")
    zero = (A == 0) | (T == 0)
    if (logv[zero] != 0).any():
        bad.append(f"log(A/T): {int((logv[zero] != 0).sum())} rows with A or T = 0 and a nonzero log")
    # a zero A64 with no edge term is exactly a zero A (every kept term is at least 2^-126)
    firm = (ref["n_edge_A"] == 0)
    if ((A == 0) != (ref["A64"] == 0))[firm].any():
        i = int(np.argmax(((A == 0) != (ref["A64"] == 0)) & firm))
        bad.append(f"A = 0 on row {i}: gpu {float(A[i])!r}, fp64 {ref['A64'][i]!r}")
    L64, bound = log_bound(ref)
    live = ~zero & (ref["A64"] > 0)
    err = np.abs(logv.astype(np.float64) - L64)
    over = live & ~(err <= bound)
    if over.any():
        i = int(np.argmax(np.where(over, err / bound, -1.0)))
        bad.append(f"log(A/T): {int(over.sum())} rows, row {i} gpu {float(logv[i])!r} fp64 {L64[i]!r} (bound {bound[i]:.3e})")
    return bad


def check_tops(tops, logv, hits, Q, num_tops):
    """tops[0] against the fp64 sum of the GPU's own per-row logs over -Q (one ulp: the finaliser's order differs); tops[1..num_tops-2]
    = hits / Q bit for bit.  hits: [3][Q] 0 / 1 flags (debug 12)."""
    bad = []
    ls = np.float32(np.float32(np.asarray(logv, np.float32).astype(np.float64).sum()) / np.float32(-Q))
    ulp = float(np.spacing(np.abs(ls))) if ls != 0 else float(np.finfo(np.float32).tiny)
    if not abs(float(tops[0]) - float(ls)) <= ulp:
        bad.append(f"tops[0] {tops[0]!r} vs per-row sum {ls!r}")
    hits = np.asarray(hits, np.float32).reshape(3, Q)
    for t in range(1, min(num_tops - 2, 3) + 1):
        want = np.float32(np.float32(int(hits[t - 1].sum())) / np.float32(Q))
        if np.float32(tops[t]) != want:
            bad.append(f"tops[{t}] {tops[t]!r} vs hits {int(hits[t - 1].sum())} / {Q} = {want!r}")
    return bad


def _ulp32(x):
    return np.spacing(np.abs(x.astype(np.float32))).astype(np.float64)


def retrieval(ref, S):
    """(hits [3][Q] of the S-domain rule, ambiguous [Q]) from the reference's statistics (module docstring)."""
    S = np.asarray(S, np.float32)
    Q, N = S.shape
    maxw, max_all, notself = ref["max_within"], ref["max_all"], ref["notself"]
    has = ref["cnt_same"] > 0
    with np.errstate(over="ignore", under="ignore"):
        pstar = np.exp((maxw - max_all).astype(np.float32)).astype(np.float32)                     # fp32, as expf
        e = np.exp((S - max_all[:, None]).astype(np.float32)).astype(np.float32)
    under = has & (pstar == 0)
    c_firm = (notself & (S >= maxw[:, None])).sum(axis=1)
    near = notself & (S < maxw[:, None]) & (np.abs(e.astype(np.float64) - pstar.astype(np.float64)[:, None])
                                            <= 2 * _ulp32(pstar)[:, None])
    c_hi = c_firm + near.sum(axis=1)
    c_firm = np.where(under, N - 1, c_firm)
    c_hi = np.where(under, N - 1, c_hi)
    hits = np.zeros((3, Q), np.int64)
    amb = np.zeros(Q, bool)
    for t, k in enumerate(KLIST):
        lim = min(k, N - 2)
        h_lo, h_hi = has & (c_firm <= lim), has & (c_hi <= lim)
        hits[t] = h_lo
        amb |= h_lo != h_hi
    return hits, amb


def check_hits(ref, S, hits_gpu):
    """Every non-ambiguous row's three flags exactly.  Returns (failures, number of ambiguous rows)."""
    Q = np.asarray(S).shape[0]
    h, amb = retrieval(ref, S)
    g = np.asarray(hits_gpu, np.float32).reshape(3, Q).astype(np.int64)
    wrong = (g != h).any(axis=0) & ~amb
    bad = []
    if wrong.any():
        i = int(np.argmax(wrong))
        bad.append(f"hits: {int(wrong.sum())} non-ambiguous rows differ, row {i} gpu {g[:, i].tolist()} ref {h[:, i].tolist()}")
    return bad, int(amb.sum())


def record_shift(A, T, k):
    """j of lse_rows_kernel: max(0, k - 127 - floor(log2 A)), A replaced by T when A = 0, 0 when both are 0."""
    A = np.asarray(A, np.float32)
    T = np.asarray(T, np.float32)
    amin = np.where(A > 0, A, T).astype(np.float64)
    with np.errstate(divide="ignore"):
        e = np.floor(np.log2(np.where(amin > 0, amin, 1.0)))
    return np.where(amin > 0, np.maximum(0, k - 127 - e), 0).astype(np.int64)


def check_records(ref, rec, A, T, lab_rows, posi, nega, mining, k, world=1):
    """rec: the [Q][8] row records (npair_row_scalars): {m2c, thr_n, m2, label, thr_p, cA, cT, 0}.  Returns (failures, j per row)."""
    bad = []
    rec = np.asarray(rec, np.float32).reshape(-1, 8)
    A = np.asarray(A, np.float32).astype(np.float64)
    T = np.asarray(T, np.float32).astype(np.float64)
    m2c, thr_n, m2, lab, thr_p, cA, cT = (rec[:, f] for f in range(7))
    j = record_shift(A, T, k)

    def bits(name, g, want):
        d = np.asarray(g, np.float32).view(np.uint32) != np.asarray(want, np.float32).view(np.uint32)
        if d.any():
            i = int(np.argmax(d))
            bad.append(f"record {name}: {int(d.sum())} rows, row {i} gpu {float(g[i])!r} want {float(want[i])!r}")

    bits("m2", m2, (ref["m2"] - j.astype(np.float32)).astype(np.float32))
    bits("label", lab, np.asarray(lab_rows, np.float32))
    tp, tn = transformed_thresholds(posi, nega, **mining)
    bits("thr_p", thr_p, tp)
    bits("thr_n", thr_n, tn)
    live = T > 0
    if not np.isfinite(np.where(live, m2c, 0)).all() or not (m2c[~live] == np.inf).all():
        bad.append("record m2c: non-finite on a row with T > 0, or not +inf on a row with T = 0")
    for name, f in (("m2", m2), ("thr_p", thr_p), ("thr_n", thr_n), ("cA", cA), ("cT", cT)):
        if name.startswith("thr"):
            if mining.get("ap_method" if name == "thr_p" else "an_method", RAND) == RAND:
                continue       # RAND selects every pair: its transformed threshold is +inf by definition
            f = f[live]        # a row with T = 0 selects nothing: its thresholds may be the sentinels' +-inf
        if not np.isfinite(f).all():
            i = int(np.argmax(~np.isfinite(f)))
            bad.append(f"record {name}: non-finite on {int((~np.isfinite(f)).sum())} rows, row {i} = {float(f[i])!r}")
    m2u = ref["m2"].astype(np.float64)
    with np.errstate(divide="ignore"):
        w_m2c = m2u + np.log2(np.where(live, T, 1.0)) + math.log2(world) - k
    tol_m2c = (np.abs(m2u) + np.abs(np.log2(np.where(live, T, 1.0))) + abs(math.log2(world)) + k) * 2.0 ** -22 + 2.0 ** -40
    d = live & ~(np.abs(m2c.astype(np.float64) - w_m2c) <= tol_m2c)
    if d.any():
        i = int(np.argmax(d))
        bad.append(f"record m2c: {int(d.sum())} rows, row {i} gpu {float(m2c[i])!r} fp64 {w_m2c[i]!r}")
    sc = np.ldexp(1.0, (k - j).astype(np.int64))
    with np.errstate(divide="ignore"):
        iA = np.where(A > 0, 1.0 / np.where(A > 0, A, 1.0), 0.0)
        iT = np.where(T > 0, 1.0 / np.where(T > 0, T, 1.0), 0.0)
    for name, g, want, tol in (("cA", cA, sc * (iT - iA), sc * (iA + iT) * 2 * U24), ("cT", cT, sc * iT, sc * iT * U24)):
        d = ~(np.abs(g.astype(np.float64) - want) <= tol + 1e-300)
        if d.any():
            i = int(np.argmax(d))
            bad.append(f"record {name}: {int(d.sum())} rows, row {i} gpu {float(g[i])!r} fp64 {want[i]!r} (j {int(j[i])})")
    return bad, j


def weighted_records(rec, w):
    """The row pass's weighted records [Q, 8] from the unweighted ones of the same forward: m2c - log2f(w) (+inf at w = 0), cA w and
    cT w; the rest unchanged.  log2 is NumPy's fp32 log2: exact for w = 2^-j, within an ulp of CUDA's log2f otherwise."""
    rec = np.array(rec, dtype=np.float32).reshape(-1, 8)
    w = np.asarray(w, dtype=np.float32)
    out = rec.copy()
    with np.errstate(divide="ignore", invalid="ignore"):
        out[:, 0] = np.where(w > 0, (rec[:, 0] - np.log2(w)).astype(np.float32), np.float32(np.inf))
    out[:, 5] = (rec[:, 5] * w).astype(np.float32)
    out[:, 6] = (rec[:, 6] * w).astype(np.float32)
    return out
