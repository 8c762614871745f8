"""NumPy restatement of NPairMultiClassLossLayer Forward_gpu/Backward_gpu.

TEST INFRASTRUCTURE ONLY -- an INDEPENDENT second restatement used to pin the C++ oracle
(oracle/npair_oracle.cpp); the two must agree (tests/test_oracle.py).  PARITY UNPINNED BY THE
REFERENCE (no tests / golden vectors upstream, Forward_cpu/Backward_cpu empty).

Written array-at-a-time (no shared code or loop structure with the C++ oracle) and following
/root/reference/npair_multi_class_loss.cu line ranges cited inline.
"""
from __future__ import annotations

import numpy as np

GLOBAL, LOCAL = 0, 1
HARD, EASY, RAND, RELATIVE_HARD, RELATIVE_EASY = 0, 1, 2, 3, 4
FLT_MAX = np.float32(3.4028234663852886e38)


class OracleError(RuntimeError):
    pass


def pos_index(sn: float, size: int) -> int:
    """.cu:285-287: size_t arithmetic for SN>=0, fp32 arithmetic otherwise (SURVEY 9.4 Q3)."""
    sn32 = np.float32(sn)
    if sn32 >= 0:  # -0.0 >= 0 is True
        return size - 1 - int(sn32)
    a = np.float32(size - 1)
    b = np.float32(sn32 * np.float32(size))
    return int(np.float32(a + b))  # int() truncates toward zero


def _thr_from_sorted(sorted_list: np.ndarray, sn: float) -> np.float32:
    if sorted_list.size == 0:
        raise OracleError("empty list")
    p = pos_index(sn, int(sorted_list.size))
    if p < 0 or p >= sorted_list.size:
        raise OracleError("pos out of range")
    v = sorted_list[p]
    return v if v >= 0 else -FLT_MAX  # .cu:288


def weighted_loss(logv, w, Z):
    """-(1/Z) sum_i w_i logv_i: the fp32 products w_i logv_i summed in fp64 (w None: the unweighted loss, DESIGN 4.5)."""
    lv = np.asarray(logv, dtype=np.float32)
    if w is not None:                                         # a row with w = 0 adds nothing, whatever its log value
        w = np.asarray(w, dtype=np.float32)
        with np.errstate(invalid="ignore"):
            lv = np.where(w == 0, np.float32(0), lv * w).astype(np.float32)
    return np.float32(np.float32(lv.astype(np.float64).sum()) / np.float32(-Z))


def forward(x_total, label_total, Q, world=1, rank=0, num_tops=5, margin_ident=0.0, margin_diff=0.0,
            identsn=-1.0, diffsn=-1.0, ap_region=LOCAL, ap_method=RAND, an_region=LOCAL, an_method=RAND,
            S_inject=None, anchor_weight=None):
    """Rank `rank`'s forward over the database x_total: (tops[5], state).  Rows past Q * world are memory rows (DESIGN 4.3), columns
    and never anchors, at world 1 only.  anchor_weight: the rank's Q weights, which change tops[0] alone (DESIGN 4.5)."""
    x_total = np.ascontiguousarray(x_total, dtype=np.float32)
    lab = np.ascontiguousarray(label_total, dtype=np.float32)
    N = x_total.shape[0]
    assert N >= Q * world and lab.shape[0] == N
    if N > Q * world and world > 1:
        raise OracleError("memory rows at world > 1")
    xl = x_total[rank * Q:(rank + 1) * Q]
    ll = lab[rank * Q:(rank + 1) * Q]
    # .cu:218 (BLAS accumulation order unspecified -> float64 accumulate, fp32 store)
    if S_inject is None:
        S = (xl.astype(np.float64) @ x_total.astype(np.float64).T).astype(np.float32)
    else:
        S = np.ascontiguousarray(S_inject, dtype=np.float32).reshape(Q, N).copy()
    # .cu:44-66
    rows = np.arange(Q)[:, None] + rank * Q
    cols = np.arange(N)[None, :]
    notself = rows != cols
    eq = ll[:, None] == lab[None, :]
    same = notself & eq
    diff = notself & ~eq
    # .cu:230-265
    min_within = np.where(same, S, FLT_MAX).min(axis=1).astype(np.float32)
    max_between = np.where(diff, S, -FLT_MAX).max(axis=1).astype(np.float32)
    max_all = np.where(notself, S, -FLT_MAX).max(axis=1).astype(np.float32)

    def is_rel(m):
        return m in (RELATIVE_HARD, RELATIVE_EASY)

    # .cu:275-337
    if ap_region == LOCAL:
        if not is_rel(ap_method):
            posi = max_between.copy()
        else:
            posi = np.array([_thr_from_sorted(np.sort(S[i][same[i]]), identsn) for i in range(Q)], dtype=np.float32)
    else:
        if not is_rel(ap_method):
            dg = S[diff]
            if dg.size == 0:
                raise OracleError("empty list")
            posi = np.full(Q, dg.max(), dtype=np.float32)
        else:
            posi = np.full(Q, _thr_from_sorted(np.sort(S[same]), identsn), dtype=np.float32)
    if an_region == LOCAL:
        if not is_rel(an_method):
            nega = min_within.copy()
        else:
            nega = np.array([_thr_from_sorted(np.sort(S[i][diff[i]]), diffsn) for i in range(Q)], dtype=np.float32)
    else:
        if not is_rel(an_method):
            ig = S[same]
            if ig.size == 0:
                raise OracleError("empty list")
            nega = np.full(Q, ig.min(), dtype=np.float32)
        else:
            nega = np.full(Q, _thr_from_sorted(np.sort(S[diff]), diffsn), dtype=np.float32)
    # .cu:69-122
    tp = (posi + np.float32(margin_ident)).astype(np.float32)[:, None]
    tn = (nega + np.float32(margin_diff)).astype(np.float32)[:, None]
    ap_rule = {HARD: S < tp, EASY: S >= tp, RAND: np.ones_like(same), RELATIVE_HARD: S <= tp, RELATIVE_EASY: S >= tp}[ap_method]
    an_rule = {HARD: S > tn, EASY: S <= tn, RAND: np.ones_like(same), RELATIVE_HARD: S >= tn, RELATIVE_EASY: S <= tn}[an_method]
    sel = (same & ap_rule) | (diff & an_rule)
    ident_num = (same & sel).sum(axis=1).astype(np.float32)
    diff_num = (diff & sel).sum(axis=1).astype(np.float32)
    # .cu:124-156 (expf in fp32: numpy's float32 exp)
    E = np.exp((S - max_all[:, None]).astype(np.float32)).astype(np.float32)
    temp1 = np.where(same & sel, E, np.float32(0)).astype(np.float32)
    temp2 = np.where(diff & sel, E, np.float32(0)).astype(np.float32)
    A = temp1.astype(np.float64).sum(axis=1).astype(np.float32)
    B = temp2.astype(np.float64).sum(axis=1).astype(np.float32)
    T = (A + B).astype(np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        logv = np.where((A == 0) | (T == 0), np.float32(0), np.log((A / T).astype(np.float32))).astype(np.float32)
    tops = np.zeros(5, dtype=np.float32)
    tops[0] = weighted_loss(logv, anchor_weight, Q)
    # .cu:173-206, :390-398
    klist = [1, 5, 10, 15]
    for t in range(max(0, num_tops - 2)):
        k = klist[t]
        hits = 0
        for i in range(Q):
            keep = notself[i]
            vals = np.sort(E[i][keep])[::-1]
            thr = vals[min(k, vals.size - 1)]
            if np.any(keep & (E[i] > thr) & eq[i]):
                hits += 1
        tops[1 + t] = np.float32(hits) / np.float32(Q)
    tops[num_tops - 1] = np.float32(np.abs(xl.astype(np.float64)).sum()) / np.float32(Q)  # .cu:400-401
    state = dict(S=S, E=E, sel=sel, temp1=temp1, temp2=temp2, A=A, B=B, T=T, posi_thr=posi, nega_thr=nega,
                 min_within=min_within, max_between=max_between, max_all=max_all,
                 ident_num=ident_num, diff_num=diff_num, logv=logv)
    return tops, state


def grad_weights(state, Q, loss_weight=1.0):
    """G = (lw/Q)(-W1+W2+W3) (.cu:405-460 folded), float64 for use as an independent check."""
    A = state["A"].astype(np.float64)[:, None]
    T = state["T"].astype(np.float64)[:, None]
    t1 = state["temp1"].astype(np.float64)
    t2 = state["temp2"].astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        W1 = np.where(A == 0, 0.0, t1 / A)
        W2 = np.where(T == 0, 0.0, t1 / T)
        W3 = np.where(T == 0, 0.0, t2 / T)
    return (np.float64(np.float32(loss_weight) / np.float32(Q))) * (-W1 + W2 + W3)


def step_world_fp64(x_total, label_total, Q, world, loss_weight=1.0, S_inject_all=None, anchor_weight=None, **kw):
    """Emulated multi-rank fwd+bwd: (tops[world,5], dX[N,D] in fp64, the ranks' forward states).  anchor_weight: the Q * world
    anchors' weights, each rank's G scaled by row.  Memory rows (world 1, rows [Q, N)) get the transposed term alone, 1/2 G[:, Q:]^T x
    (DESIGN 4.6)."""
    x_total = np.ascontiguousarray(x_total, dtype=np.float32)
    N, D = x_total.shape
    w = None if anchor_weight is None else np.asarray(anchor_weight, dtype=np.float32)
    tops = np.zeros((world, 5), dtype=np.float32)
    local = np.zeros((N, D), dtype=np.float64)
    total = np.zeros((N, D), dtype=np.float64)
    xd = x_total.astype(np.float64)
    states = []
    for r in range(world):
        rows = slice(r * Q, (r + 1) * Q)
        Sin = None if S_inject_all is None else S_inject_all[rows]
        wr = None if w is None else w[rows]
        tops[r], st = forward(x_total, label_total, Q, world, r, S_inject=Sin, anchor_weight=wr, **kw)
        G = grad_weights(st, Q, loss_weight)
        if wr is not None:
            G = G * wr.astype(np.float64)[:, None]
        local[rows] = G @ xd                                     # .cu:448-453
        total += G.T @ xd[rows]                                  # .cu:455-460 + all-reduce .cu:467
        states.append(st)
    dX = 0.5 * (total / world) + 0.5 * local                     # .cu:474, :492-497
    return tops, dX, states


def step_world(x_total, label_total, Q, world, loss_weight=1.0, S_inject_all=None, anchor_weight=None, **kw):
    """step_world_fp64 with the gradient rounded to fp32: (tops[world,5], dX[N,D])."""
    tops, dX, _ = step_world_fp64(x_total, label_total, Q, world, loss_weight, S_inject_all, anchor_weight, **kw)
    return tops, dX.astype(np.float32)
