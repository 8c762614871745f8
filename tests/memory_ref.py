"""NumPy statement of the layer step with a cross-batch memory (DESIGN 4.3), for the tests: the reference's rank-0 block over the
database [x; x_mem] of N = Q + m rows, whose anchors are the Q current rows.  It follows oracle/npair_oracle_np.forward rule for rule,
with N = Q + m columns in place of Q * world, and the backward of the world-1 blend with the transposed term restricted to the anchors'
columns and not divided by anything:

    dx = (1/2)(lw/Q)(G . X_total + G[:, 0:Q]^T . x)

At m = (W - 1) Q this is rank 0 of a world-W step on [x; x_mem]: the same tops, and the gradient d_local_half + W d_total_half[0:Q]."""
from __future__ import annotations

import numpy as np

from oracle import npair_oracle_np as onp

LOCAL, GLOBAL = onp.LOCAL, onp.GLOBAL
FLT_MAX = onp.FLT_MAX


def forward_memory(x, l, x_mem, l_mem, num_tops=5, margin_ident=0.0, margin_diff=0.0, identsn=-1.0, diffsn=-1.0, ap_region=LOCAL,
                   ap_method=onp.RAND, an_region=LOCAL, an_method=onp.RAND, S_inject=None):
    """(tops[5], state) of the step's forward; S_inject: the Q x (Q + m) similarities to use instead of x . X_total^T."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    Q = x.shape[0]
    xm = np.ascontiguousarray(x_mem, dtype=np.float32).reshape(-1, x.shape[1])
    x_total = np.concatenate([x, xm])
    ll = np.ascontiguousarray(l, dtype=np.float32)
    lab = np.concatenate([ll, np.ascontiguousarray(l_mem, dtype=np.float32).reshape(-1)])
    N = x_total.shape[0]
    if S_inject is None:
        S = (x.astype(np.float64) @ x_total.astype(np.float64).T).astype(np.float32)
    else:
        S = np.ascontiguousarray(S_inject, dtype=np.float32).reshape(Q, N).copy()
    notself = np.arange(Q)[:, None] != np.arange(N)[None, :]
    eq = ll[:, None] == lab[None, :]
    same = notself & eq
    diff = notself & ~eq
    min_within = np.where(same, S, FLT_MAX).min(axis=1).astype(np.float32)
    max_between = np.where(diff, S, -FLT_MAX).max(axis=1).astype(np.float32)
    max_all = np.where(notself, S, -FLT_MAX).max(axis=1).astype(np.float32)
    rel = (onp.RELATIVE_HARD, onp.RELATIVE_EASY)
    if ap_region == LOCAL:
        posi = max_between.copy() if ap_method not in rel else \
            np.array([onp._thr_from_sorted(np.sort(S[i][same[i]]), identsn) for i in range(Q)], dtype=np.float32)
    else:
        if ap_method not in rel:
            if not diff.any():
                raise onp.OracleError("empty list")
            posi = np.full(Q, S[diff].max(), dtype=np.float32)
        else:
            posi = np.full(Q, onp._thr_from_sorted(np.sort(S[same]), identsn), dtype=np.float32)
    if an_region == LOCAL:
        nega = min_within.copy() if an_method not in rel else \
            np.array([onp._thr_from_sorted(np.sort(S[i][diff[i]]), diffsn) for i in range(Q)], dtype=np.float32)
    else:
        if an_method not in rel:
            if not same.any():
                raise onp.OracleError("empty list")
            nega = np.full(Q, S[same].min(), dtype=np.float32)
        else:
            nega = np.full(Q, onp._thr_from_sorted(np.sort(S[diff]), diffsn), dtype=np.float32)
    tp = (posi + np.float32(margin_ident)).astype(np.float32)[:, None]
    tn = (nega + np.float32(margin_diff)).astype(np.float32)[:, None]
    ap_rule = {onp.HARD: S < tp, onp.EASY: S >= tp, onp.RAND: np.ones_like(same), onp.RELATIVE_HARD: S <= tp,
               onp.RELATIVE_EASY: S >= tp}[ap_method]
    an_rule = {onp.HARD: S > tn, onp.EASY: S <= tn, onp.RAND: np.ones_like(same), onp.RELATIVE_HARD: S >= tn,
               onp.RELATIVE_EASY: S <= tn}[an_method]
    sel = (same & ap_rule) | (diff & an_rule)
    E = np.exp((S - max_all[:, None]).astype(np.float32)).astype(np.float32)
    temp1 = np.where(same & sel, E, np.float32(0)).astype(np.float32)
    temp2 = np.where(diff & sel, E, np.float32(0)).astype(np.float32)
    A = temp1.astype(np.float64).sum(axis=1).astype(np.float32)
    B = temp2.astype(np.float64).sum(axis=1).astype(np.float32)
    T = (A + B).astype(np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        logv = np.where((A == 0) | (T == 0), np.float32(0), np.log((A / T).astype(np.float32))).astype(np.float32)
    tops = np.zeros(5, dtype=np.float32)
    tops[0] = np.float32(np.float32(logv.astype(np.float64).sum()) / np.float32(-Q))
    klist = [1, 5, 10, 15]
    for t in range(max(0, num_tops - 2)):
        k, hits = klist[t], 0
        for i in range(Q):
            vals = np.sort(E[i][notself[i]])[::-1]
            thr = vals[min(k, vals.size - 1)]
            if np.any(notself[i] & (E[i] > thr) & eq[i]):
                hits += 1
        tops[1 + t] = np.float32(hits) / np.float32(Q)
    tops[num_tops - 1] = np.float32(np.abs(x.astype(np.float64)).sum()) / np.float32(Q)
    state = dict(S=S, A=A, B=B, T=T, temp1=temp1, temp2=temp2, posi_thr=posi, nega_thr=nega, min_within=min_within,
                 max_between=max_between, max_all=max_all, x_total=x_total)
    return tops, state


def step_memory(x, l, x_mem, l_mem, loss_weight=1.0, S_inject=None, **mining):
    """(tops[5], dx[Q, D] float64, state): the forward and the gradient of the current rows (the memory rows get none)."""
    tops, st = forward_memory(x, l, x_mem, l_mem, S_inject=S_inject, **mining)
    Q = np.asarray(x).shape[0]
    G = onp.grad_weights(st, Q, loss_weight)
    xt = st["x_total"].astype(np.float64)
    dx = 0.5 * (G @ xt + G[:, :Q].T @ xt[:Q])
    return tops, dx, st
