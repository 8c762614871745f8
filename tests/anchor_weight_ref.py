"""The weighted statement of the loss (DESIGN 4.5) over both oracle restatements, and the model of the weighted row record.

    loss     tops[0] = -(1/Q) sum_i w_i log(A_i / T_i)      (fp32 products w_i logv_i, summed in fp64 as the unweighted oracles do)
    gradient G_w = diag(w) G: anchor i's row of the gradient weights scaled by w_i, its transposed terms included
    the rest of the state (S, selects, A, T, logv, tops 1-4) does not depend on w

Each restatement gives a weighted statement of its own, and tests/test_anchor_weights_cpu.py compares the two.  The NumPy form scales
the rows of npair_oracle_np.grad_weights' fp64 G by w and multiplies out in fp64 (step_world_np).  The C++ form runs the C++ oracle's
own backward, npo_backward_partial (fp32 W1, W2, W3 and its own GEMMs), on a state whose selected terms temp1 / temp2 carry w per
anchor row, then npo_step_world's all-reduce and blend (step_world_cpp).  With w = None or w = 1 each is its unweighted oracle bit for
bit.
"""
from __future__ import annotations

import numpy as np

from oracle import npair_oracle_np as onp


def weighted_loss(logv, w, Z):
    """-(1/Z) sum_i w_i logv_i in the oracles' arithmetic (w None: the unweighted loss)."""
    lv = np.asarray(logv, dtype=np.float32)
    if w is not None:                                         # a row with w = 0 adds nothing, whatever its log value
        w = np.asarray(w, dtype=np.float32)
        with np.errstate(invalid="ignore"):
            lv = np.where(w == 0, np.float32(0), lv * w).astype(np.float32)
    return np.float32(np.float32(lv.astype(np.float64).sum()) / np.float32(-Z))


def grad_weights(state, Q, w, loss_weight=1.0):
    """The NumPy oracle's fp64 gradient weights with anchor row i scaled by w_i."""
    G = onp.grad_weights(state, Q, loss_weight)
    return G if w is None else G * np.asarray(w, dtype=np.float32).astype(np.float64)[:, None]


def _step(forward_rank, x_total, Q, world, w, loss_weight):
    """(tops[world, 5], dX[N, D]) in the NumPy oracle's blend (.cu:474, :492-497); forward_rank(r) -> (tops, state)."""
    x_total = np.ascontiguousarray(x_total, dtype=np.float32)
    N, D = x_total.shape
    tops = np.zeros((world, 5), dtype=np.float32)
    local = np.zeros((N, D), dtype=np.float64)
    total = np.zeros((N, D), dtype=np.float64)
    xd = x_total.astype(np.float64)
    for r in range(world):
        t, st = forward_rank(r)
        wr = None if w is None else np.asarray(w, dtype=np.float32)[r * Q:(r + 1) * Q]
        tops[r] = t
        tops[r, 0] = weighted_loss(st["logv"], wr, Q)
        G = grad_weights(st, Q, wr, loss_weight)
        local[r * Q:(r + 1) * Q] = G @ xd
        total += G.T @ xd[r * Q:(r + 1) * Q]
    dX = 0.5 * (total / world) + 0.5 * local
    return tops, dX.astype(np.float32)


def step_world_np(x_total, label_total, Q, world, w=None, loss_weight=1.0, S_inject_all=None, **kw):
    """The weighted NumPy oracle: npair_oracle_np.step_world with anchor weights w[N] (None: that function's results, bit for bit)."""
    def fwd(r):
        Sin = None if S_inject_all is None else S_inject_all[r * Q:(r + 1) * Q]
        return onp.forward(x_total, label_total, Q, world, r, S_inject=Sin, **kw)
    return _step(fwd, x_total, Q, world, w, loss_weight)


def step_world_cpp(oracle_lib, x_total, label_total, Q, world, w=None, loss_weight=1.0, S_inject_all=None, **kw):
    """The weighted statement through the C++ oracle: its forward (npo_forward) per rank, and its own backward (npo_backward_partial,
    fp32 W1..W3 and GEMMs) on that rank's state with anchor row i of the selected terms temp1 / temp2 scaled by w_i -- which scales
    W1, W2, W3 and so G by w_i -- then npo_step_world's fp32 all-reduce and blend.  w = None or 1: oracle_lib.step_world bit for bit.
    kw: oracle_lib.make_config's fields."""
    import ctypes as C
    L = oracle_lib.lib()
    x_total = np.ascontiguousarray(x_total, dtype=np.float32)
    N, D = x_total.shape
    wv = None if w is None else np.asarray(w, dtype=np.float32)
    tops = np.zeros((world, 5), dtype=np.float32)
    local = np.zeros((N, D), dtype=np.float32)
    total = np.zeros((N, D), dtype=np.float32)
    fp = C.POINTER(C.c_float)
    for r in range(world):
        cfg = oracle_lib.make_config(Q, D, world=world, rank=r, **kw)
        Sin = None if S_inject_all is None else S_inject_all[r * Q:(r + 1) * Q]
        t, st = oracle_lib.forward(x_total, label_total, cfg, S_inject=Sin)
        wr = None if wv is None else wv[r * Q:(r + 1) * Q]
        tops[r] = t
        tops[r, 0] = weighted_loss(st["logv"], wr, Q)
        if wr is not None:                                    # views into the state buffer the C++ backward reads
            st["temp1"][:] = (st["temp1"] * wr[:, None]).astype(np.float32)
            st["temp2"][:] = (st["temp2"] * wr[:, None]).astype(np.float32)
        lh = np.zeros((Q, D), dtype=np.float32)
        th = np.zeros((N, D), dtype=np.float32)
        e = L.npo_backward_partial(C.byref(cfg), x_total.ctypes.data_as(fp), C.byref(st["_st"]), C.c_float(loss_weight),
                                   lh.ctypes.data_as(fp), th.ctypes.data_as(fp))
        if e:
            raise oracle_lib.OracleError(e)
        local[r * Q:(r + 1) * Q] = lh
        total += th                                           # the all-reduce, in rank order
    td = total * np.float32(np.float32(1.0) / np.float32(world))
    return tops, (np.float32(0.5) * td + np.float32(0.5) * local).astype(np.float32)


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


def make_weights(n, rng, zeros=True):
    """Weights in [0, 1] with exact 0, exact 1 and powers of two among uniform ones."""
    w = rng.random(n).astype(np.float32)
    k = np.arange(n)
    w[k % 5 == 1] = 1.0
    w[k % 5 == 2] = np.float32(2.0) ** -rng.integers(1, 12, size=int((k % 5 == 2).sum()))
    if zeros:
        w[k % 5 == 3] = 0.0
    return w



def grad_ref_step_world(x, lab, Q, world, S_all, w, loss_weight=1.0, **mining):
    """grad_ref.step_world with anchor weights w[N]: every rank's (G, |G|) with row i scaled by w_i (dict(R, B, R32, G))."""
    import grad_ref
    x = np.ascontiguousarray(x, dtype=np.float32)
    w64 = np.asarray(w, dtype=np.float32).astype(np.float64)
    terms, Gs = [], []
    for r in range(world):
        G, Gabs = grad_ref.weights(grad_ref._forward(x, lab, Q, world, r, S_all[r * Q:(r + 1) * Q], mining), Q, loss_weight)
        wr = w64[r * Q:(r + 1) * Q, None]
        G, Gabs = G * wr, Gabs * wr
        terms.append((G, Gabs, slice(r * Q, (r + 1) * Q), 0.5, 0.5 / world))
        Gs.append((G, Gabs))
    out = grad_ref._products(x, terms)
    out["G"] = Gs
    return out


def grad_ref_step_memory(x, lab, x_mem, lab_mem, S, w, loss_weight=1.0, **mining):
    """grad_ref.step_memory with the Q current rows' anchor weights w[Q] (the memory rows are no anchors)."""
    import grad_ref
    import memory_ref
    _, st = memory_ref.forward_memory(x, lab, x_mem, lab_mem, num_tops=2, S_inject=S, **mining)
    Q = np.asarray(x).shape[0]
    G, Gabs = grad_ref.weights(st, Q, loss_weight)
    wr = np.asarray(w, dtype=np.float32).astype(np.float64)[:, None]
    G, Gabs = G * wr, Gabs * wr
    xt = np.ascontiguousarray(st["x_total"], dtype=np.float32)
    out = grad_ref._products(xt, [(G, Gabs, slice(0, Q), 0.5, 0.0)])
    tr = grad_ref._products(np.ascontiguousarray(xt[:Q]), [(np.ascontiguousarray(G[:, :Q].T), np.ascontiguousarray(Gabs[:, :Q].T),
                                                            slice(0, Q), 0.5, 0.0)])
    res = {k: out[k][:Q] + tr[k] for k in ("R", "B", "R32")}
    res["G"] = [(G, Gabs)]
    return res
