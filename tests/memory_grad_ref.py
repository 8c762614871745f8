"""NumPy statement of the memory rows' gradient of a cross-batch memory step (DESIGN 4.6), for the tests: with G the anchors' weights
of the step (memory_ref.forward_memory, npair_oracle_np.grad_weights; anchor row i scaled by its weight w_i),

    d_mem_diff = (1/2) G[:, Q:]^T . x          (m x D; x the Q anchors as the layer reads them)

which is half the analytic gradient of the step's loss with respect to the memory rows y.  At m = (W - 1) Q it is W d_total_half[Q:]
of rank 0 of a world-W step on [x; y]."""
from __future__ import annotations

import numpy as np

import grad_ref
import memory_ref


def weights(x, l, y, ly, S=None, w=None, loss_weight=1.0, **mining):
    """(G, |G|) of the step, fp64 [Q, Q + m], anchor row i scaled by w_i (w None: unweighted)."""
    _, st = memory_ref.forward_memory(x, l, y, ly, num_tops=2, S_inject=S, **mining)
    G, Gabs = grad_ref.weights(st, np.asarray(x).shape[0], loss_weight)
    if w is not None:
        wr = np.asarray(w, dtype=np.float32).astype(np.float64)[:, None]
        G, Gabs = G * wr, Gabs * wr
    return G, Gabs


def mem_grad(x, l, y, ly, S=None, w=None, loss_weight=1.0, **mining):
    """d_mem_diff in fp64 [m, D]."""
    G, _ = weights(x, l, y, ly, S, w, loss_weight, **mining)
    Q = np.asarray(x).shape[0]
    return 0.5 * (G[:, Q:].T @ np.asarray(x, dtype=np.float64))


def mem_grad_products(x, l, y, ly, S=None, w=None, loss_weight=1.0, **mining):
    """dict(R, B, R32) of d_mem_diff for grad_ref.violations: the fp64 product, its magnitude (1/2)|G[:, Q:]|^T |x| and the fp32 SGEMM
    of the same weights (on the GPU when there is one, as grad_ref's products)."""
    import torch
    G, Gabs = weights(x, l, y, ly, S, w, loss_weight, **mining)
    Q = np.asarray(x).shape[0]
    dev = torch.device("cuda:0" if torch.cuda.is_available() else "cpu")
    X = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(dev)

    def run(g, dtype, xx):
        return (0.5 * (torch.from_numpy(np.ascontiguousarray(g[:, Q:].T)).to(dev, dtype) @ xx.to(dtype))).to(torch.float64).cpu().numpy()

    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        return dict(R=run(G, torch.float64, X), B=run(Gabs, torch.float64, X.abs()), R32=run(G, torch.float32, X))
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old


def loss(x, l, y, ly, w=None, **mining):
    """The step's loss in fp64 as a function of the memory rows y (S = x . [x; y]^T in fp64, the forward's selections and maxima
    evaluated in fp64 too): what finite differences with respect to y differentiate.  Weighted: -(1/Q) sum_i w_i log(A_i / T_i)."""
    x = np.asarray(x, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    Q = x.shape[0]
    _, st = memory_ref.forward_memory(x.astype(np.float32), l, y.astype(np.float32), ly, num_tops=2, **mining)
    sel1 = st["temp1"] > 0                                      # the forward's selections, held fixed
    sel2 = st["temp2"] > 0
    S = x @ np.concatenate([x, y]).T
    E = np.exp(S - st["max_all"].astype(np.float64)[:, None])
    A = np.where(sel1, E, 0.0).sum(axis=1)
    T = A + np.where(sel2, E, 0.0).sum(axis=1)
    with np.errstate(divide="ignore", invalid="ignore"):
        lv = np.where(A > 0, np.log(A / T), 0.0)
    wv = np.ones(Q) if w is None else np.asarray(w, dtype=np.float64)
    return -(wv * lv).sum() / Q

