"""fp64 reference of the layer's gradient and its componentwise magnitude, for the gradient precision tests.

The gradient weights G (Q x N) come from the oracle's forward state on the similarities the GPU computed (S injected), in fp64 by
npair_oracle_np.grad_weights.  Besides the gradient R, every form returns its magnitude B: the same expression with |G| and |X|, where
|G| = c (|W1| + |W2| + |W3|) is the magnitude of what the weight builder actually sums (a same-label weight c (W2 - W1) cancels), and
R32, the same gradient from the fp32-rounded weights through fp32 GEMMs (cuBLAS SGEMM with TF32 off when a GPU is present), the
precision of the reference layer's own engine.  The step forms (c = lw / Q):

    world 1             R = (1/2)(G X + G^T X)
    emulated world W    R[rank r rows] = (1/2) G_r X_total,  R += (1/2)(1/W) G_r^T X_r  for every rank r   (both exchange forms)
    cross-batch memory  R[0:Q] = (1/2)(G X_total + G[:, 0:Q]^T x),  R[Q:N] = (1/2) G[:, Q:]^T x   (the world-1 form over N = Q + m
                        rows: the memory rows are no anchors and get the transposed term alone, DESIGN 4.3, 4.6)

The checks of a gradient dx against them (violations):
    normwise       ||dx - R||     <= max(rel ||R||, k ||R32 - R||)
    per row        ||dx_i - R_i|| <= max(rel ||R_i||, k ||R32_i - R_i||)      (k = 2, more where SGEMM_FACTOR says why)
    componentwise  |dx - R|       <= tau B + TINY, elementwise
A normwise bound over the whole Q x D matrix cannot see an error confined to one weight, one K block or one split-K slice; the
componentwise bound can, since B is the sum of the magnitudes of the very terms that were added."""
from __future__ import annotations

import numpy as np

from npairloss_b200 import capi
from oracle import npair_oracle_np as onp

FP16X2, BF16X3, BF16 = capi.PREC_FP32_FP16X2, capi.PREC_FP32_BF16X3, capi.PREC_BF16
PASSES = {FP16X2: 3, BF16X3: 6, BF16: 1}      # MMA passes of a product of two split operands (mma_passes, kernels.cuh)
DEFAULT_CHUNK_COLS = 2048                     # the fused kernel's accumulation chunk when grad_chunk_cols is 0 (ctx.cu)


def tau(prec, path, N, chunk_cols=0):
    """The componentwise bound, as a fraction of B, of a gradient path over a K extent of N database columns.  A model of the tensor
    core's fp32 accumulator, which may truncate: about 2^-23 of the partial sum, hence of B, per k16 MMA, i.e. 2 passes L / 16 2^-24
    over an accumulation of L columns (the fused kernel's chunk; N on the split GEMM and on the SIMT path, whose fp32 FMAs round to
    nearest), plus 64 2^-24 for the operands' fp32-faithful splits, the chunk drains and alpha; bf16 pieces add 2^-8 per product
    (2^-7 here).  Largest ratios measured on an H100 80GB HBM3 (700 W) over test_gpu_grad_precision.py, in 2^-24 units of B (this
    bound in brackets):
      fp16x2 fused: 321 at N = 8192 in 2048-column chunks (832), 116 in 256-column chunks (160), on a cosine-0.9996 cone
      fp16x2 split: 1492 at N = 8192 (3136);  simt 33 (208)
      bf16x3 fused 57, split 35, simt 29 at N <= 1000 (814, 814, 352);  bf16 62517 (131072 + accumulation)
    The fp16x2 weights split without their 2^14 scale (weight_scale_log2) measured 1142 (fused, N = 8192), 330 (256-column chunks) and
    930 (memory step, N = 57856), above the fused kernel's bound; on the split GEMM the accumulator's share dominates either way (1511
    unscaled, 1492 scaled)."""
    L = N if path != "fused" else min(N, chunk_cols if chunk_cols > 0 else (N if chunk_cols < 0 else DEFAULT_CHUNK_COLS))
    units = 2 * PASSES[prec] * ((L + 15) // 16) + 64
    return units * U24 + (2.0 ** -7 if prec == BF16 else 0.0)


# The allowance of the normwise and per-row rules in multiples of the error of an fp32 SGEMM over the same weights: 2 on well-spread
# rows through the fused kernel and the SIMT path.  The split GEMM accumulates all N columns in one truncating fp32 accumulator, and
# on clustered rows every term of a row carries the same common direction, so that the accumulator's truncation bias does not cancel
# either.  Worst ratios measured on an H100 80GB HBM3 (700 W), with the weight scale (without it):
#   split GEMM, well-spread rows, N = 8192: normwise 70 (70), per row 9.5 (9.6); its normwise error there is 2.0e-5 .. 2.7e-5
#   clustered rows (cosine 0.99 .. 0.9996), every path: per row 93 (938 in the memory step at N = 57856)
SGEMM_FACTOR = {"spread": 2.0, "accumulator": 256.0}

U24 = 2.0 ** -24    # the componentwise ratios are reported in these units of B
TINY = 1e-30        # absolute floor of the componentwise rule: rows and columns with no selected pair must come out exactly 0


def cone_inputs(N, D, eps, seed, dup=0, all_equal=False):
    """N unit rows normalize(u + eps g / sqrt(D)) around one random unit u (pairwise cosine about 1 / (1 + eps^2)) and labels in pairs
    as synth.make_inputs.  dup > 1: rows come in groups of dup exact copies (a group holds dup / 2 classes), so that many similarities
    are bitwise equal and many pairs sit exactly at the mining thresholds.  all_equal: every row is u."""
    rng = np.random.default_rng(seed)
    u = rng.standard_normal(D)
    u /= np.linalg.norm(u)
    x = u[None, :] + (0.0 if all_equal else eps) * rng.standard_normal((N, D)) / np.sqrt(D)
    if dup > 1:
        x = x[np.arange(N) // dup * dup]
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    lab = (np.arange(N) // 2).astype(np.float32)
    return np.ascontiguousarray(x, dtype=np.float32), lab


def make_weights(n, rng, zeros=True):
    """Anchor weights in [0, 1] with exact 0, exact 1 and powers of two among uniform ones."""
    w = rng.random(n).astype(np.float32)
    k = np.arange(n)
    w[k % 5 == 1] = 1.0
    w[k % 5 == 2] = np.float32(2.0) ** -rng.integers(1, 12, size=int((k % 5 == 2).sum()))
    if zeros:
        w[k % 5 == 3] = 0.0
    return w


def weights(state, Q, loss_weight=1.0):
    """(G, |G|) of one rank's forward state, fp64: G = c (-W1 + W2 + W3) (npair_oracle_np.grad_weights), |G| = c (W1 + W2 + W3)."""
    A = state["A"].astype(np.float64)[:, None]
    T = state["T"].astype(np.float64)[:, None]
    t1 = state["temp1"].astype(np.float64)
    t2 = state["temp2"].astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        mag = np.where(A == 0, 0.0, t1 / A) + np.where(T == 0, 0.0, (t1 + t2) / T)
    return onp.grad_weights(state, Q, loss_weight), np.float64(np.float32(loss_weight) / np.float32(Q)) * mag


def unit_weights(state):
    """The weights before the factor c, as the weight builders form them: g' = -W1 + W2 + W3 (each |g'| <= 1 is the premise of the
    fp16x2 weight scale, weight_scale_log2 in kernels.cuh)."""
    return onp.grad_weights(state, 1, 1.0)


def _products(x, terms):
    """R, B and R32 of sum over terms (G, |G|, rows, a, t): out[rows] += a G X, and, when t != 0, out += t G^T X[rows]."""
    import torch
    dev = torch.device("cuda:0" if torch.cuda.is_available() else "cpu")

    def run(dtype, absval):
        X = torch.from_numpy(x).to(dev, dtype)
        X = X.abs() if absval else X
        out = torch.zeros_like(X)
        for G, Gabs, rows, a, t in terms:
            g = torch.from_numpy(Gabs if absval else G).to(dev, dtype)
            out[rows] += a * (g @ X)
            if t:
                out += t * (g.T @ X[rows])
        return out.to(torch.float64).cpu().numpy()

    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False       # R32: cuBLAS SGEMM, the reference layer's engine
    try:
        return dict(R=run(torch.float64, False), B=run(torch.float64, True), R32=run(torch.float32, False))
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old


def step(x_total, lab, Q, world, S, anchor_weight=None, loss_weight=1.0, **mining):
    """The emulated world-W step on the database x_total (the Q * world anchors, then at world 1 any memory rows), S the
    (Q * world) x N similarities of the anchors' rows (None: the oracle's own): dict(R, B, R32, G) over all N rows, so that rows
    [Q, N) are the memory rows' gradient.  anchor_weight: the Q * world anchors' weights, each rank's (G, |G|) scaled by row.
    G: the ranks' weights [(G, |G|)]."""
    x = np.ascontiguousarray(x_total, dtype=np.float32)
    w = None if anchor_weight is None else np.asarray(anchor_weight, dtype=np.float32).astype(np.float64)
    terms, Gs = [], []
    for r in range(world):
        rows = slice(r * Q, (r + 1) * Q)
        # num_tops = 2: no retrieval counters, which the gradient does not need and which cost a sort per row
        _, st = onp.forward(x, lab, Q, world, r, num_tops=2, S_inject=None if S is None else S[rows], **mining)
        G, Gabs = weights(st, Q, loss_weight)
        if w is not None:
            G, Gabs = G * w[rows, None], Gabs * w[rows, None]
        terms.append((G, Gabs, rows, 0.5, 0.5 / world))
        Gs.append((G, Gabs))
    out = _products(x, terms)
    out["G"] = Gs
    return out


def violations(dx, ref, tau, rel=1e-5, k_sgemm=2.0, floor=TINY, row_extra=0.0):
    """The rules of the module docstring that dx breaks (empty: it passes), and the measured quantities: normwise error, the worst row's
    error over its allowance (rel and k_sgemm times the SGEMM's error), and the largest |dx - R| / B in units of 2^-24.  floor: the
    componentwise rule's absolute floor (TINY, or an array broadcast against dx); row_extra: an allowance added to every row's."""
    dx = np.asarray(dx, dtype=np.float64)
    R, B, R32 = ref["R"], ref["B"], ref["R32"]
    e = dx - R
    bad = []
    nR, nE, n32 = np.linalg.norm(R), np.linalg.norm(e), np.linalg.norm(R32 - R)
    if not np.isfinite(dx).all():
        bad.append("non-finite gradient")
    if not nE <= max(rel * nR, k_sgemm * n32):
        bad.append(f"normwise {nE / max(nR, TINY):.3e} of |R| (allowed {max(rel * nR, k_sgemm * n32) / max(nR, TINY):.3e})")
    rR, rE, r32 = (np.linalg.norm(a, axis=1) for a in (R, e, R32 - R))
    allow = np.maximum(rel * rR, k_sgemm * r32) + row_extra + TINY
    row_ratio = rE / allow
    if not (row_ratio <= 1).all():
        i = int(np.nanargmax(row_ratio))
        bad.append(f"per row: {int((~(row_ratio <= 1)).sum())} rows, worst row {i} at {row_ratio[i]:.3g}x its allowance")
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.where(np.abs(e) <= TINY, 0.0, np.abs(e) / B)
    comp = float(np.nanmax(ratio)) / U24 if ratio.size else 0.0
    over = ~(np.abs(e) <= tau * B + floor)
    if over.any():
        i, j = np.unravel_index(int(np.argmax(np.where(over, ratio, -1.0))), e.shape)
        bad.append(f"componentwise: {int(over.sum())} elements, worst ({i}, {j}) at {comp:.1f} x 2^-24 of B (tau {tau / U24:.1f})")
    return bad, dict(normwise=nE / max(nR, TINY), sgemm=n32 / max(nR, TINY), row=float(np.nanmax(row_ratio)) if row_ratio.size else 0.0,
                     comp=comp)
