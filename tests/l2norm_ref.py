"""fp64 reference of the L2Normalize producer (l2norm_fwd_kernel / l2norm_bwd_kernel) and its componentwise rules.

The layer:  y = x / ||x||,  inv = 1 / ||x||,  dx = (dy - y (y . dy)) inv.  Besides the values, the reference returns their magnitudes, so
that every rule is componentwise:

    forward    |y - y64|     <= tau_f(D) |y64|   + FLOOR     y64 = x / ||x||, inv64 = 1 / ||x||, from x in fp64
               |inv - inv64| <= tau_f(D) inv64   + FLOOR
    backward   |dx - dx64|   <= tau_b(D) B       + FLOOR     dx64 from the kernel's own fp32 y, inv and dy, in fp64 (this isolates
                                                             the backward kernel); B = (|dy| + |y| (|y| . |dy|)) inv
    chain      |dx - J^T dy| <= tau_c(D) B       + FLOOR     the fused layer x -> y -> dx against the exact Jacobian of x / ||x||

Where the bounds come from.  The kernel gives each row to one warp.  Lane l accumulates its partial sum of squares with fmaf in a fixed
order: n(D) = ceil(D / 128) * 4 terms (D % 4 == 0: quads of 4 features at 4 l, 4 l + 128, ...) or ceil(D / 32) terms (otherwise:
features l, l + 32, ...); then a 5-level xor shuffle tree adds the 32 partials.  Every term is >= 0, so the sum carries at most
(n + 5) u of relative error (u = 2^-24, one rounding per fmaf and per tree level).  sqrtf halves that and adds u; the division x / nrm
(and 1 / nrm) adds u:  tau_f = ((n + 5) / 2 + 2) u.  The fast path accepts ss only in [2^-64, FLT_MAX]; there at most D partial sums
round in the subnormal range, 2^-150 each, which is D 2^-86 of ss at most (the D 2^-62 u term).  A row outside that range is redone
on x 2^-e (pre_scale's clamp of the exponent of max|x|), which is exact except where x 2^-e or the result is subnormal, which the
absolute FLOOR = 2^-149 covers (one rounding in the subnormal range of the input, one of the output).
The backward's dot has the same order: (n + 5) u of sum |y| |dy|; it enters dx times |y| inv.  dy - y dot is one fused multiply-add
(one rounding of |t| <= |dy| + |y| |dot|) and the product with inv one more:  tau_b = (n + 8) u, with one u of slack.
The chain: y's error tau_f |y| enters dx through dy - y (y . dy) twice (as y and inside the dot), and the stored inv once:
tau_c = tau_b + 3 tau_f.

Non-finite inputs: a row with any NaN or +-inf element gives an all-NaN y row and a NaN inv, and its backward is NaN; the other rows
are bit for bit unchanged.  A zero row gives y = 0, inv = 0 and dx = 0.  Where 1 / ||x|| > FLT_MAX (||x|| < 2^-128) inv is +inf and
dx is +-inf, or exactly 0 where dy - y (y . dy) is 0, never NaN.

Largest ratios measured on an H100 80GB HBM3 (700 W) over test_gpu_l2norm_precision.py, as a fraction of each bound: MEASURED.
The fp32 emulation's adversarial rows (test_l2norm_ref_cpu.py) reach more than half of tau_f and tau_b as well."""
from __future__ import annotations

import numpy as np

F32, F64 = np.float32, np.float64
U = 2.0 ** -24
FLOOR = 2.0 ** -149
FLT_MAX = float(np.finfo(np.float32).max)
SS_MIN = 2.0 ** -64            # the fast path's lower limit on the sum of squares (L2_SS_MIN, kernels.cu)

# largest |error| / bound over test_gpu_l2norm_precision.py::test_componentwise_every_path, as that test prints them (L2NORM_RATIO) on
# an H100 80GB HBM3 (700 W).  The same test holds the kernels to emulate_forward / emulate_backward bit for bit, so the emulation on
# the CPU gives these ratios to the last digit as well.
MEASURED = {"y": 0.519, "inv": 0.476, "dx": 0.493, "chain": 0.693}


def terms_per_lane(D: int) -> int:
    """n(D): the fmaf terms of one lane's partial sum (the quad path when D % 4 == 0, the scalar path otherwise)."""
    return (D + 127) // 128 * 4 if D % 4 == 0 else (D + 31) // 32


def tau_f(D: int) -> float:
    n = terms_per_lane(D)
    return ((n + 5) / 2 + 2 + D * 2.0 ** -62) * U


def tau_b(D: int) -> float:
    return (terms_per_lane(D) + 8) * U


def tau_c(D: int) -> float:
    return tau_b(D) + 3 * tau_f(D)


def _bad_rows(a):
    return ~np.isfinite(a).all(axis=1)


def forward(x):
    """(y64, inv64) of fp32 rows x, in fp64; NaN rows for non-finite input, zeros for zero rows."""
    x64 = np.asarray(x, dtype=np.float32).astype(np.float64)
    bad = _bad_rows(x64)
    xs = np.where(bad[:, None], 0.0, x64)
    nrm = np.sqrt(np.einsum("ij,ij->i", xs, xs))           # fp64 holds every fp32 square: no overflow, no underflow
    with np.errstate(divide="ignore", invalid="ignore"):
        y = np.where(nrm[:, None] > 0, xs / np.where(nrm > 0, nrm, 1.0)[:, None], 0.0)
        inv = np.where(nrm > 0, 1.0 / np.where(nrm > 0, nrm, 1.0), 0.0)
    y[bad] = np.nan
    inv[bad] = np.nan
    return y, inv


def backward(y, inv, dy):
    """(dx64, B, t64) from the kernel's fp32 y, inv and dy: dx64 = t64 inv with t64 = dy - y (y . dy), and B its magnitude."""
    y64 = np.asarray(y, np.float32).astype(np.float64)
    dy64 = np.asarray(dy, np.float32).astype(np.float64)
    inv64 = np.asarray(inv, np.float32).astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        dot = np.einsum("ij,ij->i", y64, dy64)
        t = dy64 - y64 * dot[:, None]
        mag = np.abs(dy64) + np.abs(y64) * np.einsum("ij,ij->i", np.abs(y64), np.abs(dy64))[:, None]
        dx = np.where((t == 0) & (inv64[:, None] == np.inf), 0.0, t * inv64[:, None])
        B = mag * inv64[:, None]
    return dx, B, t


def chain(x, dy):
    """(J^T dy, B) of the exact Jacobian of x / ||x|| at fp32 rows x (finite, non-zero rows), in fp64."""
    y, inv = forward(x)
    dy64 = np.asarray(dy, np.float32).astype(np.float64)
    dot = np.einsum("ij,ij->i", y, dy64)
    g = (dy64 - y * dot[:, None]) * inv[:, None]
    B = (np.abs(dy64) + np.abs(y) * np.einsum("ij,ij->i", np.abs(y), np.abs(dy64))[:, None]) * inv[:, None]
    return g, B


def _err(got, want, tau):
    """|got - want|, 0 where got is the fp32 overflow (+-inf) of a want within tau of FLT_MAX or beyond."""
    with np.errstate(invalid="ignore", over="ignore"):
        e = np.abs(got - want)
        return np.where(np.isinf(got) & (np.sign(got) == np.sign(want)) & (np.abs(want) * (1 + tau) >= FLT_MAX), 0.0, e)


def _ratio(err, bound):
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(bound > 0, err / bound, np.where(err > 0, np.inf, 0.0))


def check_forward(x, y, inv):
    """Violations of the forward rules (a list of strings) and the largest ratios err / bound of y and inv."""
    x = np.asarray(x, np.float32)
    y = np.asarray(y, np.float32)
    inv = np.asarray(inv, np.float32)
    R, D = x.shape
    out, t = [], tau_f(D)
    y64, inv64 = forward(x)
    bad = _bad_rows(x)
    if bad.any():
        if not np.isnan(y[bad]).all() or not np.isnan(inv[bad]).all():
            out.append(f"non-finite rows {np.flatnonzero(bad)[:8]}: y and inv must be NaN")
    ok = ~bad
    yo, y6 = y[ok].astype(np.float64), y64[ok]
    if not np.isfinite(yo).all():
        out.append("finite rows gave a non-finite y")
    ry = _ratio(np.abs(yo - y6), t * np.abs(y6) + FLOOR)
    io, i6 = inv[ok].astype(np.float64), inv64[ok]
    huge = i6 * (1 - t) > FLT_MAX                         # 1 / ||x|| beyond FLT_MAX: inv must be +inf
    near = (i6 * (1 + t) > FLT_MAX) & ~huge               # the rounding may go either way
    if (io[huge] != np.inf).any():
        out.append(f"inv of rows with 1/||x|| > FLT_MAX must be +inf, got {io[huge][io[huge] != np.inf][:4]}")
    fin = ~huge & ~(near & np.isinf(io))
    ri = _ratio(np.abs(io[fin] - i6[fin]), t * i6[fin] + FLOOR)
    my = float(np.nanmax(ry)) if ry.size else 0.0
    mi = float(np.nanmax(ri)) if ri.size else 0.0
    if not my <= 1.0:
        r, d = np.unravel_index(int(np.nanargmax(ry)), ry.shape)
        out.append(f"y: ratio {my:.3g} at row {np.flatnonzero(ok)[r]} col {d}: {yo[r, d]!r} vs {y6[r, d]!r}")
    if not mi <= 1.0:
        r = int(np.nanargmax(ri))
        out.append(f"inv: ratio {mi:.3g} at row {np.flatnonzero(ok)[fin][r]}: {io[fin][r]!r} vs {i6[fin][r]!r}")
    return out, {"y": my, "inv": mi}


def check_backward(y, inv, dy, dx, tau=None):
    """Violations of the backward rule (dx64 from the kernel's own y, inv, dy) and the largest ratio err / bound."""
    y = np.asarray(y, np.float32)
    dx = np.asarray(dx, np.float32).astype(np.float64)
    R, D = y.shape
    t = tau_b(D) if tau is None else tau
    dx64, B, t64 = backward(y, inv, dy)
    inv = np.asarray(inv, np.float32)
    out = []
    nanrow = np.isnan(inv) | _bad_rows(y)
    if nanrow.any() and not np.isnan(dx[nanrow]).all():
        out.append(f"rows with a NaN y or inv must give a NaN dx: rows {np.flatnonzero(nanrow)[:8]}")
    infrow = np.isinf(inv) & ~nanrow
    if infrow.any():
        d = dx[infrow]
        if np.isnan(d).any() or not ((d == 0) | np.isinf(d)).all():
            out.append(f"rows with inv = +inf must give dx in {{0, +-inf}}: rows {np.flatnonzero(infrow)[:8]}")
        tt = t64[infrow]
        yi, gi = y[infrow].astype(np.float64), np.asarray(dy, np.float32)[infrow].astype(np.float64)
        m0 = np.abs(gi) + np.abs(yi) * np.einsum("ij,ij->i", np.abs(yi), np.abs(gi))[:, None]
        sure = np.abs(tt) > t * m0                          # the sign of t is certain where |t| exceeds its error bound
        if (np.sign(d[sure]) != np.sign(tt[sure])).any():
            out.append("rows with inv = +inf: dx has the wrong sign")
    ok = ~nanrow & ~infrow
    r = _ratio(_err(dx[ok], dx64[ok], t), t * B[ok] + FLOOR)
    m = float(np.nanmax(r)) if r.size else 0.0
    if not m <= 1.0:
        i, j = np.unravel_index(int(np.nanargmax(r)), r.shape)
        out.append(f"dx: ratio {m:.3g} at row {np.flatnonzero(ok)[i]} col {j}: {dx[ok][i, j]!r} vs {dx64[ok][i, j]!r}")
    return out, m


def check_chain(x, dy, dx):
    """Violations of the composed rule (the fused layer's dx against the exact Jacobian) on finite non-zero rows, and the ratio."""
    x = np.asarray(x, np.float32)
    D = x.shape[1]
    g, B = chain(x, dy)
    inv64 = forward(x)[1]
    ok = np.isfinite(x).all(axis=1) & (np.abs(x).max(axis=1) > 0) & (inv64 * (1 + tau_f(D)) < FLT_MAX)   # inv finite in fp32
    dx = np.asarray(dx, np.float32).astype(np.float64)
    r = _ratio(_err(dx[ok], g[ok], tau_c(D)), tau_c(D) * B[ok] + FLOOR)
    m = float(np.nanmax(r)) if r.size else 0.0
    return ([] if m <= 1.0 else [f"chain: ratio {m:.3g}"]), m


# ----------------------------------------------------------------------------------------------- fp32 emulation of the kernels' order
# Lane partial sums by fmaf in the documented order, the 5-level xor shuffle tree, sqrtf, IEEE division, the rescued pass on x 2^-e:
# l2norm_fwd_kernel / l2norm_bwd_kernel give these bits.  `fault` plants one mistake (test_l2norm_ref_cpu.py).
def _fma(a, b, c):
    """fmaf(a, b, c) elementwise, rounded once: the fp64 product of two fp32 values is exact; s = fl64(p + c) and its error e (TwoSum)
    give the fp32 rounding of p + c, except where s is an fp32 midpoint and e != 0, where the exact sum lies on the side of e."""
    p, c = a.astype(F64) * b.astype(F64), c.astype(F64)
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    r = s.astype(F32)
    toward = np.nextafter(r, np.where(s > r.astype(F64), F32(np.inf), F32(-np.inf)).astype(F32))
    mid = (s != r.astype(F64)) & (s == (r.astype(F64) + toward.astype(F64)) / 2)
    fix = mid & (e != 0)
    # at a midpoint s, ties-to-even picked r or toward; the exact sum s + e lies on one side: take the neighbour on that side
    lo, hi = np.minimum(r, toward), np.maximum(r, toward)
    r = np.where(fix, np.where(e > 0, hi, lo), r)
    return r.astype(F32)


def _lane_order(D, fault=None):
    """(32, n) feature indices each lane visits in order (-1: none), on the quad (D % 4 == 0) or the scalar path."""
    if D % 4 == 0:
        lanes = [[d + e for d in range(4 * l, D, 128) for e in range(4)] for l in range(32)]
        if fault == "drop_last_quad" and D % 128:
            lanes = [o[:-4] if len(o) == 4 * ((D + 127) // 128) else o for o in lanes]
    else:
        lanes = [list(range(l, D, 32)) for l in range(32)]
        if fault == "scalar_reads_d_plus_1":
            lanes = [[d + 1 for d in o] for o in lanes]
    n = max(len(o) for o in lanes)
    return np.array([o + [-1] * (n - len(o)) for o in lanes], dtype=np.int64)


def _warp_sum(p, fault=None):
    lane = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        if fault == "skip_shuffle_level" and o == 4:
            continue
        p = (p + p[:, lane ^ o]).astype(F32)
    return p[:, 0]


def _row_dot(a, b, fault=None):
    R, D = a.shape
    idx = _lane_order(D, fault)
    ap = np.concatenate([a, np.zeros((R, 1), F32)], axis=1)       # index D (and -1) read as 0
    bp = np.concatenate([b, np.zeros((R, 1), F32)], axis=1)
    idx = np.where(idx < 0, D, np.minimum(idx, D))
    p = np.zeros((R, 32), F32)
    for k in range(idx.shape[1]):
        if fault == "dot_missing_quad" and k < 4:
            kk = idx[:, k].copy(); kk[0] = D                     # lane 0's first quad (features 0..3) left out
            p = _fma(ap[:, kk], bp[:, kk], p)
        else:
            p = _fma(ap[:, idx[:, k]], bp[:, idx[:, k]], p)
    return _warp_sum(p, fault)


def _pre_scale(mx):
    e = np.frexp(mx.astype(F64))[1]
    e = np.clip(e, -126, 127)
    return np.ldexp(np.ones_like(mx, F32), -e).astype(F32)


def emulate_forward(x, fault=None):
    """(y, inv) of the kernel's order in fp32; `fault` plants one mistake."""
    x = np.asarray(x, F32)
    R, D = x.shape
    with np.errstate(all="ignore"):
        ss = _row_dot(x, x, fault)
        fast = (ss >= F32(SS_MIN)) & (ss <= F32(FLT_MAX))
        if fault == "no_rescue":
            fast = np.ones(R, bool)
        nrm = np.sqrt(ss)
        y = np.zeros_like(x)
        inv = np.zeros(R, F32)
        nb = nrm[np.arange(R) ^ 1 if R % 2 == 0 else np.arange(R)] if fault == "neighbour_norm" else nrm
        f = fast
        y[f] = np.where(nrm[f, None] > 0, x[f] / nb[f, None], F32(0))        # (nrm > 0: the parent's guard, for "no_rescue")
        inv[f] = np.where(nrm[f] > 0, F32(1) / nrm[f], F32(0))
        s = ~fast
        if s.any():
            xs = x[s]
            mx = np.fmax.reduce(np.abs(xs), axis=1)
            nonfinite = np.isnan(ss[s]) | ~(mx <= F32(FLT_MAX))
            zero = (mx == 0) & ~nonfinite
            sc = _pre_scale(np.where(nonfinite | zero, F32(1), mx))
            xsc = (xs * sc[:, None]).astype(F32)
            n2 = np.sqrt(_row_dot(xsc, xsc, fault))
            ys = (xsc / n2[:, None]).astype(F32) if fault != "rescue_scales_ss_only" else (xs / n2[:, None]).astype(F32)
            invs = ((F32(1) / n2) * sc).astype(F32)
            ys[zero], invs[zero] = 0, 0
            ys[nonfinite], invs[nonfinite] = np.nan, np.nan
            y[s], inv[s] = ys, invs
    return y, inv


def emulate_backward(y, inv, dy, fault=None):
    y, dy, inv = np.asarray(y, F32), np.asarray(dy, F32), np.asarray(inv, F32)
    with np.errstate(all="ignore"):
        dot = _row_dot(y, dy, fault)
        t = _fma(-y, np.broadcast_to(dot[:, None], y.shape), dy)         # dy - y dot: one fused multiply-add
        return np.where((t == 0) & (inv[:, None] == np.inf), t, (t * inv[:, None]).astype(F32)).astype(F32)
