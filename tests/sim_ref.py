"""Exact and fp64 references of the similarity sweep S = X_a X_b^T (DESIGN 5), and the rules S is held to on every path that computes it.

The sweep splits each pre-scaled fp32 value into 2-byte pieces (split3 after pre_scale, kernels.cuh / device.cuh) and sums products of
pieces in an fp32 accumulator.  Products of two 2-byte pieces are exact, so the sum the sweep means to form is known exactly:

    M  = inv^2 sum over the format's piece pairs (p, q) of A_p B_q^T       fp16x2: hh + hl + lh;  bf16x3: hh + hm + mh + mm + hl + lh;  bf16: hh
    B  = the same sum over |A_p| |B_q|^T, the magnitude of what the accumulator added
    S64 = X_a X_b^T in fp64

The rules (violations):
    (i)   |S - M|   <= tau B + sub + TINY elementwise (sub: see model), and S = 0 exactly where B = 0 (no product was non-zero);
    (ii)  |S - S64| <= tau B + rep + TINY, rep the operand formats' error (DESIGN 5's table, as a bound per element: rep_elem);
    (iii) S is finite wherever S64 is within fp32's range.
Rule (i) sees a wrong piece, chunk or row in any single instruction, since B is the sum of the magnitudes of the very terms that were
added; rule (ii) ties M to the exact product.  Everything is computed with fp64 torch, on the GPU when there is one."""
from __future__ import annotations

import numpy as np

from npairloss_b200 import capi
import eval_ref
import grad_ref

FP16X2, BF16X3, BF16 = capi.PREC_FP32_FP16X2, capi.PREC_FP32_BF16X3, capi.PREC_BF16
PRECS = [FP16X2, BF16X3, BF16]
PASSES = grad_ref.PASSES
U24 = grad_ref.U24
TINY = 2.0 ** -149          # fp32's smallest subnormal: the epilogue's product may round to it or to 0
FLT_MAX = float(np.finfo(np.float32).max)
# the piece pairs each format's sweep forms (pass_pieces, gemm_wgmma.cuh)
PAIRS = {FP16X2: [(0, 0), (0, 1), (1, 0)], BF16X3: [(0, 0), (0, 1), (1, 0), (1, 1), (0, 2), (2, 0)], BF16: [(0, 0)]}
NPIECES = {FP16X2: 2, BF16X3: 3, BF16: 1}
EPILOGUE = 8                # tau's constant, in 2^-24 units of B


def _torch():
    import torch
    return torch, torch.device("cuda:0" if torch.cuda.is_available() else "cpu")


def pieces(x, prec, absmax=None):
    """(pieces, inv): the format's 2-byte pieces of x as split3 forms them after pre_scale, as float32 arrays in the scaled domain, and
    the inverse pre-scale 2^e (a Python float).  fp16 by numpy's conversion, bf16 by torch.bfloat16's, both round to nearest even with
    subnormals kept.  absmax: max|x| over the whole operand set (fp16x2's pre-scale); default max|x|."""
    import torch
    x = np.asarray(x, np.float32)
    if prec == FP16X2:
        e = eval_ref.sigma_exp(np.float32(np.abs(x).max() if absmax is None else absmax))
        v = (x * np.float32(2.0 ** -e)).astype(np.float32)
        hi = v.astype(np.float16).astype(np.float32)
        lo = (v - hi).astype(np.float16).astype(np.float32)
        return [hi, lo], 2.0 ** e

    def bf(a):
        return torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(torch.bfloat16).to(torch.float32).numpy()
    h = bf(x)
    if prec == BF16:
        return [h], 1.0
    r1 = (x - h).astype(np.float32)
    m = bf(r1)
    return [h, m, bf((r1 - m).astype(np.float32))], 1.0


def groups(P, D):
    """[rows, ceil(D / 16)] 0/1: whether a row has a non-zero piece among the features of each 16-feature group"""
    nz = np.zeros(P[0].shape, bool)
    for p in P:
        nz |= p != 0
    G = (D + 15) // 16
    pad = np.zeros((nz.shape[0], G * 16), bool)
    pad[:, :D] = nz
    return pad.reshape(nz.shape[0], G, 16).any(2).astype(np.float64)


def model(xa, xb, prec, absmax=None):
    """dict(M, B, S64, rep, L, sub) of the sweep of rows xa against rows xb, fp64 torch tensors [na, nb]: M, B and S64 of the module
    docstring, rep the bound of rule (ii) from rep_elem, and L = 16 times the number of 16-feature groups in which both rows are non-zero (the
    products of the instructions that can change the accumulator).  absmax: fp16x2's pre-scale operand, default max|x| over both sets."""
    torch, dev = _torch()
    xa, xb = np.asarray(xa, np.float32), np.asarray(xb, np.float32)
    if absmax is None:
        absmax = max(float(np.abs(xa).max(initial=0)), float(np.abs(xb).max(initial=0)))
    Pa, inv = pieces(xa, prec, absmax)
    Pb, _ = pieces(xb, prec, absmax)

    def t(a):
        return torch.from_numpy(np.ascontiguousarray(a)).to(dev, torch.float64)
    ta, tb = [t(p) for p in Pa], [t(p) for p in Pb]
    M = sum(ta[p] @ tb[q].T for p, q in PAIRS[prec]) * inv * inv
    B = sum(ta[p].abs() @ tb[q].abs().T for p, q in PAIRS[prec]) * inv * inv
    xa64, xb64 = t(xa), t(xb)
    S64 = xa64 @ xb64.T
    D = xa.shape[1]
    L = 16.0 * (t(groups(Pa, D)) @ t(groups(Pb, D)).T)
    # rep: |pieces - x| per element, then |a b - sum of the formed products| <= da |b| + |a| db + da db + the pairs not formed
    da, db = rep_elem(xa, prec, inv), rep_elem(xb, prec, inv)
    rep = t(da) @ xb64.abs().T + xa64.abs() @ t(db).T + t(da) @ t(db).T
    n = NPIECES[prec]
    for p in range(n):
        for q in range(n):
            if (p, q) not in PAIRS[prec]:
                rep = rep + (ta[p].abs() @ tb[q].abs().T) * inv * inv
    # fp16x2 elements whose hi piece is an fp16 subnormal (below 2^-14 of the pre-scale): the tensor cores' sum departs from M there
    # (measured, not modelled): rule (i) allows 2^-11 of their products' magnitude
    sub = torch.zeros_like(M)
    if prec == FP16X2:
        sa, sb = [np.where((P[0] != 0) & (np.abs(P[0]) < 2.0 ** -14), np.abs(x), 0.0) for P, x in ((Pa, xa), (Pb, xb))]
        if sa.any() or sb.any():
            sub = 2.0 ** -11 * (t(sa) @ xb64.abs().T + xa64.abs() @ t(sb).T)
    return dict(M=M, B=B, S64=S64, rep=rep, L=L, sub=sub)


def rep_elem(x, prec, inv):
    """DESIGN 5's operand error as a bound on |sum of x's pieces - x| per element (unscaled): fp16x2 max(2^-22 |x|, 2^-25 2^e) (the lo
    piece is relative to the element down to fp16's subnormal spacing 2^-24 at the pre-scale, i.e. relative to max|x|); bf16x3
    max(2^-24 |x|, 2^-134) (relative per element, floored by bf16's subnormal spacing 2^-133); bf16 max(2^-8 |x|, 2^-134) (round to
    nearest of an 8-bit significand)."""
    a = np.abs(np.asarray(x, np.float64))
    if prec == FP16X2:
        return np.maximum(2.0 ** -22 * a, 2.0 ** -25 * inv)
    if prec == BF16X3:
        return np.maximum(2.0 ** -24 * a, 2.0 ** -134)
    return np.maximum(2.0 ** -8 * a, 2.0 ** -134)


def tau(prec, path, L):
    """The bound of rule (i), as a fraction of B, over instructions whose products span L features (a number or a tensor).  A model of
    the tensor core's fp32 accumulator, which may truncate: about 2^-23 of the partial sum, hence of B, per k16 instruction, i.e.
    2 passes ceil(L / 16) units of 2^-24, and 2 units more per 16 features for the alignment of the products inside an instruction
    (bf16, one pass, measured 36 units at L = 128 on a spike), plus EPILOGUE units.  An instruction whose products are all 0 leaves the accumulator's bits
    as they are, so L counts the 16-feature groups in which both rows are non-zero (model's L); for dense rows it is D rounded up to 16.
    path "simt" is the SIMT check: piece sums in fp32 (2 roundings per operand), then one fp32 FMA per feature, rounded to nearest:
    L + 4 + EPILOGUE units.  Largest ratios |S - M| / B measured on an H100 80GB HBM3 (700 W) over test_gpu_sim_precision.py, in units
    of 2^-24 (this bound at D = 512 in brackets):
      fp16x2 75.5 at HL (8192 x 512, cosine-0.99 cone) (264);  bf16x3 74.8 at HL (456);  bf16 36.4 on a spike at D = 129 (72)
      fp16x2 on elements whose hi piece is an fp16 subnormal (rows 2^-12 .. 2^12 in norm, spikes): up to 333 (mixed_norm) and 74
      (spike at D = 33) against the model, within rule (ii).  The model does not explain it, so rule (i) allows 2^-11 of those
      elements' products there (model's sub).  Subnormal lo pieces under a normal hi need no allowance (memory rows 2^-6 of the
      batch: 22)."""
    if path == "simt":
        return (L + 4 + EPILOGUE) * U24
    groups16 = np.ceil(L / 16) if not hasattr(L, "ceil") else (L / 16).ceil()
    return (2 * (PASSES[prec] + 1) * groups16 + EPILOGUE) * U24


def violations(S, ref, tau_):
    """The rules of the module docstring that S breaks (empty: it passes), and dict(ratio = max |S - M| / B in units of 2^-24, worst =
    max |S - M| / (tau B + TINY), the share of rule (i)'s allowance used).  Elements where S64 overflows fp32 are exempt."""
    torch, dev = _torch()
    S = torch.from_numpy(np.ascontiguousarray(S, np.float32)).to(dev, torch.float64)
    M, B, S64, rep = ref["M"], ref["B"], ref["S64"], ref["rep"]
    if not torch.is_tensor(tau_):
        tau_ = torch.full_like(B, float(tau_))
    big = S64.abs() > FLT_MAX
    fin = torch.isfinite(S)
    bad = []
    n = int((~fin & ~big).sum())
    if n:
        bad.append(f"(iii) {n} non-finite elements where S64 is finite in fp32")
    ok = fin & ~big
    e1 = torch.where(ok, (S - M).abs(), torch.zeros_like(S))
    e2 = torch.where(ok, (S - S64).abs(), torch.zeros_like(S))
    zero = (B == 0) & ok
    n = int((zero & (S != 0)).sum())
    if n:
        bad.append(f"(i) {n} elements non-zero where no product was")
    allow = tau_ * B + ref.get("sub", 0.0) + TINY
    over1 = ok & (e1 > allow)
    ratio = torch.where((B > 0) & (e1 > TINY), e1 / B, torch.zeros_like(B))     # what the TINY floor absorbs is not a ratio
    r = float(ratio.max()) / U24 if ratio.numel() else 0.0
    if bool(over1.any()):
        i, j = np.unravel_index(int(torch.argmax(torch.where(over1, e1 / allow, torch.zeros_like(B)))), tuple(S.shape))
        bad.append(f"(i) {int(over1.sum())} elements over tau B, worst ({i}, {j}): |S - M| = {float(e1[i, j]):.3e}, "
                   f"{float(e1[i, j] / B[i, j]) / U24:.1f} x 2^-24 of B (tau {float(tau_[i, j]) / U24:.1f})")
    over2 = ok & (e2 > allow + rep)
    if bool(over2.any()):
        i, j = np.unravel_index(int(torch.argmax(torch.where(over2, e2 / (allow + rep), torch.zeros_like(B)))), tuple(S.shape))
        bad.append(f"(ii) {int(over2.sum())} elements over tau B + rep, worst ({i}, {j}): |S - S64| = {float(e2[i, j]):.3e}, "
                   f"allowed {float(allow[i, j] + rep[i, j]):.3e}")
    worst = float((e1 / allow).max()) if e1.numel() else 0.0
    return bad, dict(ratio=r, worst=worst)


def old_l1_passes(S, S64):
    """The L1 rule S was held to before: |S - S64| <= 1e-6 + 1.5e-5 |S64| (fp16x2), elementwise"""
    S64 = np.asarray(S64, np.float64)
    return bool((np.abs(np.asarray(S, np.float64) - S64) <= 1e-6 + 1.5e-5 * np.abs(S64)).all())


# ------------------------------------------------------------------------------------------------------------------------------ inputs
def _full_mantissa(rng, shape, lo=-3, hi=3):
    """Values of both signs with all 24 significand bits random and exponents in [lo, hi)"""
    m = rng.integers(2 ** 23, 2 ** 24, size=shape).astype(np.float64) / 2 ** 24
    return (m * np.exp2(rng.integers(lo, hi, size=shape)) * rng.choice([-1.0, 1.0], size=shape)).astype(np.float32)


def chunk_probe(n, D, seed):
    """n rows whose support is one 8-feature chunk each (the last one ragged when D % 8 != 0): row r lies in chunk (r + r // 8) mod C,
    C = ceil(D / 8), so that with n >= 8 C every chunk meets every row position mod 8.  Values have full 24-bit significands, so the lo
    and mid pieces are non-zero.  Pairs in different chunks must come out exactly 0."""
    rng = np.random.default_rng(seed)
    C = (D + 7) // 8
    x = np.zeros((n, D), np.float32)
    for r in range(n):
        c = (r + r // 8) % C
        w = min(8, D - 8 * c)
        x[r, 8 * c:8 * c + w] = _full_mantissa(rng, w)
    return x


def mixed_norm(n, D, seed):
    """Random directions with norms log-uniform over 2^-12 .. 2^12"""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, D))
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    return (x * np.exp2(rng.uniform(-12, 12, (n, 1)))).astype(np.float32)


def spike(n, D, seed):
    """Unit-scale random rows with one feature per row (a random one) 2^10 times the rest"""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, D)) / np.sqrt(D)
    x[np.arange(n), rng.integers(0, D, n)] *= 2.0 ** 10
    return x.astype(np.float32)


def dense(n, D, seed):
    """Well-spread unit rows (synth.make_inputs)"""
    from npairloss_b200 import synth
    return synth.make_inputs(n, D, seed)[0]


def cone(n, D, seed, cosine):
    """Unit rows around one direction at pairwise cosine about `cosine` (grad_ref.cone_inputs)"""
    return grad_ref.cone_inputs(n, D, float(np.sqrt(1.0 / cosine - 1.0)), seed)[0]


def dup(n, D, seed):
    """Cone rows (cosine 0.99) in groups of four exact copies"""
    return grad_ref.cone_inputs(n, D, 0.1, seed, dup=4)[0]


def tiny(n, D, seed):
    """Every |x| <= 2^-130 (fp32 subnormals): the pre-scale exponent's lower clamp"""
    rng = np.random.default_rng(seed)
    return (rng.uniform(-1.0, 1.0, (n, D)) * 2.0 ** -130).astype(np.float32)


def huge(n, D, seed):
    """Row 0 holds 1.5 2^127 in one feature, every other row is 0: the pre-scale exponent's upper clamp.  Only S[0][0] overflows."""
    x = np.zeros((n, D), np.float32)
    x[0, seed % D] = np.float32(1.5 * 2.0 ** 127)
    return x


KINDS = {"dense": dense, "probe": chunk_probe, "mixed": mixed_norm, "spike": spike, "dup": dup, "tiny": tiny, "huge": huge,
         "cone0.5": lambda n, D, s: cone(n, D, s, 0.5), "cone0.99": lambda n, D, s: cone(n, D, s, 0.99),
         "cone0.9996": lambda n, D, s: cone(n, D, s, 0.9996)}


def check(S, xa, xb, prec, path="tc", absmax=None, block=2048):
    """violations of S [na, nb] against the model of xa against xb, in blocks of `block` rows (the references hold five fp64 matrices
    of a block's size); absmax as in model, default max|x| over both sets.  Returns (bad, dict(ratio, worst)) over all blocks."""
    xa, xb = np.asarray(xa, np.float32), np.asarray(xb, np.float32)
    if absmax is None:
        absmax = max(float(np.abs(xa).max(initial=0)), float(np.abs(xb).max(initial=0)))
    bad, worst = [], dict(ratio=0.0, worst=0.0)
    for r0 in range(0, xa.shape[0], block):
        ref = model(xa[r0:r0 + block], xb, prec, absmax)
        b, m = violations(np.asarray(S)[r0:r0 + block], ref, tau(prec, path, ref["L"]))
        bad += [f"rows {r0}+: {x}" for x in b]
        worst = {k: max(worst[k], m[k]) for k in worst}
        del ref
    return bad, worst
