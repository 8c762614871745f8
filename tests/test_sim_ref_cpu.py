"""sim_ref against per-element loops and the oracles, its operand-error bound, and the sensitivity of its rules to the ways the similarity
sweep's instruction sequence (sim_kblock_mmas, gemm_wgmma.cuh) goes wrong, through a CPU emulation of that sequence, without a GPU."""
import numpy as np
import pytest

import sim_ref
from sim_ref import BF16, BF16X3, FP16X2, PRECS, U24
from oracle import npair_oracle_np as onp

BK = {FP16X2: 32, BF16X3: 16, BF16: 64}          # SimLayout::bk_of


def _half(v):
    """fp16 round to nearest even of one fp32 value by hand: subnormals kept, overflow to inf"""
    v = float(v)
    if v == 0 or not np.isfinite(v):
        return v
    e = max(int(np.floor(np.log2(abs(v)))), -14)
    q = 2.0 ** (e - 10)
    r = v / q
    f = np.floor(r)
    f = f + 1 if (r - f > 0.5 or (r - f == 0.5 and f % 2 == 1)) else f
    out = f * q
    return float("inf") * np.sign(v) if abs(out) > 65504 else out


def _bf16(v):
    v = float(v)
    if v == 0:
        return v
    e = max(int(np.floor(np.log2(abs(v)))), -126)
    q = 2.0 ** (e - 7)
    r = v / q
    f = np.floor(r)
    f = f + 1 if (r - f > 0.5 or (r - f == 0.5 and f % 2 == 1)) else f
    return f * q


def _pieces_loop(x, prec, absmax):
    out = []
    for v in np.asarray(x, np.float32).ravel():
        if prec == FP16X2:
            e = min(max(int(np.frexp(np.float32(absmax))[1]), -126), 127)
            s = float(np.float32(v) * np.float32(2.0 ** -e))
            h = _half(s)
            out.append((h, _half(float(np.float32(s - h)))))
        else:
            h = _bf16(v)
            r1 = float(np.float32(float(v) - h))
            m = _bf16(r1)
            out.append((h,) if prec == BF16 else (h, m, _bf16(float(np.float32(r1 - m)))))
    return np.array(out)


@pytest.mark.parametrize("prec", PRECS)
def test_pieces_agree_with_a_loop(prec):
    """Subnormal lo pieces, ties, full mantissas and both ends of the fp32 range"""
    rng = np.random.default_rng(3)
    vals = [1.0, 1 + 2 ** -11, 1 + 3 * 2 ** -11, 1 + 2 ** -8, 1 + 3 * 2 ** -8, 2 ** -20 + 2 ** -40, 0.75 + 2 ** -30, -0.3,
            1.5 * 2 ** 127, 2 ** -130, 3 * 2 ** -149, 0.0]
    x = np.concatenate([np.float32(vals), sim_ref._full_mantissa(rng, 40), sim_ref.mixed_norm(4, 8, 1).ravel()]).astype(np.float32)
    for absmax in (1.0, 2.0 ** 10, 2.0 ** -20, 1.5 * 2 ** 127, 2.0 ** -140):
        if prec != FP16X2 and absmax != 1.0:
            continue
        xs = x[np.abs(x) <= absmax] if prec == FP16X2 else x
        P, inv = sim_ref.pieces(xs, prec, absmax)
        np.testing.assert_array_equal(np.stack(P, 1), _pieces_loop(xs, prec, absmax), err_msg=f"absmax {absmax}")
        assert np.isfinite(inv) and inv > 0
    # the pre-scale's clamp: finite scale and inverse at both ends, and the subnormal lo piece at a small element
    assert sim_ref.pieces(np.float32([2.0 ** -130]), FP16X2)[1] == 2.0 ** -126
    assert sim_ref.pieces(np.float32([1.5 * 2 ** 127]), FP16X2)[1] == 2.0 ** 127
    (h, l), _ = sim_ref.pieces(np.float32([1 + 2 ** -23, 2 ** -12]), FP16X2, absmax=1.5)
    assert l[0] == 2.0 ** -24 and h[1] == 2.0 ** -13 and l[1] == 0       # 2^-24 at scale 2^-1: fp16's smallest subnormal


@pytest.mark.parametrize("prec", PRECS)
def test_model_agrees_with_the_oracles(oracle, prec):
    """M against the S of both oracles (the C++ one's fp32 GEMM, the NumPy one's fp64 rounded to fp32): within the format's error
    (rep) plus an fp32 sum of D terms"""
    from npairloss_b200 import synth
    Q, D = 48, 40
    x, lab = synth.make_inputs(Q, D, 5)
    ref = sim_ref.model(x, x, prec)
    M, rep = ref["M"].cpu().numpy(), ref["rep"].cpu().numpy()
    ax = np.abs(x.astype(np.float64))
    allow = rep + D * U24 * (ax @ ax.T)
    S_c = oracle.forward(x, lab, oracle.make_config(Q, D, faithful_sorts=0, **synth.DEFAULT_MINING))[1]["S"]
    S_n = onp.forward(x, lab, Q, 1, 0, num_tops=2, **synth.DEFAULT_MINING)[1]["S"]
    for S in (S_c, S_n):
        assert (np.abs(M - np.asarray(S, np.float64).reshape(Q, Q)) <= allow).all()


@pytest.mark.parametrize("kind", sorted(sim_ref.KINDS))
@pytest.mark.parametrize("prec", PRECS)
def test_rep_holds_on_every_kind(prec, kind):
    x = sim_ref.KINDS[kind](64, 40, 9)
    ref = sim_ref.model(x, x, prec)
    ok = ref["S64"].abs() <= sim_ref.FLT_MAX
    assert bool((((ref["M"] - ref["S64"]).abs() <= ref["rep"]) | ~ok).all())


@pytest.mark.parametrize("prec", PRECS)
def test_rep_is_approached(prec):
    """One feature per row, so that every element of S is one product and the bound is not a sum of magnitudes: worst / bound > 1/4"""
    rng = np.random.default_rng(4)
    x = sim_ref._full_mantissa(rng, (400, 1), -2, 0)
    ref = sim_ref.model(x, x, prec)
    r = float((((ref["M"] - ref["S64"]).abs()) / ref["rep"]).max())
    assert 0.25 < r <= 1.0, r


def test_fp16x2_error_is_relative_to_max_and_bf16x3_per_element():
    """Rows 2^-12 .. 2^12 in norm: fp16x2's error on the small rows is far above 2^-22 of their own similarity, bf16x3's is not"""
    x = sim_ref.mixed_norm(200, 32, 2)
    n = np.linalg.norm(x, axis=1)
    small = n < 2.0 ** -8
    rel = {}
    for prec in (FP16X2, BF16X3):
        ref = sim_ref.model(x, x, prec)
        err = ((ref["M"] - ref["S64"]).abs() / ref["S64"].abs().clamp_min(1e-300)).cpu().numpy()
        rel[prec] = float(np.diagonal(err)[small].max())
    assert rel[FP16X2] > 2.0 ** -16 and rel[BF16X3] < 2.0 ** -22, rel


# ------------------------------------------------------------------------------------- the sweep's instruction sequence, emulated
def _trunc24(v):
    """fp32 accumulator truncated to 24 significant bits (toward zero)"""
    m, e = np.frexp(v)
    return np.ldexp(np.trunc(m * 2.0 ** 24) / 2.0 ** 24, e)


def emulate(xa, xb, prec, fault=None, absmax=None, exact=False):
    """S of sim_kblock_mmas's instruction sequence: per K block of BK features the hh (and mm) instructions per 16 features, then per
    piece x after hi and per 8-feature chunk one cross instruction hi_a x_b + x_a hi_b; the fp32 accumulator truncated after each
    instruction (exact: no rounding at all); then acc * inv * inv.  fault plants one of the defects the rules must see."""
    rnd = (lambda v: v) if exact else _trunc24
    if absmax is None:
        absmax = max(float(np.abs(xa).max()), float(np.abs(xb).max()))
    Pa, inv = sim_ref.pieces(xa, prec, absmax)
    Pb, _ = sim_ref.pieces(xb, prec, absmax)
    D = xa.shape[1]
    Dp = (D + 63) // 64 * 64
    pad = lambda P: [np.pad(p.astype(np.float64), ((0, 0), (0, Dp - D))) for p in P]
    Pa, Pb = pad(Pa), pad(Pb)
    if fault == "row_swap":                       # rows 2 and 5 of row group 0 exchanged in A's lo piece
        Pa[1][[2, 5]] = Pa[1][[5, 2]]
    n = len(Pa)
    acc = np.zeros((xa.shape[0], xb.shape[0]))
    bk = BK[prec]
    nkb = Dp // bk
    c_fault = (D // 8) // 2                       # the chunk a single-chunk fault hits
    for kb in range(nkb):
        if fault == "drop_last_kblock" and kb == (D - 1) // bk:
            continue
        k0 = kb * bk
        for s in range(2 if n == 3 else 1):
            for k in range(k0, k0 + bk, 16):
                acc = rnd(acc + Pa[s][:, k:k + 16] @ Pb[s][:, k:k + 16].T)
        for x in range(1, n):
            for c in range(k0, k0 + bk, 8):
                cs = slice(c, c + 8)
                if fault == "drop_cross" and c == 8 * c_fault and x == 1:
                    continue
                b_x = Pb[x][:, c + 8:c + 16] if (fault == "next_chunk" and c == 8 * c_fault and x == 1) else Pb[x][:, cs]
                lo_hi = Pa[0][:, cs] @ b_x.T if fault == "twice" else Pa[x][:, cs] @ Pb[0][:, cs].T
                acc = rnd(acc + Pa[0][:, cs] @ b_x.T + lo_hi)
                if fault == "lolo" and x == n - 1:
                    acc = rnd(acc + Pa[x][:, cs] @ Pb[x][:, cs].T)
    S = acc.astype(np.float32) * np.float32(inv)
    return S if fault == "inverse_once" else S * np.float32(inv)


def _flagged(S, x, prec):
    return sim_ref.check(S, x, x, prec)[0]


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("kind", ["dense", "cone0.99", "probe", "mixed", "spike"])
def test_emulation_stays_within_tau(prec, kind):
    x = sim_ref.KINDS[kind](136, 100, 12)
    bad, m = sim_ref.check(emulate(x, x, prec), x, x, prec)
    assert not bad, (bad, m)
    assert m["worst"] > 0 if kind != "probe" else True


FAULTS = ["drop_cross", "next_chunk", "twice", "row_swap", "drop_last_kblock", "inverse_once"]


def test_planted_faults_are_flagged():
    """Each fault, on well-spread dense rows and on one-chunk probes at D = 100 (ragged) in fp16x2; the rule that catches it is
    recorded (dense or probe).  Adding lo * lo, which is more accurate, is not flagged."""
    D = 100
    dense = sim_ref.dense(136, D, 13) * np.float32(3.0)          # max|x| above 1, so that the pre-scale is not 1
    probe = sim_ref.chunk_probe(136, D, 14)
    caught = {}
    for f in FAULTS:
        caught[f] = [name for name, x in (("dense", dense), ("probe", probe)) if _flagged(emulate(x, x, FP16X2, f), x, FP16X2)]
    print("caught by:", caught)
    assert all(caught[f] for f in FAULTS), caught
    # the single-chunk faults are seen by the probes whatever the data; the whole-operand ones by both
    assert "probe" in caught["drop_cross"] and "probe" in caught["next_chunk"], caught
    for x in (dense, probe):
        assert not _flagged(emulate(x, x, FP16X2, "lolo"), x, FP16X2)


def test_the_old_l1_rule_misses_single_chunk_faults_on_a_cone():
    """On the cosine-0.99 cone at D = 512 the previous rule |S - S64| <= 1e-6 + 1.5e-5 |S64| passes a dropped cross instruction and a
    cross instruction reading the next chunk, at every element, when the sweep is emulated in exact arithmetic; the probes flag both."""
    x = sim_ref.cone(96, 512, 15, 0.99)
    S64 = x.astype(np.float64) @ x.astype(np.float64).T
    for f in ("drop_cross", "next_chunk"):
        assert sim_ref.old_l1_passes(emulate(x, x, FP16X2, f, exact=True), S64), f
        p = sim_ref.chunk_probe(136, 512, 16)
        assert _flagged(emulate(p, p, FP16X2, f), p, FP16X2), f


def test_range_edges():
    """The clamped pre-scale at both ends of the fp32 range: the tiny batch gives 0 (or a subnormal), the zero rows next to a huge row
    give exactly 0; the unclamped scale (inf) would give NaN"""
    for kind in ("tiny", "huge"):
        x = sim_ref.KINDS[kind](20, 24, 1)
        S = emulate(x, x, FP16X2)
        bad, _ = sim_ref.check(S, x, x, FP16X2)
        assert not bad, (kind, bad)
    assert np.isinf(emulate(sim_ref.huge(4, 8, 0), sim_ref.huge(4, 8, 0), FP16X2)[0, 0])
