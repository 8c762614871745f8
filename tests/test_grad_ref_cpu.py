"""The fp64 gradient reference (grad_ref.py) against the oracles, the |w| <= 1 premise of the fp16x2 weight scale, and the sensitivity
of the componentwise and per-row checks to the ways a gradient kernel goes wrong, without a GPU."""
import itertools

import numpy as np
import pytest

from npairloss_b200 import synth
import grad_ref
import sim_ref
from grad_ref import U24
from oracle import npair_oracle_np as onp

ALL_MININGS = [dict(margin_ident=0.02, margin_diff=-0.03, identsn=-0.4, diffsn=-0.3, ap_region=apR, ap_method=apM, an_region=anR,
                    an_method=anM)
               for apR, apM, anR, anM in itertools.product([0, 1], range(5), [0, 1], range(5))]
SAMPLE = ALL_MININGS[::7]                 # every (region, method) of either side appears
WEIGHT_LOG2 = 14                          # weight_scale_log2(PREC_FP16X2), kernels.cuh
OPERANDS_ONLY = 16 * U24                  # tau's operand term: an emulation without the tensor core's accumulator


def _S(x, rows=None):
    xd = x.astype(np.float64)
    return ((xd if rows is None else xd[rows]) @ xd.T).astype(np.float32)


def _or_refusal(f):
    try:
        return f()
    except onp.OracleError:
        return None


@pytest.mark.parametrize("world", [1, 2, 3])
def test_reference_is_the_oracle_step(oracle, world):
    Q, D = 36, 24
    x, lab = grad_ref.cone_inputs(Q * world, D, 0.5, 7 + world, dup=3)
    S = _S(x)
    done = 0
    for mining in SAMPLE:
        cfg = oracle.make_config(Q, D, world=world, faithful_sorts=0, **mining)
        try:
            _, dx_o = oracle.step_world(x, lab, cfg, 1.0, S_inject_all=S)
        except oracle.OracleError:
            assert _or_refusal(lambda: grad_ref.step(x, lab, Q, world, S, **mining)) is None, mining
            continue
        ref = grad_ref.step(x, lab, Q, world, S, **mining)
        # the C++ oracle runs the reference's fp32 GEMMs: within 1e-5 of the magnitude B; the NumPy one is fp64 rounded to fp32
        assert (np.abs(ref["R"] - dx_o) <= 1e-5 * ref["B"] + 1e-30).all(), mining
        _, dx_np = onp.step_world(x, lab, Q, world, S_inject_all=S, num_tops=2, **mining)
        assert (np.abs(ref["R"] - dx_np) <= 2.0 ** -24 * np.abs(ref["R"]) + 1e-30).all(), mining
        assert (np.abs(ref["R"]) <= ref["B"] * (1 + 1e-12)).all() and (np.abs(ref["R32"] - ref["R"]) <= 1e-5 * ref["B"] + 1e-30).all()
        done += 1
    assert done >= len(SAMPLE) // 2


def test_memory_form_is_the_numpy_oracle_step():
    """The memory step's products on the anchors' rows against the NumPy oracle's fp64 step over [x; x_mem]."""
    Q, m, D = 32, 52, 24
    x, lab = grad_ref.cone_inputs(Q + m, D, 0.5, 5, dup=2)
    lab[Q:] %= Q // 2
    S = _S(x, slice(0, Q))
    done = 0
    for mining in SAMPLE:
        ref = _or_refusal(lambda: grad_ref.step(x, lab, Q, 1, S, **mining))
        if ref is None:
            continue
        _, dx, _ = onp.step_world_fp64(x, lab, Q, 1, S_inject_all=S, **mining)
        dx = dx[:Q]
        np.testing.assert_allclose(ref["R"][:Q], dx, rtol=1e-12, atol=1e-15 * np.abs(dx).max(), err_msg=str(mining))
        done += 1
    assert done >= len(SAMPLE) // 2


@pytest.mark.parametrize("world", [1, 3])
@pytest.mark.parametrize("kind", ["ties", "all_equal"])
def test_every_weight_is_at_most_one(world, kind):
    """|g'| <= 1 for every weight, so |g'| / world <= 1 for the transposed ones and the world-1 operand g'(j, m) + g'(m, j) is at most 2:
    2^14 times it stays below fp16's largest finite 65504.  Over all 100 mining combinations, with pairs exactly at the thresholds."""
    Q, D = 40, 16
    x, lab = grad_ref.cone_inputs(Q * world, D, 0.3, 3, dup=4, all_equal=kind == "all_equal")
    S = _S(x)
    worst = 0.0
    for mining in ALL_MININGS:
        for r in range(world):
            st = _or_refusal(lambda: onp.forward(x, lab, Q, world, r, num_tops=2, S_inject=S[r * Q:(r + 1) * Q], **mining)[1])
            if st is None:
                continue
            g = grad_ref.unit_weights(st)
            assert np.abs(g).max() <= 1.0, mining
            if world == 1:
                H = g + g.T
                assert np.abs(H).max() <= 2.0 and 2.0 ** WEIGHT_LOG2 * np.abs(H).max() < 65504, mining
            worst = max(worst, float(np.abs(g).max()))
    assert worst > 0.5      # the bound is approached, not vacuous


# ----------------------------------------------------------------------------------------- the fp16x2 weight split, emulated
def _split(w, k):
    """fp16 hi + lo pieces of 2^k w (round to nearest, subnormals kept, as __floats2half2_rn), undone in fp64: sim_ref's emulation of
    the fp16x2 split at pre-scale 1."""
    v = (np.asarray(w, np.float32) * np.float32(2.0 ** k)).astype(np.float32)
    (hi, lo), _ = sim_ref.pieces(v, sim_ref.FP16X2, absmax=0.5)
    return (hi.astype(np.float64) + lo.astype(np.float64)) / 2.0 ** k


def test_scaled_split_is_fp32_faithful():
    """At 2^14 a weight of [2^-17, 2] keeps 2^-22 relative precision, and every smaller one 2^-39 absolute; unscaled, the lo piece of a
    weight below 2^-3 is subnormal and the error is up to 2^-25 absolute."""
    rng = np.random.default_rng(1)
    w = (np.exp2(rng.uniform(-24, 1, 200000)) * rng.choice([-1.0, 1.0], 200000)).astype(np.float32)
    w64 = w.astype(np.float64)
    big = np.abs(w64) >= 2.0 ** -17
    err = np.abs(_split(w, WEIGHT_LOG2) - w64)
    assert (err[big] <= 2.0 ** -22 * np.abs(w64[big])).all()
    assert (err[~big] <= 2.0 ** -39).all()
    err0 = np.abs(_split(w, 0) - w64)
    assert not (err0[big] <= 2.0 ** -22 * np.abs(w64[big])).all() and err0.max() > 2.0 ** -27
    assert np.abs(_split(np.float32([2.0, -2.0]), WEIGHT_LOG2)).max() == 2.0          # the largest world-1 operand: no overflow


def _world1_operand(G, Q, lw=1.0):
    """The world-1 weight operand as the kernels form it: H = g'(j, m) + g'(m, j) in fp32 (unit weights), and c = lw / Q."""
    c = np.float64(np.float32(lw) / np.float32(Q))
    g = (G / c).astype(np.float32)
    return (g + g.T).astype(np.float32), c


def _emulated(H, c, x, k):
    return 0.5 * c * (_split(H, k) @ x.astype(np.float64))


@pytest.mark.parametrize("eps", [0.1, 0.02])
def test_checks_flag_the_unscaled_split_on_clustered_rows(eps):
    """The fp16x2 split of unscaled weights, emulated exactly (no accumulator error): the componentwise and per-row rules flag it on
    rows in a cone of cosine 0.99 and 0.9996, where the whole-matrix normwise 1e-5 rule passes it at 0.99.  The same split after the
    2^14 scale passes all three."""
    Q, D = 2048, 64
    x, lab = grad_ref.cone_inputs(Q, D, eps, 21)
    ref = grad_ref.step(x, lab, Q, 1, _S(x), **synth.DEFAULT_MINING)
    H, c = _world1_operand(ref["G"][0][0], Q)
    dx = _emulated(H, c, x, 0)
    bad, m = grad_ref.violations(dx, ref, OPERANDS_ONLY)
    assert any(b.startswith("componentwise") for b in bad) and any(b.startswith("per row") for b in bad), (bad, m)
    if eps == 0.1:
        assert m["normwise"] <= 1e-5, m
    bad, m = grad_ref.violations(_emulated(H, c, x, WEIGHT_LOG2), ref, OPERANDS_ONLY)
    assert not bad, (bad, m)


def test_checks_flag_kernel_faults():
    """Faults confined to one weight, one 64-column K block of one 128-row tile, or one 256-column K chunk added twice, at the fused
    kernel's tau: the componentwise and per-row rules flag each.  The whole-matrix normwise 1e-5 rule misses the dropped weight (it
    catches a dropped K block of dense weights at this N; below 1e-5 of the norm such a block falls only from about N = 40000 on)."""
    Q, D = 4096, 64
    x, lab = synth.make_inputs(Q, D, 22, noise=2.5)
    ref = grad_ref.step(x, lab, Q, 1, _S(x), **synth.DEFAULT_MINING)
    G = ref["G"][0][0]
    H = G + G.T                                        # the world-1 operand, c included
    xd = x.astype(np.float64)
    R = ref["R"]
    tau = grad_ref.tau(grad_ref.FP16X2, "fused", Q)

    def flagged(dx):
        bad, _ = grad_ref.violations(dx, ref, tau)
        return any(b.startswith("componentwise") for b in bad) and any(b.startswith("per row") for b in bad)

    # one selected pair's weight dropped: a weight of median size in row 5
    row = np.abs(H[5])
    j = int(np.argmin(np.abs(row - np.median(row[row > 0]))))
    dx = R.copy()
    dx[5] -= 0.5 * H[5, j] * xd[j]
    assert flagged(dx) and np.linalg.norm(dx - R) <= 1e-5 * np.linalg.norm(R)
    # one 64-column K block of the second 128-row tile dropped
    dx = R.copy()
    dx[128:256] -= 0.5 * H[128:256, 1024:1088] @ xd[1024:1088]
    assert flagged(dx)
    # one 256-column K chunk of the first tile added twice
    dx = R.copy()
    dx[:128] += 0.5 * H[:128, 256:512] @ xd[256:512]
    assert flagged(dx)
