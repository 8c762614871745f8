"""The forward row reference (forward_ref.py) against both oracles, and the sensitivity of its rules to the ways a row pass or a
similarity epilogue goes wrong, without a GPU."""
import itertools

import numpy as np
import pytest

from npairloss_b200 import synth
import forward_ref as fr
from oracle import npair_oracle_np as onp

ALL_MININGS = [dict(margin_ident=0.02, margin_diff=-0.03, identsn=-0.4, diffsn=-0.3, ap_region=apR, ap_method=apM, an_region=anR,
                    an_method=anM)
               for apR, apM, anR, anM in itertools.product([0, 1], range(5), [0, 1], range(5))]
SAMPLE = ALL_MININGS[::7] + [synth.USAGE_MINING, synth.DEFAULT_MINING]
K = 14                                     # weight_scale_log2(PREC_FP16X2)


def _S(x, rows):
    xd = x.astype(np.float64)
    return (xd[rows] @ xd.T).astype(np.float32)


def _rank(x, lab, Q, world, rank, mining, cpp=None):
    """(reference, oracle state, oracle tops, S, self columns) of one rank; cpp: the C++ oracle to run as well."""
    rows = slice(rank * Q, (rank + 1) * Q)
    S = _S(x, rows)
    tops, st = onp.forward(x, lab, Q, world, rank, num_tops=5, S_inject=S, **mining)
    self_cols = np.arange(Q) + rank * Q
    ref = fr.reference(S, lab[rows], lab, self_cols, st["posi_thr"], st["nega_thr"], mining)
    if cpp is None:
        return ref, st, tops, S, self_cols
    tc, sc = cpp.forward(x, lab, cpp.make_config(Q, x.shape[1], world=world, rank=rank, num_tops=5, faithful_sorts=0, **mining),
                         S_inject=S)
    return ref, [(st, tops), (sc, tc)], None, S, self_cols


def _emulate(ref, S, mining, world=1):
    """What a correct row pass reports for the reference's rows: A, T, log(A/T), hits and records in fp32 as lse_rows_kernel forms them."""
    Q = S.shape[0]
    A = ref["A64"].astype(np.float32)
    T = ref["T64"].astype(np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        logv = np.where((A == 0) | (T == 0), np.float32(0), np.log(A / T).astype(np.float32)).astype(np.float32)
        iA = np.where(A == 0, np.float32(0), np.float32(1) / A).astype(np.float32)
        iT = np.where(T == 0, np.float32(0), np.float32(1) / T).astype(np.float32)
        m2c = np.where(T == 0, np.float32(np.inf),
                       ref["m2"] + np.log2(T).astype(np.float32) + np.float32(np.log2(world) - K)).astype(np.float32)
    j = fr.record_shift(A, T, K)
    sc = np.ldexp(np.float32(1), K - j).astype(np.float32)
    tp, tn = fr.transformed_thresholds(ref["posi"], ref["nega"], **mining)
    rec = np.stack([m2c, tn, (ref["m2"] - j.astype(np.float32)).astype(np.float32), ref["lab"], tp,
                    ((iT - iA) * sc).astype(np.float32), (iT * sc).astype(np.float32), np.zeros(Q, np.float32)], axis=1)
    hits, _ = fr.retrieval(ref, S)
    return dict(A=A, T=T, logv=logv, hits=hits.astype(np.float32).ravel(), rec=rec.astype(np.float32))


def _check_all(ref, S, g, mining, world=1):
    bad = fr.check_stats(ref, ref)
    bad += fr.check_sums(ref, g["A"], g["T"])[0]
    bad += fr.check_log(ref, g["logv"], g["A"], g["T"])
    bad += fr.check_hits(ref, S, g["hits"])[0]
    bad += fr.check_records(ref, g["rec"], g["A"], g["T"], ref["lab"], ref["posi"], ref["nega"], mining, K, world)[0]
    return bad


def _with_inputs(ref, lab_rows, posi, nega):
    ref.update(lab=np.asarray(lab_rows, np.float32), posi=np.asarray(posi, np.float32), nega=np.asarray(nega, np.float32))
    return ref


# ----------------------------------------------------------------------------------------------- the reference against the oracles
@pytest.mark.parametrize("world", [1, 2])
@pytest.mark.parametrize("mining", range(len(SAMPLE)))
def test_reference_is_the_oracle(oracle, world, mining):
    mining = SAMPLE[mining]
    Q, D = 48, 24
    x, lab = synth.make_inputs(Q * world, D, 3 + world, noise=2.5)
    for r in range(world):
        try:
            ref, oracles, _, S, _ = _rank(x, lab, Q, world, r, mining, cpp=oracle)
        except onp.OracleError:
            continue                                        # the mining refuses this set (an empty list): nothing to compare
        hits, amb = fr.retrieval(ref, S)
        for name, (st, tops) in zip(("numpy", "C++"), oracles):
            for k in ("min_within", "max_between", "max_all"):
                np.testing.assert_array_equal(ref[k], st[k], err_msg=f"{name} {k}")
            np.testing.assert_array_equal(ref["sel"], np.asarray(st["sel"]).astype(bool), err_msg=name)
            # the oracles' fp32 sums of fp32 expf against fp64 (nothing near the flush here)
            np.testing.assert_allclose(ref["A64"], st["A"], rtol=4e-6, atol=0, err_msg=name)
            np.testing.assert_allclose(ref["T64"], st["T"], rtol=4e-6, atol=0, err_msg=name)
            for t in range(3):
                d = abs(int(hits[t].sum()) - int(round(float(tops[1 + t]) * Q)))
                assert d <= int(amb.sum()), f"{name} k = {fr.KLIST[t]}: S-domain hits differ by {d} rows ({int(amb.sum())} ambiguous)"


def test_sentinels_of_a_row_without_a_same_label_column():
    Q, D = 16, 8
    x, _ = synth.make_inputs(Q, D, 5)
    lab = np.arange(Q, dtype=np.float32)                    # singletons: no same-label column anywhere
    S = _S(x, slice(0, Q))
    ref = fr.reference(S, lab, lab, np.arange(Q), np.zeros(Q, np.float32), np.zeros(Q, np.float32), synth.DEFAULT_MINING)
    assert (ref["min_within"] == fr.FLT_MAX).all() and (ref["max_within"] == -fr.FLT_MAX).all() and (ref["cnt_same"] == 0).all()
    assert (ref["A64"] == 0).all() and (ref["T64"] > 0).all()
    assert not fr.retrieval(ref, S)[0].any()


def test_flush_rule_drops_terms_below_2_pow_minus_126():
    """A row whose only positive lies 88 nats below its maximum: the positive is flushed, A64 = 0; at 86 nats it is kept."""
    for gap, kept in ((86.0, True), (88.0, False), (95.0, False)):
        S = np.array([[0.0, 10.0, 10.0 - gap, 0.0]], np.float32)
        lab = np.array([0, 1, 0, 2], np.float32)
        ref = fr.reference(S, lab[:1], lab, [0], [0.0], [0.0], synth.DEFAULT_MINING)
        assert (ref["A64"][0] > 0) == kept, gap
        assert ref["T64"][0] >= 1.0


# ----------------------------------------------------------------------------------------------- planted faults
def _case(world=1, mining=synth.USAGE_MINING, negative_row=False):
    Q, D = 64, 20
    x, lab = synth.make_inputs(Q * world, D, 9, noise=2.5)
    if negative_row:                                        # row 0 = u, every other row in the -u hemisphere
        u = x[0].copy()
        for i in range(1, Q * world):
            if x[i] @ u >= 0:
                x[i] -= 2 * (x[i] @ u) * u
                x[i] -= 1e-3 * u
        x /= np.linalg.norm(x, axis=1, keepdims=True)
        assert (_S(x, slice(0, 1))[0, 1:] < 0).all()
    ref, st, tops, S, selfc = _rank(x, lab, Q, world, world - 1, mining)
    _with_inputs(ref, lab[(world - 1) * Q:world * Q], st["posi_thr"], st["nega_thr"])
    return ref, S, mining, world, selfc


@pytest.mark.parametrize("world", [1, 2])
def test_correct_rows_pass(world):
    ref, S, mining, world, _ = _case(world)
    assert _check_all(ref, S, _emulate(ref, S, mining, world), mining, world) == []


def test_flags_self_column_in_max_all():
    ref, S, mining, world, selfc = _case()
    gpu = {k: ref[k].copy() for k in ("min_within", "max_within", "max_between", "max_all", "cnt_same")}
    gpu["max_all"] = np.maximum(gpu["max_all"], S[np.arange(S.shape[0]), selfc])
    assert any(b.startswith("max_all") for b in fr.check_stats(ref, gpu))


def test_flags_padding_zero_in_an_all_negative_row():
    ref, S, mining, world, _ = _case(negative_row=True)
    assert ref["max_between"][0] < 0 and ref["max_all"][0] < 0
    gpu = {k: ref[k].copy() for k in ("min_within", "max_within", "max_between", "max_all", "cnt_same")}
    gpu["max_between"][0] = max(gpu["max_between"][0], np.float32(0))
    assert any(b.startswith("max_between") for b in fr.check_stats(ref, gpu))


def test_flags_one_dropped_column_in_T():
    ref, S, mining, world, _ = _case(mining=synth.DEFAULT_MINING)
    g = _emulate(ref, S, mining)
    i = 7
    js = np.flatnonzero(ref["kept"][i])
    e = np.exp(np.float64(S[i, js[len(js) // 2]]) - np.float64(ref["max_all"][i]))
    g["T"][i] = np.float32(ref["T64"][i] - e)
    bad = fr.check_sums(ref, g["A"], g["T"])[0]
    assert any(b.startswith("T:") for b in bad), bad


def test_flags_one_flipped_hit():
    ref, S, mining, world, _ = _case()
    g = _emulate(ref, S, mining)
    _, amb = fr.retrieval(ref, S)
    i = int(np.flatnonzero(~amb)[3])
    g["hits"][ref["A64"].size + i] = 1 - g["hits"][ref["A64"].size + i]
    bad, n_amb = fr.check_hits(ref, S, g["hits"])
    assert n_amb == 0 and bad and bad[0].startswith("hits")


def test_flags_a_minus_inf_cA():
    ref, S, mining, world, _ = _case()
    g = _emulate(ref, S, mining)
    g["rec"][5, 5] = -np.inf
    bad, _ = fr.check_records(ref, g["rec"], g["A"], g["T"], ref["lab"], ref["posi"], ref["nega"], mining, K)
    assert any(b.startswith("record cA") for b in bad), bad


def test_flags_an_unshifted_record_whose_factor_overflows():
    """The overflow of 2^14 / A: a row with A = 2^-115 needs j = 2 (and only then is every factor finite)."""
    A = np.array([2.0 ** -115, 0.5], np.float32)
    T = np.array([1.0, 1.0], np.float32)
    assert fr.record_shift(A, T, K).tolist() == [2, 0]
    assert fr.record_shift(A, T, 0).tolist() == [0, 0]
    with np.errstate(over="ignore"):
        assert not np.isfinite(np.float32(np.float32(1) / A[0]) * np.float32(2.0 ** K))
