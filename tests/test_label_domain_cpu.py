"""The references the GPU label-domain tests rely on (tests/test_gpu_label_domain.py), on the same label families at small sizes: the
C++ oracle and the NumPy oracle agree on shuffled, interleaved and unbalanced classes, on negative, fractional, ~1e7, 2^24 + 2m, +-0 and
+-inf labels, and on NaN-labelled rows (no positive, not even themselves); select_ref's relative thresholds equal the oracle's."""
import itertools

import numpy as np
import pytest

import select_ref
from npairloss_b200 import synth
from oracle import npair_oracle_np as onp
from test_gpu_label_domain import FAMILIES, _nan_anchor_inputs, family_inputs, relabel

REL = (synth.RELATIVE_HARD, synth.RELATIVE_EASY)
REL_AP = {synth.GLOBAL: synth.RELATIVE_HARD, synth.LOCAL: synth.HARD}   # the NaN-anchor case's AP side (a NaN row's AP list is empty)


def _both(oracle, x, lab, Q, world, kw):
    """(tops, dx) of both oracles, or None when both refuse the batch (one refusing alone fails)."""
    cfg = oracle.make_config(Q, x.shape[1], world=world, **kw)
    try:
        a = oracle.step_world(x, lab, cfg, 0.7)
    except oracle.OracleError:
        a = None
    try:
        b = onp.step_world(x, lab, Q, world, 0.7, **kw)
    except onp.OracleError:
        b = None
    assert (a is None) == (b is None), (kw, a is None)
    return a, b


@pytest.mark.parametrize("world", [1, 2])
@pytest.mark.parametrize("family", FAMILIES)
def test_oracles_agree_on_every_family(oracle, family, world):
    """All 100 (region, method)^2 minings, both oracles, at Q = 24 per rank and three images per class."""
    Q, D = 24, 16
    x, lab = family_inputs(family, Q * world, D, seed=5 + world, per_class=3, noise=0.7)
    if family == "values":
        assert np.isinf(lab).any() and (np.signbit(lab) & (lab == 0)).any() and ((lab == 0) & ~np.signbit(lab)).any()
    if family == "nan":
        assert np.isnan(lab).sum() >= 3
    refused = 0
    for apR, apM, anR, anM in itertools.product([0, 1], range(5), [0, 1], range(5)):
        kw = dict(margin_ident=0.02, margin_diff=-0.03, identsn=-0.4, diffsn=-0.3, ap_region=apR, ap_method=apM, an_region=anR,
                  an_method=anM)
        a, b = _both(oracle, x, lab, Q, world, kw)
        if a is None:
            refused += 1
            continue
        np.testing.assert_allclose(a[0], b[0], rtol=2e-6, atol=1e-7, err_msg=f"{family} {kw}")
        assert np.isfinite(a[1]).all(), kw
        assert np.linalg.norm(a[1] - b[1]) <= 2e-6 * max(np.linalg.norm(b[1]), 1e-12), (family, kw)
    # rows without a positive (singletons, NaN rows) make the LOCAL relative AP side refuse: 2 x 2 x 5 minings
    assert refused == (20 if family in ("unbalanced", "nan") else 0), refused


@pytest.mark.parametrize("family", FAMILIES)
def test_relabelling_leaves_the_oracle_unchanged(oracle, family):
    """The injective renaming of the GPU relabelling test (permuted ids, +0 <-> -0, NaN payloads) changes nothing in the oracle."""
    Q, D = 48, 16
    x, lab = family_inputs(family, Q, D, seed=9, per_class=3, noise=0.7)
    lab2 = relabel(lab, seed=3)
    assert (np.isnan(lab) == np.isnan(lab2)).all()
    for kw in (dict(margin_diff=-0.05, identsn=-0.0, diffsn=-0.3, ap_region=0, ap_method=3, an_region=1, an_method=0),
               dict(margin_ident=0.01, margin_diff=-0.02, identsn=-0.4, diffsn=-0.3, ap_region=0, ap_method=4, an_region=1, an_method=3)):
        cfg = oracle.make_config(Q, D, **kw)
        t0, g0 = oracle.step_world(x, lab, cfg, 0.7)
        t1, g1 = oracle.step_world(x, lab2, cfg, 0.7)
        np.testing.assert_array_equal(t1, t0)
        np.testing.assert_array_equal(g1, g0)


def _relative_minings(region, has_positive):
    """Minings whose selected sides are relative with a general SN; the AP side of LOCAL only where every row has a positive."""
    out = []
    for an_method, diffsn in itertools.product(REL, (-0.3, -0.7, 3.0)):
        if region == 0:
            out.append(dict(identsn=-0.4, diffsn=diffsn, ap_region=0, ap_method=REL[0] + REL[1] - an_method, an_region=0, an_method=an_method))
        else:
            out.append(dict(identsn=-1.0, diffsn=diffsn, ap_region=1, ap_method=0, an_region=1, an_method=an_method))
            if has_positive:
                out.append(dict(identsn=-0.5, diffsn=diffsn, ap_region=1, ap_method=an_method, an_region=1, an_method=an_method))
    return out


@pytest.mark.parametrize("world", [1, 2])
@pytest.mark.parametrize("family", FAMILIES)
def test_select_ref_matches_the_oracle(oracle, family, world):
    """select_ref.relative_thresholds on the oracle's own S equals the oracle's thresholds bit for bit, LOCAL and GLOBAL, every rank."""
    Q, D = 66, 16
    x, lab = family_inputs(family, Q * world, D, seed=21 + world, per_class=3, noise=1.5)
    has_positive = bool(select_ref.side_masks(lab, lab, 0)[0].any(axis=1).all())
    assert has_positive == (family not in ("unbalanced", "nan")), family
    for region in (0, 1):
        for kw in _relative_minings(region, has_positive):
            for r in range(world):
                _, st = oracle.forward(x, lab, oracle.make_config(Q, D, world=world, rank=r, **kw))
                rows = slice(r * Q, (r + 1) * Q)
                ref = select_ref.relative_thresholds(st["S"], lab[rows], lab, r * Q, region, kw["identsn"], kw["diffsn"])
                if kw["ap_method"] in REL:
                    np.testing.assert_array_equal(ref["posi"].view(np.uint32), st["posi_thr"].view(np.uint32), err_msg=f"{family} {kw}")
                np.testing.assert_array_equal(ref["nega"].view(np.uint32), st["nega_thr"].view(np.uint32), err_msg=f"{family} {kw}")


@pytest.mark.parametrize("world", [1, 2])
def test_nan_anchor_inputs_reach_the_self_pair(oracle, world):
    """The inputs of the GPU's NaN-anchor case: the oracle's AN threshold of every NaN row (LOCAL) and of each rank (GLOBAL) lies above
    that row's S_ii, and a list that kept S_ii -- what a select that drops the self pair by label alone would see -- picks a different
    value.  So the GPU case can tell the two apart."""
    B, D = 256, 64
    Q = B // world
    x, lab, nan_rows = _nan_anchor_inputs(B, D, seed=31)
    S = (x.astype(np.float64) @ x.astype(np.float64).T).astype(np.float32)
    assert (S > 0).all()
    for region, an_method, diffsn in itertools.product((0, 1), REL, (-0.3, -0.7, 3.0)):
        kw = dict(identsn=-0.4 if region == 0 else -1.0, diffsn=diffsn, ap_region=region, ap_method=REL_AP[region], an_region=region,
                  an_method=an_method)
        for r in range(world):
            rows = slice(r * Q, (r + 1) * Q)
            _, st = oracle.forward(x, lab, oracle.make_config(Q, D, world=world, rank=r, **kw), S_inject=S[rows])
            mine = nan_rows[(nan_rows >= r * Q) & (nan_rows < (r + 1) * Q)]
            assert mine.size
            same, diff = select_ref.side_masks(lab[rows], lab, r * Q)
            for i in mine:
                assert S[i, i] < st["nega_thr"][i - r * Q], (kw, i)
            diff[mine - r * Q, mine] = True                          # the self pairs of the NaN rows kept in the diff-label list
            if region == 1:
                for i in mine:
                    vals = S[i, diff[i - r * Q]]
                    kept = np.partition(vals, select_ref.pos(diffsn, vals.size - 1))[select_ref.pos(diffsn, vals.size - 1)]
                    assert kept != st["nega_thr"][i - r * Q], (kw, i)
            else:
                vals = S[rows][diff]
                p = select_ref.pos(diffsn, vals.size - len(mine))
                assert np.partition(vals, p)[p] != st["nega_thr"][0], kw

