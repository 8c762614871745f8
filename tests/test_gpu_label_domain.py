"""The layer on the labels training feeds it.  synth.make_inputs gives sorted, contiguous, small non-negative labels in classes of
equal size; a training pipeline gives shuffled classes (an m-per-class sampler), class ids in the tens of thousands, singletons and one
dominant class, and sometimes NaN-marked rows.  Several kernels branch on labels: the similarity epilogue skips a 32-column chunk whose
label range leaves out the row's label (and the mirrored statistics a 32-row group), the GLOBAL select and the row pass take a fast path
for four diff-label columns, the LOCAL selects keep short same-label lists.  Sorted labels send almost every chunk far from the diagonal
down the skip; interleaved labels send none.

The self pair is in neither list whatever its label (reference .cu:54).  A NaN-labelled row is its own diff-label column by label, so a
select that drops the self pair only because it carries the row's label keeps it; `test_nan_anchor_self_pair` puts that entry below
the pick, where it moves the AN threshold by one rank.

Every GPU result is checked with gpu_harness.check_parity (the oracle on the GPU's own S); where the oracle refuses a batch, the
library must refuse it with the same error."""
import itertools

import numpy as np
import pytest

import select_ref
from npairloss_b200 import capi, synth

pytestmark = pytest.mark.gpu

FP16X2, TC, SIMT = capi.PREC_FP32_FP16X2, capi.GEMM_TCGEN05, capi.GEMM_SIMT_CHECK
REL_H, REL_E = synth.RELATIVE_HARD, synth.RELATIVE_EASY
ORACLE_TO_NPAIR = {1: -1, 2: -4, 3: -5}       # NPO_ERR_* -> NPAIR_E_*
FAMILIES = ("shuffled", "interleaved", "unbalanced", "values", "nan")
ROWS = (1, 2, 3, 4, 5, 6, 7, 8, 9)           # npair_debug_read selectors of the per-row arrays


# ------------------------------------------------------------------------------------------------------------------ label families
def _class_layout(family, B, rng, per_class):
    """Class index of every row (-1: a NaN-labelled row), in the order the batch holds them."""
    if family == "interleaved":
        return np.arange(B) % -(-B // per_class)                     # every 32-column chunk spans the whole label range
    if family == "unbalanced":
        big, single = max(B // 4, 2), max(1, round(0.05 * B))
        sizes = [big] + [1] * single
        left, k = B - big - single, 0
        while left > 0:
            s = min(2 + k % 2, left)                                  # classes of 2 and 3 (the last one may be a singleton)
            sizes.append(s)
            left -= s
            k += 1
        cls = np.repeat(np.arange(len(sizes)), sizes)
    else:
        cls = np.arange(B) // per_class
    if family == "nan":
        cls = cls.copy()
        cls[rng.choice(B, max(3, B // 100), replace=False)] = -1
    return rng.permutation(cls)


def _class_values(family, n_cls, rng):
    """fp32 label value of each class index."""
    if family == "values":
        v = np.empty(n_cls, np.float64)
        for k in range(n_cls):
            kind = k % 4
            v[k] = (-1.0 - k if kind == 0 else                      # negative
                    1000.0 + 0.5 * k if kind == 1 else              # fractional (k odd): steps of 0.5
                    1e7 + k if kind == 2 else                       # around 1e7
                    2.0 ** 24 + 2 * (k // 4))                      # 2^24 + 2m: neighbours one fp32 ulp apart
        v[:3] = (0.0, np.inf, -np.inf)                              # class 0 mixes +0.0 and -0.0 (below)
        return v.astype(np.float32)
    if family in ("shuffled", "nan"):
        return rng.choice(100_000, n_cls, replace=False).astype(np.float32)    # SOP / iNaturalist-sized class ids
    return np.arange(n_cls, dtype=np.float32)


def family_inputs(family, B, D, seed, per_class=4, noise=1.0):
    """(x, lab) of one label family: x = normalize(centre of the row's class + noise * g) as synth.make_inputs, every NaN row with a
    centre of its own.  Families: shuffled (classes of `per_class` in random order, ids up to 1e5), interleaved (label = i % C),
    unbalanced (one class of B/4, classes of 2 and 3, 5 % singletons), values (negative, fractional, ~1e7, 2^24 + 2m, +-0 in one class,
    +inf, -inf), nan (shuffled plus max(3, B/100) NaN rows)."""
    rng = np.random.default_rng(seed)
    cls = _class_layout(family, B, rng, per_class)
    n_cls = int(cls.max()) + 1
    vals = _class_values(family, n_cls, rng)
    lab = np.where(cls >= 0, vals[np.maximum(cls, 0)], np.float32(np.nan)).astype(np.float32)
    if family == "values":
        zero = np.flatnonzero(cls == 0)
        lab[zero[::2]] = np.float32(-0.0)
    centres = rng.standard_normal((n_cls + B, D)).astype(np.float32)
    key = np.where(cls >= 0, cls, n_cls + np.arange(B))
    x = centres[key] + np.float32(noise) * rng.standard_normal((B, D)).astype(np.float32)
    x /= np.linalg.norm(x.astype(np.float64), axis=1, keepdims=True).astype(np.float32)
    return np.ascontiguousarray(x, np.float32), np.ascontiguousarray(lab, np.float32)


def relabel(lab, seed):
    """An injective renaming that scrambles the label order: the distinct values permuted among themselves, +0.0 <-> -0.0, and every
    NaN given other payload bits (sign bit set on every other one)."""
    rng = np.random.default_rng(seed)
    lab = np.asarray(lab, np.float32)
    finite = ~np.isnan(lab)
    uniq = np.unique(lab[finite])                                   # +0.0 and -0.0 are one value
    perm = uniq[rng.permutation(uniq.size)]
    out = lab.copy()
    out[finite] = perm[np.searchsorted(uniq, lab[finite])]
    bits = out.view(np.uint32)
    zero = out == 0
    bits[zero] ^= np.uint32(0x80000000)                             # +0 <-> -0
    nan_idx = np.flatnonzero(~finite)
    bits[nan_idx] = (np.uint32(0x7FC00000) | (np.arange(nan_idx.size, dtype=np.uint32) * 977 + 5)) ^ \
        np.where(np.arange(nan_idx.size) % 2 == 1, np.uint32(0x80000000), np.uint32(0)).astype(np.uint32)
    assert np.isnan(out[nan_idx]).all()
    return out


@pytest.fixture(scope="module")
def cuda():
    import torch
    assert torch.cuda.is_available(), "GPU tests need an H100"
    assert torch.cuda.get_device_capability(0) == (9, 0)
    return torch


def _bits(a):
    return np.ascontiguousarray(np.asarray(a, np.float32)).view(np.uint32)


def _parity_or_refusal(oracle, x, lab, Q, world, mining, backend=TC, tag="", **cfg):
    """check_parity; where the oracle refuses the batch, the library must refuse it with the same code.  Returns the GPU result, or
    None for a refused batch."""
    from gpu_harness import check_parity, gpu_step_world
    N = x.shape[0]
    try:                        # a refusal depends on the list sizes only, not on S: a zero S stands in for the oracle's own
        oracle.step_world(x, lab, oracle.make_config(Q, x.shape[1], world=world, faithful_sorts=0, **mining), 0.7,
                          S_inject_all=np.zeros((N, N), np.float32), want_grad=False)
    except oracle.OracleError as e:
        with pytest.raises(capi.NpairError) as ge:
            gpu_step_world(x, lab, Q, world, mining, FP16X2, backend, want_grad=False, **cfg)
        assert ge.value.code == ORACLE_TO_NPAIR[e.code], (tag, ge.value.code, e.code)
        return None
    g = gpu_step_world(x, lab, Q, world, mining, FP16X2, backend, loss_weight=0.7, **cfg)
    check_parity(oracle, x, lab, Q, world, mining, FP16X2, backend, loss_weight=0.7, tag=tag, gpu=g, **cfg)
    return g


def _assert_select_ref(g, lab, Q, world, mining, tag):
    """The GPU's thresholds of every relative side equal select_ref's on the GPU's own S, bit for bit."""
    for r in range(world):
        rows = slice(r * Q, (r + 1) * Q)
        ref = select_ref.relative_thresholds(g["S"][rows], lab[rows], lab, r * Q, mining["an_region"], mining["identsn"],
                                             mining["diffsn"])
        if mining["ap_method"] in (REL_H, REL_E) and mining["ap_region"] == mining["an_region"]:
            assert np.array_equal(_bits(g["posi"][rows]), _bits(ref["posi"])), f"{tag} posi vs select_ref, rank {r}"
        if mining["an_method"] in (REL_H, REL_E):
            bad = np.flatnonzero(_bits(g["nega"][rows]) != _bits(ref["nega"]))
            assert bad.size == 0, f"{tag} nega vs select_ref, rank {r}: rows {bad[:8]} labels {lab[rows][bad[:8]]}"


# ------------------------------------------------------------------------------------------------------------------ 1. every mining
@pytest.mark.parametrize("backend", [SIMT, TC], ids=["simt", "tc"])
@pytest.mark.parametrize("world,bwd_exchange", [(1, 0), (3, 0), (3, 1)])
@pytest.mark.parametrize("family", ["shuffled", "unbalanced", "nan"])
def test_all_minings_small(cuda, oracle, family, world, bwd_exchange, backend):
    """Every (region, method)^2 at Q = 48 per rank, about three images per class, with the mining parameters of
    test_gpu_parity.py::test_all_mining_modes_small.  Rows without a positive make the LOCAL relative AP side refuse the batch."""
    Q, D = 48, 40
    x, lab = family_inputs(family, Q * world, D, seed=100 + world + 7 * FAMILIES.index(family), per_class=3, noise=0.7)
    refused = 0
    for apR, apM, anR, anM in itertools.product([0, 1], range(5), [0, 1], range(5)):
        mining = dict(margin_ident=0.02, margin_diff=-0.03, identsn=-0.4, diffsn=-0.3, ap_region=apR, ap_method=apM, an_region=anR,
                      an_method=anM)
        g = _parity_or_refusal(oracle, x, lab, Q, world, mining, backend, tag=f"{family} w{world} x{bwd_exchange} {apR}{apM}{anR}{anM}",
                               bwd_exchange=bwd_exchange)
        refused += g is None
    print(f"{family} w{world} x{bwd_exchange} b{backend}: {refused} of 100 minings refused")
    assert refused < 100


# ------------------------------------------------------------------------------------------------------------------ 2. medium shapes
MEDIUM_MININGS = {
    "usage": synth.USAGE_MINING,
    "local_rel": dict(synth.DEFAULT_MINING, ap_method=REL_H, an_method=REL_H, identsn=0.0, diffsn=-0.3, margin_diff=-0.01),
    # the AN side alone: defined on rows without a positive, where local_rel's AP list is empty
    "local_rel_an": dict(synth.DEFAULT_MINING, ap_method=synth.HARD, an_method=REL_H, identsn=0.0, diffsn=-0.3, margin_diff=-0.01),
    "global_hard": dict(synth.DEFAULT_MINING, ap_region=synth.GLOBAL, ap_method=synth.HARD, an_region=synth.GLOBAL, an_method=synth.HARD,
                        margin_diff=-0.05),
    "global_rel": dict(margin_ident=0.01, margin_diff=-0.02, identsn=-0.4, diffsn=-0.3, ap_region=synth.GLOBAL, ap_method=REL_H,
                       an_region=synth.GLOBAL, an_method=REL_H),
}


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("Q,D", [(999, 101), (2048, 512)])
def test_medium_shapes(cuda, oracle, Q, D, family):
    """The LOCAL relative minings go through both LOCAL select kernels, whose thresholds must be bitwise equal to each other and to
    select_ref's; so must the GLOBAL select's."""
    x, lab = family_inputs(family, Q, D, seed=Q + D + FAMILIES.index(family), noise=2.5)
    for name, mining in MEDIUM_MININGS.items():
        if name.startswith("local_rel"):
            gs = [_parity_or_refusal(oracle, x, lab, Q, 1, mining, tag=f"{family} Q{Q} {name} f{f}", flags=f) for f in (0, capi.FLAG_LSEL_WARP)]
            if gs[0] is None:
                assert name == "local_rel" and family in ("unbalanced", "nan") and gs[1] is None, (family, name)
                continue
            assert np.array_equal(_bits(gs[0]["S"]), _bits(gs[1]["S"]))
            for key in ("posi", "nega"):
                assert np.array_equal(_bits(gs[0][key]), _bits(gs[1][key])), f"{family} Q{Q} {name}: {key} of the two LOCAL kernels"
            _assert_select_ref(gs[0], lab, Q, 1, mining, f"{family} Q{Q} {name}")
        else:
            g = _parity_or_refusal(oracle, x, lab, Q, 1, mining, tag=f"{family} Q{Q} {name}")
            assert g is not None, (family, name)
            if name == "global_rel":
                _assert_select_ref(g, lab, Q, 1, mining, f"{family} Q{Q} {name}")


# ------------------------------------------------------------------------------------------------------------------ 3. NaN self pair
def _nan_anchor_inputs(B, D, seed):
    """Collapsed unit rows (every cosine positive) in shuffled classes of 4, and 6 NaN-labelled rows scaled by 1/8: S_ii = 1/64 lies
    below every entry of the row except those against the other NaN rows."""
    from test_gpu_select_paths import _collapsed
    rng = np.random.default_rng(seed)
    x = _collapsed(B, D, seed=seed + 1, eps=0.1)
    lab = rng.permutation(np.arange(B) // 4).astype(np.float32)
    nan_rows = np.sort(np.concatenate([rng.choice(B // 2, 3, replace=False), B // 2 + rng.choice(B // 2, 3, replace=False)]))
    lab[nan_rows] = np.nan
    x[nan_rows] *= np.float32(0.125)
    return np.ascontiguousarray(x), lab, nan_rows


@pytest.mark.parametrize("region,world,flags", [(synth.LOCAL, 1, 0), (synth.LOCAL, 1, capi.FLAG_LSEL_WARP), (synth.GLOBAL, 1, 0),
                                                (synth.GLOBAL, 2, 0)], ids=["local-block", "local-warp", "global-w1", "global-w2"])
def test_nan_anchor_self_pair(cuda, oracle, region, world, flags):
    """The AN side relative (diffsn -0.3, -0.7, 3.0), the AP side not LOCAL relative (a NaN row's same-label list is empty).  A select
    that counts S_ii of a NaN row in the diff-label list picks one order statistic too low."""
    from test_gpu_select_paths import G_TOL_CLUSTER, _run
    B, D = 256, 64
    Q = B // world
    x, lab, nan_rows = _nan_anchor_inputs(B, D, seed=31)
    assert {r // Q for r in nan_rows} == set(range(world))
    for an_method, diffsn in itertools.product((REL_H, REL_E), (-0.3, -0.7, 3.0)):
        if region == synth.LOCAL:
            m = dict(margin_ident=0.01, margin_diff=-0.02, identsn=-1.0, diffsn=diffsn, ap_region=synth.LOCAL, ap_method=synth.HARD,
                     an_region=synth.LOCAL, an_method=an_method)
        else:
            m = dict(margin_ident=0.01, margin_diff=-0.02, identsn=-0.4, diffsn=diffsn, ap_region=synth.GLOBAL, ap_method=REL_H,
                     an_region=synth.GLOBAL, an_method=an_method)
        tag = f"nan anchors r{region} w{world} f{flags} m{an_method} sn{diffsn}"
        S, _ = _run(oracle, x, lab, Q, world, m, tag=tag, g_tol=G_TOL_CLUSTER, flags=flags)
        # the precondition: every NaN row's S_ii lies below the oracle's AN threshold of that row (LOCAL) or of its rank (GLOBAL)
        for r in range(world):
            _, st = oracle.forward(x, lab, oracle.make_config(Q, D, world=world, rank=r, faithful_sorts=0, **m),
                                   S_inject=S[r * Q:(r + 1) * Q])
            for i in nan_rows[(nan_rows >= r * Q) & (nan_rows < (r + 1) * Q)]:
                assert S[i, i] < st["nega_thr"][i - r * Q], (tag, i, S[i, i], st["nega_thr"][i - r * Q])


# ------------------------------------------------------------------------------------------------------------------ 4. relabelling
RELABEL_MININGS = {
    "usage": synth.USAGE_MINING,
    "relative": dict(margin_ident=0.01, margin_diff=-0.02, identsn=-0.4, diffsn=-0.3, ap_region=synth.GLOBAL, ap_method=REL_E,
                     an_region=synth.LOCAL, an_method=REL_H),
}


@pytest.mark.parametrize("flags", [0, capi.FLAG_LSEL_WARP], ids=["block", "warp"])
@pytest.mark.parametrize("Q,world", [(999, 1), (333, 3)])
@pytest.mark.parametrize("family", FAMILIES)
def test_relabelling_is_bitwise(cuda, family, Q, world, flags):
    """Labels enter only through equality, every statistic is a max, min or count, and the row pass and the fused gradient sum in
    column order with skipped pairs adding nothing: an injective renaming that scrambles the label order leaves tops, gradient and
    every per-row array bit for bit unchanged.  A difference means the label-range skip and the slow statistics path disagree."""
    from test_gpu_sim_blocks import _step
    D = 101 if world == 1 else 128          # each rank's slice of the gradient must start on the 16-byte grid
    x, lab = family_inputs(family, Q * world, D, seed=Q + world + FAMILIES.index(family), noise=2.5)
    lab2 = relabel(lab, seed=world + 17)
    assert not np.array_equal(_bits(lab), _bits(lab2))
    for name, mining in RELABEL_MININGS.items():
        t0, g0, r0 = _step(x, lab, Q, world, flags=flags, **mining)
        t1, g1, r1 = _step(x, lab2, Q, world, flags=flags, **mining)
        tag = f"{family} Q{Q} w{world} f{flags} {name}"
        assert np.array_equal(_bits(t1), _bits(t0)), f"{tag}: tops {t1} vs {t0}"
        assert np.array_equal(_bits(g1), _bits(g0)), f"{tag}: gradient differs by up to {np.abs(g1 - g0).max():.3e}"
        for k, w in enumerate(ROWS):
            bad = np.flatnonzero(_bits(r1[k]) != _bits(r0[k]))
            assert bad.size == 0, f"{tag}: debug_read({w}) differs in rows {bad[:8]}"
        assert np.isfinite(g0).all() and np.abs(g0).max() > 0, tag


# ------------------------------------------------------------------------------------------------------------------ 5. row blocks
@pytest.mark.parametrize("family,world", [("shuffled", 1), ("nan", 1), ("shuffled", 2), ("nan", 2)],
                         ids=["shuffled", "nan", "shuffled-w2", "nan-w2"])
def test_row_blocks(cuda, family, world):
    """NPAIR_SIM_BLOCK_ROWS(256) at Q = 999 per rank is bit for bit the materialised path (checked against the oracle in
    test_medium_shapes).  At world 2 a block's self columns are offset by both the rank and the block, and with NaN labels only their
    position keeps the self pairs out of the LOCAL selects.  Row-block mode refuses a GLOBAL relative side with a general SN, so the
    GLOBAL mining here is global_hard."""
    from test_gpu_sim_blocks import _compare
    Q = 999
    D = 101 if world == 1 else 128          # each rank's slice of the gradient must start on the 16-byte grid
    x, lab = family_inputs(family, Q * world, D, seed=Q + D + FAMILIES.index(family), noise=2.5)
    for name in ("usage", "local_rel_an", "global_hard"):
        for flags in ((0, capi.FLAG_LSEL_WARP) if name.startswith("local") else (0,)):
            _compare(x, lab, Q, world, 256, f"{family} w{world} {name} f{flags} row blocks", flags=flags, **MEDIUM_MININGS[name])


# ------------------------------------------------------------------------------------------------------------------ 6. headline size
def test_headline_size_shuffled(cuda, oracle):
    """B = 8192, D = 512, usage mining, shuffled classes of 4 with ids up to 1e5: almost no 32-column chunk can be skipped."""
    from gpu_harness import check_parity
    x, lab = family_inputs("shuffled", 8192, 512, seed=20171230, noise=2.5)
    r = check_parity(oracle, x, lab, 8192, 1, synth.USAGE_MINING, FP16X2, TC, tag="HL shuffled")
    print("HL shuffled", r)
