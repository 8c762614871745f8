"""The relative-mining selects on every path they take (DESIGN §4.1): GLOBAL buckets beyond the candidate buffer (three sweeps) and rows
that overflow the compaction's staging area, the LOCAL warp kernel's lane-list overflow and its default use for rows past 8192 columns,
the same-label list's size boundaries, exact ties across digit boundaries, and un-normalised embeddings.

Collapsed embeddings -- every row close to one direction, as a freshly initialised or collapsing network gives -- put almost every
similarity in one leading-digit bucket; that is what sends the selects to their fallbacks.  Every case runs the two-level oracle parity of
gpu_harness.check_parity, compares the GPU's thresholds bit for bit with tests/select_ref.py on the GPU's own S, and asserts the predicate
of the path it is named after, so a change of a constant that moves a case off its path fails the case."""
import numpy as np
import pytest

import select_ref
from npairloss_b200 import capi, synth

pytestmark = pytest.mark.gpu

FP16X2, BF16X3 = capi.PREC_FP32_FP16X2, capi.PREC_FP32_BF16X3
REL_H, REL_E = synth.RELATIVE_HARD, synth.RELATIVE_EASY


@pytest.fixture(scope="module")
def cuda():
    import torch
    assert torch.cuda.is_available(), "GPU tests need an H100"
    assert torch.cuda.get_device_capability(0) == (9, 0)
    return torch


def _unit(x):
    x = np.asarray(x, np.float32)
    return np.ascontiguousarray(x / np.linalg.norm(x.astype(np.float64), axis=1, keepdims=True).astype(np.float32))


def _collapsed(B, D, seed, eps=0.03, direction=None):
    """Rows normalize(e + eps * g): every similarity between two rows lies close to 1 / (1 + eps^2 D)."""
    rng = np.random.default_rng(seed)
    e = np.zeros(D, np.float32) if direction is None else direction
    if direction is None:
        e[0] = 1.0
    return _unit(e[None, :] + np.float32(eps) * rng.standard_normal((B, D)).astype(np.float32))


def _labels(B, per_class):
    return (np.arange(B) // per_class).astype(np.float32)


def _mining(region, identsn, diffsn, ap_method=REL_H, an_method=REL_H, ap_region=None):
    return dict(margin_ident=0.01, margin_diff=-0.02, identsn=identsn, diffsn=diffsn, ap_region=region if ap_region is None else ap_region,
                ap_method=ap_method, an_region=region, an_method=an_method)


def _bits(a):
    return np.ascontiguousarray(np.asarray(a, np.float32)).view(np.uint32)


# Normwise gradient bound for a tight cluster of rows.  Every row of the gradient weights G sums to zero, so in dX = G X the components
# along the cluster's common direction cancel, and the result is 100-200 times smaller than the terms it sums: operand rounding of
# 2^-22 (fp16x2) then shows as 1e-5 .. 5e-5 normwise.  Measured on an H100: collapsed set 2.5e-5, staging-overflow set 5.0e-5 (fp16x2).
# The thresholds, loss and tops of these cases are still held to check_parity's bounds.
G_TOL_CLUSTER = 1e-4


def _run(oracle, x, lab, Q, world, mining, prec=FP16X2, tag="", g_tol=None, **cfg):
    """One forward per rank for the GPU's S and thresholds; select_ref's thresholds on that S must be bitwise the GPU's for every side
    the region selects; then the full oracle parity (with the gradient bound `g_tol` instead of the harness's, if given).  Returns
    (S, select_ref results per rank)."""
    import gpu_harness
    from gpu_harness import check_parity, gpu_step_world
    g = gpu_step_world(x, lab, Q, world, mining, prec, capi.GEMM_TCGEN05, want_grad=False, **cfg)
    refs = []
    for r in range(world):
        rows = slice(r * Q, (r + 1) * Q)
        ref = select_ref.relative_thresholds(g["S"][rows], lab[rows], lab, r * Q, mining["an_region"], mining["identsn"], mining["diffsn"])
        refs.append(ref)
        if mining["ap_region"] == mining["an_region"] and mining["ap_method"] in (REL_H, REL_E):
            assert np.array_equal(_bits(g["posi"][rows]), _bits(ref["posi"])), f"{tag} posi vs select_ref, rank {r}: rows " \
                f"{np.flatnonzero(_bits(g['posi'][rows]) != _bits(ref['posi']))[:8]}"
        if mining["an_method"] in (REL_H, REL_E):
            assert np.array_equal(_bits(g["nega"][rows]), _bits(ref["nega"])), f"{tag} nega vs select_ref, rank {r}: rows " \
                f"{np.flatnonzero(_bits(g['nega'][rows]) != _bits(ref['nega']))[:8]}"
    saved = gpu_harness.G_TOL[prec]
    try:
        if g_tol is not None:
            gpu_harness.G_TOL[prec] = g_tol
        res = check_parity(oracle, x, lab, Q, world, mining, prec, capi.GEMM_TCGEN05, loss_weight=0.7, tag=tag, **cfg)
    finally:
        gpu_harness.G_TOL[prec] = saved
    print(f"{tag}: gradient normwise error {res['g_rel']:.2e}")
    return g["S"], refs


def _gbucket(S, lab, Q, r, side, sn):
    rows = slice(r * Q, (r + 1) * Q)
    return select_ref.global_bucket(S[rows], lab[rows], lab, r * Q, side, sn)


# ---------------------------------------------------------------------------------------------------------------------------------
# 1. collapsed set: the GLOBAL select's chosen bucket holds more than the candidate buffer on both sides -> three sweeps of S
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [1, 2])
@pytest.mark.parametrize("sn", [-0.3, -0.5, -0.97, 3.0, 1000.0])
def test_global_three_sweep_collapsed(cuda, oracle, sn, world):
    """B = 1024, D = 64, rows normalize(e0 + 0.03 g), 4 classes of 256: every off-diagonal similarity is in [0.875, 1), one 11-bit
    bucket.  world 2 is emulated with Q = 512 (self_offset 512 on rank 1 in the third sweep)."""
    B, D = 1024, 64
    Q = B // world
    x, lab = _collapsed(B, D, seed=101), _labels(B, 256)
    for apM, anM in ((REL_H, REL_H), (REL_E, REL_E)):
        m = _mining(synth.GLOBAL, sn, sn, apM, anM)
        S, refs = _run(oracle, x, lab, Q, world, m, tag=f"collapsed sn{sn} w{world} m{apM}", g_tol=G_TOL_CLUSTER)
        for r in range(world):
            for side in (0, 1):
                b = _gbucket(S, lab, Q, r, side, sn)
                print(f"rank {r} side {side}: bucket {b['pop']:,} > cap {b['cap']:,}")
                assert b["pop"] > b["cap"], b
            assert refs[r]["posi_raw"][0] >= 0 and refs[r]["nega_raw"][0] >= 0


# ---------------------------------------------------------------------------------------------------------------------------------
# 2. two antipodal clusters: the picks sit in the positive bucket, above a whole bucket of negative entries
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("region,flags", [(synth.GLOBAL, 0), (synth.LOCAL, 0), (synth.LOCAL, capi.FLAG_LSEL_WARP)])
def test_antipodal_clusters(cuda, oracle, region, flags):
    """Rows 0..511 near +e0, rows 512..1023 near -e0; each class of 8 has 4 rows in each cluster.  The AN list is half and the AP list
    4/7 negative, so a miscounted negative bucket moves the pick, and the pick (>= 0) is visible through the clamp."""
    B, D = 1024, 64
    x = _collapsed(B, D, seed=202)
    x[B // 2:] = -x[B // 2:]
    lab = np.concatenate([_labels(B // 2, 4), _labels(B // 2, 4)])
    for identsn, diffsn in ((-0.2, -0.3), (-0.1, -0.45), (2.0, 40.0)):
        m = _mining(region, identsn, diffsn)
        S, refs = _run(oracle, x, lab, B, 1, m, tag=f"antipodal r{region} f{flags} sn{identsn},{diffsn}", flags=flags)
        same, diff = select_ref.side_masks(lab, lab, 0)
        for name, mask in (("posi_raw", same), ("nega_raw", diff)):
            below = (S[mask] < 0).sum()
            print(f"{name}: {below:,} negative entries below picks >= {refs[0][name].min():.4f}")
            assert refs[0][name].min() >= 0 and below > mask.sum() // 3


# ---------------------------------------------------------------------------------------------------------------------------------
# 3. GLOBAL compaction with rows of more than 2048 bucket entries: the staging area overflows into direct global stores
# ---------------------------------------------------------------------------------------------------------------------------------
def test_global_staging_overflow(cuda, oracle):
    """B = 8192, D = 128: random rows plus a tight cluster of 2400 rows (two images per class).  AN GLOBAL relative with diffsn = 1e6:
    the pick is the 10^6-th largest diff-label similarity, inside the cluster's bucket of about 5.7 M entries (cap 8.39 M)."""
    B, D, C = 8192, 128, 2400
    x, lab = synth.make_inputs(B, D, seed=303, imgs_per_class=2, noise=2.5)
    rng = np.random.default_rng(304)
    x[:C] = _collapsed(C, D, seed=305, eps=0.02, direction=_unit(rng.standard_normal((1, D)))[0])
    m = _mining(synth.GLOBAL, -0.5, 1e6, ap_method=REL_E)
    S, refs = _run(oracle, x, lab, B, 1, m, tag="staging overflow", g_tol=G_TOL_CLUSTER)
    b = _gbucket(S, lab, B, 0, 1, 1e6)
    print(f"bucket {b['pop']:,} <= cap {b['cap']:,}; row {b['row']}: {b['row_max']:,} candidates in the bucket")
    assert b["pop"] <= b["cap"] and b["row_max"] > select_ref.GSEL_STAGE, b
    assert refs[0]["nega_raw"][0] >= 0


# ---------------------------------------------------------------------------------------------------------------------------------
# 4. exact ties: wanted ranks inside runs of equal keys, and consecutive ranks on both sides of a binade boundary
# ---------------------------------------------------------------------------------------------------------------------------------
def _inside_run(vals, p):
    s = np.sort(vals)
    return 0 < p < s.size - 1 and s[p - 1] == s[p] == s[p + 1]


@pytest.mark.parametrize("region,flags", [(synth.GLOBAL, 0), (synth.LOCAL, 0), (synth.LOCAL, capi.FLAG_LSEL_WARP)])
def test_ties_sixteen_vectors(cuda, oracle, region, flags):
    """16 distinct unit vectors, each repeated 64 times over B = 1024 (random order), 8 classes of 128: every list is made of runs of
    equal keys (about 8 per value in a row's same-label list, hundreds in the other lists)."""
    B, D = 1024, 32
    rng = np.random.default_rng(404)
    base = _unit(rng.standard_normal((16, D)))
    x = np.ascontiguousarray(base[rng.permutation(np.arange(B) % 16)])
    lab = rng.permutation(_labels(B, 128))
    same, diff = select_ref.side_masks(lab, lab, 0)
    for identsn, diffsn in ((-0.3, -0.3), (-0.6, -0.15), (5.0, 300.0)):
        m = _mining(region, identsn, diffsn, REL_H, REL_E)
        S, refs = _run(oracle, x, lab, B, 1, m, tag=f"ties16 r{region} f{flags} sn{identsn},{diffsn}", flags=flags)
        for key, mask, p in (("pos_ap", same, refs[0]["pos_ap"]), ("pos_an", diff, refs[0]["pos_an"])):
            if region == synth.GLOBAL:
                inside = _inside_run(S[mask], p)
            else:
                inside = np.mean([_inside_run(S[i, mask[i]], p[i]) for i in range(B)]) > 0.5
            print(f"{key}: wanted rank inside a run of equal keys: {inside}")
            assert inside


def _binade_set():
    """Five vectors with exact dot products in {0, 0.25, 0.5, 1}, repeated 40 times each (B = 200), 10 classes of 20."""
    v = np.array([[1, 0, 0, 0], [0.5, 0.5, 0.5, 0.5], [0.5, 0, 0, 0], [0, 0, 0, 1], [0, 0.5, 0, 0]], np.float32)
    rng = np.random.default_rng(405)
    x = np.ascontiguousarray(v[rng.permutation(np.arange(200) % 5)])
    lab = rng.permutation(_labels(200, 20))
    return x, lab


def _boundary_sns(vals):
    """Absolute SNs whose ranks are the last entry below and the first entry at or above 0.25, 0.5 and 1 (0 -> 0.25 included)."""
    s = np.sort(vals)
    out = []
    for edge in (0.25, 0.5, 1.0):
        k = int(np.searchsorted(s, np.float32(edge)))
        if 0 < k < s.size:
            out += [float(s.size - 1 - (k - 1)), float(s.size - 1 - k)]
    return sorted(set(sn for sn in out if sn >= 1))           # SN < 1 picks the maximum: a closed form, no select


@pytest.mark.parametrize("region,flags", [(synth.GLOBAL, 0), (synth.LOCAL, 0), (synth.LOCAL, capi.FLAG_LSEL_WARP)])
def test_ties_across_binade_boundaries(cuda, oracle, region, flags):
    x, lab = _binade_set()
    B = x.shape[0]
    S64 = x.astype(np.float64) @ x.astype(np.float64).T
    same, diff = select_ref.side_masks(lab, lab, 0)
    if region == synth.GLOBAL:
        ap_sns, an_sns = _boundary_sns(S64[same]), _boundary_sns(S64[diff])
    else:                       # the boundaries of row 0; rows with the same vector and label have the same lists
        ap_sns, an_sns = _boundary_sns(S64[0, same[0]]), _boundary_sns(S64[0, diff[0]])
    assert len(ap_sns) >= 2 and len(an_sns) >= 4, (ap_sns, an_sns)
    n = max(len(ap_sns), len(an_sns))
    for k in range(n):
        identsn, diffsn = ap_sns[k % len(ap_sns)], an_sns[k % len(an_sns)]
        m = _mining(region, identsn, diffsn)
        S, refs = _run(oracle, x, lab, B, 1, m, tag=f"binades r{region} f{flags} sn{identsn},{diffsn}", flags=flags)
        assert np.array_equal(S, S64.astype(np.float32)), "the similarities are exact"
        for key, mask, sn in (("posi_raw", same, identsn), ("nega_raw", diff, diffsn)):
            vals = np.sort(S[mask] if region == synth.GLOBAL else S[0, mask[0]])
            p = select_ref.pos(sn, vals.size)
            print(f"{key}: rank {p} = {vals[p]} next to {vals[max(p - 1, 0)]} / {vals[min(p + 1, vals.size - 1)]}")
            assert refs[0][key][0] == vals[p]
            assert vals[max(p - 1, 0)] != vals[p] or vals[min(p + 1, vals.size - 1)] != vals[p], "the rank sits at a boundary"


# ---------------------------------------------------------------------------------------------------------------------------------
# 5. LOCAL warp kernel: a lane gets more than 48 entries of the chosen bin -> slow_select_row for the AN side
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("flags", [capi.FLAG_LSEL_WARP, 0])
def test_local_lane_list_overflow(cuda, oracle, flags):
    """Collapsed rows at B = 2048, D = 128, 8 images per class (7 same-label entries: the AN side keeps the fast path up to its
    candidate lists).  Every row's chosen 10-bit bin, [0.75, 1), holds about 2040 entries.  Without the flag the same rows go through
    the block kernel's refinement of a crowded value bin."""
    B, D = 2048, 128
    x, lab = _collapsed(B, D, seed=505), _labels(B, 8)
    for identsn, diffsn in ((-0.3, -0.3), (-0.5, -0.7), (2.0, 100.0)):
        m = _mining(synth.LOCAL, identsn, diffsn, REL_E, REL_H)
        S, refs = _run(oracle, x, lab, B, 1, m, tag=f"lane overflow f{flags} sn{identsn},{diffsn}", flags=flags)
        w = select_ref.local_warp_bins(S, lab, lab, 0, diffsn)
        i = int(w["pop"].argmax())
        print(f"row {i}: {w['pop'][i]:,} entries in the chosen bin, {w['lane_max'][i]} in one lane")
        assert w["pop"].min() > 32 * select_ref.LSEL_LANE_CAP and w["lane_max"].min() > select_ref.LSEL_LANE_CAP
        assert (refs[0]["nega_raw"] >= 0).all() and (np.array(refs[0]["pos_an"]) > 0).all()


# ---------------------------------------------------------------------------------------------------------------------------------
# 6. rows longer than 8192 columns: the warp kernel is the default, also block by block in row-block mode
# ---------------------------------------------------------------------------------------------------------------------------------
def _long_rows():
    """world 2, Q = 4608 (N = 9216), D = 128, classes of 4; every other class collapsed near e0, the rest random."""
    B, D = 9216, 128
    x, lab = synth.make_inputs(B, D, seed=606, imgs_per_class=4, noise=1.5)
    col = (np.arange(B) // 4) % 2 == 0
    x[col] = _collapsed(int(col.sum()), D, seed=607)
    return x, lab


def test_local_rows_past_8192_columns(cuda, oracle):
    x, lab = _long_rows()
    Q, world = 4608, 2
    m = _mining(synth.LOCAL, -0.3, -0.1, REL_H, REL_E)
    S, refs = _run(oracle, x, lab, Q, world, m, tag="N 9216")
    lanes = np.concatenate([select_ref.local_warp_bins(S[r * Q:(r + 1) * Q], lab[r * Q:(r + 1) * Q], lab, r * Q, -0.1)["lane_max"]
                            for r in range(world)])
    n_over = int((lanes > select_ref.LSEL_LANE_CAP).sum())
    print(f"N = {x.shape[0]} > 8192; {n_over:,} rows overflow a lane list, {lanes.size - n_over:,} keep the fast path")
    assert x.shape[0] > 8192 and 0 < n_over < lanes.size
    assert np.mean(np.concatenate([r["nega_raw"] for r in refs]) >= 0) > 0.9


def test_local_rows_past_8192_columns_row_blocks(cuda):
    """The same batch with blocks of 1024 rows: the warp kernel reads each block through the row arrays' offsets, and every output is
    bit for bit that of the materialised run."""
    from test_gpu_sim_blocks import _compare
    x, lab = _long_rows()
    _compare(x, lab, 4608, 2, 1024, "N 9216 row blocks", **_mining(synth.LOCAL, -0.3, -0.1, REL_H, REL_E))


# ---------------------------------------------------------------------------------------------------------------------------------
# 7. same-label list sizes at the kernels' boundaries: 32 / 33 (counted in the warp) and 128 / 129 (kept list)
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ns", [31, 32, 33, 128, 129])
def test_same_label_list_boundaries(cuda, oracle, ns):
    """16 classes of ns + 1 images.  Both LOCAL kernels with both sides relative, and with the AN side alone (the warp kernel then
    keeps its histogram path while the same-label list fits its 128 slots); GLOBAL on the same data."""
    B, D = 16 * (ns + 1), 64
    x, lab = synth.make_inputs(B, D, seed=700 + ns, imgs_per_class=ns + 1, noise=1.5)
    same, _ = select_ref.side_masks(lab, lab, 0)
    assert (same.sum(axis=1) == ns).all()
    cases = [(synth.LOCAL, f, _mining(synth.LOCAL, -0.3, -0.4)) for f in (0, capi.FLAG_LSEL_WARP)]
    cases += [(synth.LOCAL, f, _mining(synth.LOCAL, -0.3, -0.4, ap_method=synth.HARD)) for f in (0, capi.FLAG_LSEL_WARP)]
    cases += [(synth.GLOBAL, 0, _mining(synth.GLOBAL, -0.3, -0.4, REL_E, REL_H))]
    for region, flags, m in cases:
        _run(oracle, x, lab, B, 1, m, tag=f"ns{ns} r{region} f{flags} ap{m['ap_method']}", flags=flags)
    print(f"ns = {ns} same-label entries per row")


# ---------------------------------------------------------------------------------------------------------------------------------
# 8. un-normalised embeddings in bf16x3: similarities over many binades, outliers stretching the block kernel's value range
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("region,flags", [(synth.GLOBAL, 0), (synth.LOCAL, 0), (synth.LOCAL, capi.FLAG_LSEL_WARP)])
def test_unnormalised_bf16x3(cuda, oracle, region, flags):
    """B = 1024, D = 64: directions normalize(e0 + 0.1 g) (cosines 0.3 .. 0.9, so every similarity keeps fp32's relative accuracy)
    scaled by norms 10^U(-2, 1): similarities from about 1e-5 to 90.  (Norms up to 100 would push exp(S - row max) of every positive
    below fp32's range in some rows, an infinite loss that says nothing about the selects.)"""
    B, D = 1024, 64
    rng = np.random.default_rng(808)
    x = _collapsed(B, D, seed=809, eps=0.1) * (10.0 ** rng.uniform(-2, 1, B)).astype(np.float32)[:, None]
    x = np.ascontiguousarray(x, np.float32)
    lab = _labels(B, 4)
    for identsn, diffsn in ((-0.3, -0.3), (-0.7, -0.05)):
        m = _mining(region, identsn, diffsn, REL_E, REL_H)
        S, _ = _run(oracle, x, lab, B, 1, m, prec=BF16X3, tag=f"unnormalised r{region} f{flags} sn{identsn},{diffsn}", flags=flags)
        off = np.abs(S[~np.eye(B, dtype=bool)])
        span = np.log2(off.max() / off.min())
        print(f"similarities span {span:.1f} binades")
        assert off.min() > 0 and span > 16
