"""k-means on the GPU (DESIGN 8.2): the first assignment against an exact host argmax with planted ties; the fixed-point centroid update
against a numpy loop, bit for bit; the assignment as the argmin for the returned centroids within the format's error bound; convergence
on planted blobs; repeatability; the torch API's NMI / F1 against a numpy oracle; and an SOP-sized run with its device memory."""
import numpy as np
import pytest

from eval_ref import cuda, update_ref

pytestmark = pytest.mark.gpu

PRECS = (0, 1, 2)          # capi.PREC_FP32_BF16X3, PREC_BF16, PREC_FP32_FP16X2


def _unit_rows(n, D, rng):
    x = rng.standard_normal((n, D)).astype(np.float32)
    return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)


def _lowdim(n, D, rng):
    """Points near a random 3-dimensional subspace: Lloyd's iterations take a dozen or more sweeps to settle, unlike random unit vectors
    in many dimensions, which settle in two or three"""
    z = rng.standard_normal((n, 3)) @ rng.standard_normal((3, D))
    return (z / np.sqrt(D) + 0.02 * rng.standard_normal((n, D))).astype(np.float32)


def _kmeans(x, k, init, max_iter, prec, ev=None):
    from npairloss_b200 import capi
    own = ev is None
    if own:
        ev = capi.Evaluator(x.shape[0], k, x.shape[1], prec)
    try:
        r = ev.kmeans(x, k, init, max_iter)
        return {"assign": r["assign"].cpu().numpy(), "centroids": r["centroids"].cpu().numpy(), "inertia": float(r["inertia"]),
                "stats": (r["iterations"], r["changed"], r["empty"])}
    finally:
        if own:
            ev.close()


def test_first_assignment_exact_with_planted_ties():
    """Entries k/8: every similarity, bias and score is exact in every format, so the assignment is the int64 argmax, lowest index on
    ties.  Centroid pairs with identical vectors (a copied row, a repeated init index) tie for every point: the higher one is empty."""
    from npairloss_b200 import capi
    n, k, D = 3000, 300, 200
    rng = np.random.default_rng(20260811)
    K = rng.integers(-8, 9, size=(n, D)).astype(np.int64)
    init = rng.choice(n, size=k, replace=False)
    for lo, hi in ((3, 7), (10, 20), (50, 299), (0, 150)):
        K[init[hi]] = K[init[lo]]                      # same vector under two indices
    init[200] = init[40]                               # the same row twice
    x = (K / 8.0).astype(np.float32)
    Kc = K[init]
    score = 2 * K @ Kc.T - (Kc * Kc).sum(1)[None, :]   # 128 * (s - 0.5 ||mu||^2), exact
    want = np.argmax(score, axis=1)                    # first maximum: lowest index
    planted = [7, 20, 299, 150, 200]
    assert not np.isin(planted, want).any()
    xt = cuda(x)
    for prec in PRECS:
        r = _kmeans(xt, k, init.tolist(), 1, prec)
        np.testing.assert_array_equal(r["assign"], want, err_msg=f"prec {prec}")
        np.testing.assert_array_equal(r["centroids"], x[init])
        empty = k - len(np.unique(want))
        assert r["stats"] == (1, n, empty), (prec, r["stats"], empty)
        assert capi.eval_kmeans_bytes(n, k, D) > 0


@pytest.mark.parametrize("prec", PRECS)
def test_update_rule_bit_for_bit(prec):
    """C_{t+1} of the run with max_iter = t + 1 is the numpy fixed-point update of the assignment and centroids of the run with
    max_iter = t; a repeated init row gives an empty cluster, which keeps its centroid."""
    n, k, D = 3000, 300, 200
    rng = np.random.default_rng(20260812 + prec)
    x = _lowdim(n, D, rng)
    init = rng.choice(n, size=k, replace=False)
    init[250] = init[5]
    xt = cuda(x)
    prev = _kmeans(xt, k, init.tolist(), 1, prec)
    for t in range(1, 5):
        nxt = _kmeans(xt, k, init.tolist(), t + 1, prec)
        assert prev["stats"][0] == t and nxt["stats"][0] == t + 1, (t, prev["stats"], nxt["stats"])
        want = update_ref(x, prev["assign"], prev["centroids"])
        np.testing.assert_array_equal(nxt["centroids"].view(np.uint32), want.view(np.uint32), err_msg=f"t={t}")
        empty = np.setdiff1d(np.arange(k), prev["assign"])
        if t == 1:
            assert 250 in empty                        # ties with centroid 5 in the first sweep
        np.testing.assert_array_equal(nxt["centroids"][empty], prev["centroids"][empty])
        prev = nxt


def _score_bound(prec, xd, Cd, M):
    """Bound on |library score - exact score| for every (point, centroid), from the operand error of DESIGN 5 (per point i and
    centroid c: L1 = ||x_i||_1, m = max|mu_c|, n2 = ||mu_c||^2, exact similarity |s| <= L1 * m):
      fp16x2: a pre-scaled operand piece pair hi + lo misses x * sigma by <= 2^-22, i.e. x by <= 2^-22 / sigma <= 2^-21 M (M = max|x|
              bounds every centroid too), and the dropped lo.lo product is <= 2^-22 / sigma^2 <= 2^-20 M^2 per feature:
              2^-21 M (L1 + ||mu_c||_1) + D 2^-20 M^2
      bf16x3: hi + mid + lo is 2^-24 relative and the dropped products are as small: 2^-22 L1 m (a factor 4 of slack)
      bf16  : each operand rounded to 2^-9 relative, (1 + 2^-9)^2 - 1 < 2^-7.9: 2^-7 L1 m
    plus the fp32 accumulation of passes * D products (passes * D * 2^-24 L1 m), the fp32 bias (a chain of D / 32 fmaf per lane and a
    5-level tree: (D / 32 + 6) 2^-24 n2 / 2) and the rounding of the difference (2^-24 (L1 m + n2 / 2))."""
    import torch
    D = xd.shape[1]
    L1 = xd.abs().sum(1, keepdim=True)
    m = Cd.abs().max(1).values[None, :]
    n2 = (Cd * Cd).sum(1)[None, :]
    passes = {0: 6, 1: 1, 2: 3}[prec]
    u = 2.0 ** -24
    if prec == 2:
        op = 2.0 ** -21 * M * (L1 + Cd.abs().sum(1)[None, :]) + D * 2.0 ** -20 * M * M
    elif prec == 0:
        op = 2.0 ** -22 * L1 * m
    else:
        op = 2.0 ** -7 * L1 * m
    b = op + passes * D * u * L1 * m + (D / 32 + 6) * u * n2 / 2 + u * (L1 * m + n2 / 2)
    return b.to(torch.float64)


def _check_argmin(prec, xt, assign, C, rows=None):
    """Every point's score for its centroid is within the bound of the best score, and a point whose best beats every other centroid by
    more than twice the bound is assigned to it exactly.  Returns the number of points checked exactly."""
    import torch
    xd = xt.double() if rows is None else xt[rows].double()
    a = torch.as_tensor(assign, device=xd.device).long()
    if rows is not None:
        a = a[rows]
    Cd = torch.as_tensor(C, device=xd.device).double()
    M = float(xt.abs().max())
    score = xd @ Cd.T - 0.5 * (Cd * Cd).sum(1)[None, :]
    bound = _score_bound(prec, xd, Cd, M)
    best, arg = score.max(1)
    r = torch.arange(len(a), device=xd.device)
    chosen = score[r, a]
    tol = bound[r, a] + bound[r, arg]
    assert bool((best - chosen <= tol).all()), float((best - chosen - tol).max())
    second = score.clone()
    second[r, arg] = -float("inf")
    clear = best - second.max(1).values > 2 * bound.max(1).values
    assert bool((a[clear] == arg[clear]).all())
    return int(clear.sum())


@pytest.mark.parametrize("prec", PRECS)
def test_assignment_is_argmin_after_updates(prec):
    n, k, D = 3000, 300, 200
    rng = np.random.default_rng(20260813 + prec)
    x = _lowdim(n, D, rng)
    init = rng.choice(n, size=k, replace=False)
    xt = cuda(x)
    r = _kmeans(xt, k, init.tolist(), 5, prec)
    assert r["stats"][0] == 5
    exact = _check_argmin(prec, xt, r["assign"], r["centroids"])
    assert exact > (n // 2 if prec != 1 else 0), exact        # bf16's bound leaves few clear winners


def _blobs(n_per, k, D, rng):
    centers = _unit_rows(k, D, rng) * np.float32(4.0)
    lab = np.repeat(np.arange(k), n_per)
    x = (centers[lab] + 0.05 * rng.standard_normal((n_per * k, D))).astype(np.float32)
    return x, lab


@pytest.mark.parametrize("prec", PRECS)
def test_converges_on_planted_blobs(prec):
    from npairloss_b200.torch_api import clustering_scores
    import torch
    k, n_per, D = 20, 100, 72
    rng = np.random.default_rng(20260814 + prec)
    x, lab = _blobs(n_per, k, D, rng)
    init = [c * n_per + int(rng.integers(n_per)) for c in range(k)]      # one row per blob, in blob order
    xt = cuda(x)
    r = _kmeans(xt, k, init, 20, prec)
    it, changed, empty = r["stats"]
    assert changed == 0 and it < 20 and empty == 0, r["stats"]
    np.testing.assert_array_equal(r["assign"], lab)
    nmi, f1 = clustering_scores(torch.from_numpy(lab.astype(np.float32)), torch.from_numpy(r["assign"]))
    assert nmi == 1.0 and f1 == 1.0, (nmi, f1)
    C = r["centroids"].astype(np.float64)
    ref = float(((x.astype(np.float64) - C[r["assign"]]) ** 2).sum())
    assert abs(r["inertia"] - ref) <= 1e-12 * ref, (r["inertia"], ref)


@pytest.mark.parametrize("prec", PRECS)
def test_repeatable(prec):
    from npairloss_b200 import capi
    n, k, D = 2500, 130, 96
    rng = np.random.default_rng(20260815 + prec)
    x = _unit_rows(n, D, rng)
    init = rng.choice(n, size=k, replace=False).tolist()
    xt = cuda(x)
    ev = capi.Evaluator(n, k, D, prec)
    try:
        runs = [_kmeans(xt, k, init, 8, prec, ev), _kmeans(xt, k, init, 8, prec, ev)]
    finally:
        ev.close()
    runs.append(_kmeans(xt, k, init, 8, prec))
    a = runs[0]
    for b in runs[1:]:
        np.testing.assert_array_equal(a["assign"], b["assign"])
        np.testing.assert_array_equal(a["centroids"].view(np.uint32), b["centroids"].view(np.uint32))
        assert np.float64(a["inertia"]).view(np.uint64) == np.float64(b["inertia"]).view(np.uint64)
        assert a["stats"] == b["stats"]


def _nmi_f1_ref(lab, assign):
    """numpy oracle: contingency table by a dense bincount over the non-empty labels and clusters"""
    _, y = np.unique(lab, return_inverse=True)
    _, c = np.unique(assign, return_inverse=True)
    L, K, n = y.max() + 1, c.max() + 1, len(y)
    T = np.bincount(y * K + c, minlength=L * K).reshape(L, K).astype(np.float64)
    nl, nc = T.sum(1), T.sum(0)
    nz = T > 0
    mi = (T[nz] / n * np.log(n * T[nz] / np.outer(nl, nc)[nz])).sum()
    hy, hc = -(nl / n * np.log(nl / n)).sum(), -(nc / n * np.log(nc / n)).sum()
    nmi = 1.0 if hy + hc == 0 else 2 * mi / (hy + hc)
    comb = lambda m: (m * (m - 1) / 2).sum()
    tp, pc, pl = comb(T), comb(nc), comb(nl)
    p, r = (tp / pc if pc else 0.0), (tp / pl if pl else 0.0)
    return nmi, (2 * p * r / (p + r) if p + r > 0 else 0.0)


def test_clustering_metrics_api():
    import torch
    from npairloss_b200 import capi
    from npairloss_b200.torch_api import clustering_metrics
    rng = np.random.default_rng(20260816)
    n_lab, per, D = 60, 5, 128
    centers = _unit_rows(n_lab, D, rng)
    lab = np.repeat(np.arange(n_lab), per).astype(np.float32) * 3.0 - 7.0
    x = centers[np.repeat(np.arange(n_lab), per)] + 0.35 * rng.standard_normal((n_lab * per, D)).astype(np.float32)
    x = (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)
    xt, lt = cuda(x), cuda(lab).to(torch.int64)
    out, assign, cent = clustering_metrics(xt, lt, seed=3)
    assert cent.shape == (n_lab, D) and assign.shape == (n_lab * per,)           # k=None: the number of labels
    nmi, f1 = _nmi_f1_ref(lab, assign.cpu().numpy())
    assert abs(out["nmi"] - nmi) <= 1e-12 and abs(out["f1"] - f1) <= 1e-12, (out, nmi, f1)
    assert 0.5 < out["nmi"] <= 1.0 and 0.0 < out["f1"] <= 1.0
    assert out["iterations"] >= 1 and isinstance(out["converged"], bool) and out["empty_clusters"] >= 0
    again, assign2, cent2 = clustering_metrics(xt, lt, seed=3)
    assert again == out
    assert torch.equal(assign, assign2) and torch.equal(cent, cent2)
    out7, _, c7 = clustering_metrics(xt, lt, k=7, seed=1, max_iter=3, precision=capi.PREC_FP32_BF16X3)
    assert c7.shape == (7, D) and out7["iterations"] <= 3
    with pytest.raises(TypeError):
        clustering_metrics(xt.cpu(), lt.cpu())
    with pytest.raises(ValueError):
        clustering_metrics(xt[:5], lt[:5], k=6)
    ev = capi.Evaluator(100, 10, D)
    try:
        with pytest.raises(capi.NpairError):
            ev.kmeans(xt[:100], 10, [0] * 9 + [100], 5)                      # row index out of range
        with pytest.raises(capi.NpairError):
            ev.kmeans(xt[:100], 10, list(range(10)), 0)                      # max_iter < 1
        with pytest.raises(capi.NpairError):
            ev.kmeans(xt[:100], 11, list(range(11)), 5)                      # beyond the gallery capacity
    finally:
        ev.close()


def test_sop_sized_run():
    """60 502 x 512 into k = 11 316 (Stanford Online Products' test set and its number of classes), fp16x2, 5 iterations."""
    import torch
    from npairloss_b200 import capi
    n, k, D, prec = 60502, 11316, 512, 2
    rng = np.random.default_rng(20260817)
    centers = _unit_rows(k, D, rng)
    x = centers[rng.integers(0, k, size=n)] + 0.6 * rng.standard_normal((n, D)).astype(np.float32) / np.sqrt(D)
    x = (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)
    xt = cuda(x)
    init = rng.choice(n, size=k, replace=False).tolist()
    ws, km = capi.eval_workspace_bytes(n, k, D, prec), capi.eval_kmeans_bytes(n, k, D)
    _kmeans(xt[:512], 16, list(range(16)), 2, prec)                            # loads the kernels
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    ev = capi.Evaluator(n, k, D, prec)
    try:
        res = ev.kmeans(xt, k, init, 5)
        torch.cuda.synchronize()
        used = free0 - torch.cuda.mem_get_info()[0]
    finally:
        ev.close()
    outputs = k * D * 4 + n * 4 + 8
    assert ws + km <= used <= ws + km + outputs + (64 << 20), (ws, km, used)
    assert res["iterations"] == 5
    C = res["centroids"]
    assert not bool(torch.isnan(C).any()) and not np.isnan(float(res["inertia"]))
    a = res["assign"]
    assert int(a.min()) >= 0 and int(a.max()) < k
    rows = torch.from_numpy(rng.choice(n, size=2048, replace=False)).cuda()
    exact = _check_argmin(prec, xt, a, C, rows)
    print(f"SOP-sized: workspace {ws / 1e6:.1f} MB + k-means {km / 1e6:.1f} MB, allocated {used / 1e6:.1f} MB, "
          f"inertia {float(res['inertia']):.6f}, empty {res['empty']}, {exact} of 2048 sampled rows checked exactly")
