"""k-means++ seeding on the GPU (npair_eval_kmeans_seed, DESIGN 8.2): rows and potential bit for bit against the host reference
(tests/kmeans_seed_ref.py) over sizes, trial counts, formats and seeds; edge sets; independence of the stream, the evaluator and earlier
calls; refusals that launch nothing; an SOP-sized run with its device memory; restarts through clustering_metrics; and planted blobs of
unequal sizes, which k-means++ seeds completely where random rows do not."""
import ctypes as C

import numpy as np
import pytest

import kmeans_seed_ref as R
from eval_ref import cuda

pytestmark = pytest.mark.gpu

FP16X2, BF16X3 = 2, 0


def _seed(ev, xt, k, seed, L):
    return ev.kmeans_seed(xt, k, seed, L)


def _evaluator(n, D, prec=FP16X2, k=1):
    from npairloss_b200 import capi
    return capi.Evaluator(n, k, D, prec)


@pytest.mark.parametrize("D", [1, 3, 100, 512, 1024])
@pytest.mark.parametrize("n", [1, 2, 31, 1000, 4099])
def test_rows_and_phi_bit_for_bit(n, D):
    rng = np.random.default_rng(20261017 + 7 * n + D)
    x = (rng.standard_normal((n, D)) * rng.uniform(0.1, 3.0)).astype(np.float32)
    P = R.Points(x)
    xt = cuda(x)
    ks = sorted({1, min(2, n), max(1, n // 3), n})
    evs = {p: _evaluator(n, D, p) for p in (FP16X2, BF16X3)}
    try:
        for ki, k in enumerate(ks):
            L = (1, 2, 0)[(ki + n + D) % 3]
            for si, seed in enumerate((ki + 1000 * n + D, 2 ** 64 - 1 - ki)):
                want = R.seed_rows(x, k, seed, L, points=P)
                prec = (FP16X2, BF16X3)[(ki + si) % 2]
                got = _seed(evs[prec], xt, k, seed, L)
                assert got == want, (n, D, k, L, seed, prec)
            assert _seed(evs[BF16X3], xt, k, seed, L) == _seed(evs[FP16X2], xt, k, seed, L)   # no dependence on the format
    finally:
        for ev in evs.values():
            ev.close()


def _check_set(x, k, seeds, L=0):
    P, xt = R.Points(x), cuda(x)
    ev = _evaluator(x.shape[0], x.shape[1])
    try:
        out = []
        for s in seeds:
            got = _seed(ev, xt, k, s, L)
            assert got == R.seed_rows(x, k, s, L, points=P), (k, s, L)
            out.append(got)
        return out
    finally:
        ev.close()


def test_edge_sets():
    rng = np.random.default_rng(11)
    same = np.tile(rng.standard_normal((1, 40)).astype(np.float32), (50, 1))
    for rows, phi in _check_set(same, 20, (0, 5), 2):                      # phi = 0 from the start: uniform rows
        assert phi == 0
    for rows, phi in _check_set(np.zeros((33, 8), np.float32), 33, (1,), 1):
        assert phi == 0
    base = rng.standard_normal((5, 16)).astype(np.float32)
    few = base[rng.integers(0, 5, size=60)]
    for rows, phi in _check_set(few, 12, (2, 3)):                          # k > the 5 distinct points
        assert phi == 0 and len({tuple(few[r]) for r in rows}) == 5
    dup = rng.standard_normal((300, 24)).astype(np.float32)
    dup[150:200] = dup[100:150]                                             # planted duplicates
    for rows, phi in _check_set(dup, 100, (4, 9), 3):
        assert len(set(rows)) == 100 and phi > 0
        assert len({dup[r].tobytes() for r in rows}) == 100                 # a copy of a centre is at distance 0: never drawn
    far = (0.01 * rng.standard_normal((500, 32))).astype(np.float32)
    far[277] = 100.0
    res = _check_set(far, 2, range(20), 1)
    assert sum(rows[1] == 277 for rows, _ in res) >= 18


def test_independence():
    import torch
    from npairloss_b200 import capi
    rng = np.random.default_rng(12)
    n, D, k = 3000, 96, 300
    x = rng.standard_normal((n, D)).astype(np.float32)
    xt = cuda(x)
    want = R.seed_rows(x, k, 77, 0)
    ev = capi.Evaluator(n, k, D)
    try:
        assert _seed(ev, xt, k, 77, 0) == want
        assert _seed(ev, xt, k, 77, 0) == want                              # repeated
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            assert _seed(ev, xt, k, 77, 0) == want                          # another stream
        torch.cuda.synchronize()
        ev.kmeans(xt, k, want[0], 3)
        ev.knn(xt, xt[:k], 5)
        assert _seed(ev, xt, k, 77, 0) == want                              # after kmeans / knn
        assert _seed(ev, xt[:1000], 100, 77, 0) == R.seed_rows(x[:1000], 100, 77, 0)   # a smaller set on the grown buffers
        assert _seed(ev, xt, k, 77, 0) == want
    finally:
        ev.close()
    big = capi.Evaluator(2 * n, 2 * k, D, BF16X3)                           # fresh, another capacity
    try:
        assert _seed(big, xt, k, 77, 0) == want
    finally:
        big.close()


def test_refusals_launch_nothing():
    import torch
    from npairloss_b200 import capi
    n, D = 64, 16
    x = cuda(np.random.default_rng(13).standard_normal((n, D)).astype(np.float32))
    ev = capi.Evaluator(n, 8, D)
    L = capi.lib()
    rows = (C.c_int32 * 200)()
    phi = C.c_uint64()
    try:
        _seed(ev, x, 3, 0, 1)                                               # loads the kernels
        torch.cuda.synchronize()
        n0 = capi.kernel_launches()
        bad = [(ev._h, x.data_ptr(), n, 0, 0, 0, rows), (ev._h, x.data_ptr(), n, n + 1, 0, 0, rows),
               (ev._h, x.data_ptr(), n, 3, 0, -1, rows), (ev._h, x.data_ptr(), n, 3, 0, 256, rows),
               (ev._h, x.data_ptr(), 0, 1, 0, 0, rows), (ev._h, x.data_ptr(), n + 1, 3, 0, 0, rows),
               (ev._h, None, n, 3, 0, 0, rows), (ev._h, x.data_ptr(), n, 3, 0, 0, None), (None, x.data_ptr(), n, 3, 0, 0, rows)]
        for h, xp, nn, k, seed, lt, rp in bad:
            assert L.npair_eval_kmeans_seed(h, xp, nn, k, seed, lt, rp, C.byref(phi), None) == -1, (nn, k, lt)
        assert capi.kernel_launches() == n0, "a refused call launched kernels"
        assert L.npair_eval_kmeans_seed(ev._h, x.data_ptr(), n, 3, 0, 255, rows, None, None) == 0   # L = 255, no phi
        assert capi.eval_kmeans_seed_bytes(n, D, 256) == 0 and capi.eval_kmeans_seed_bytes(0, D, 1) == 0
        for v in (float("nan"), float("inf")):
            y = x.clone()
            y[5, 3] = v
            with pytest.raises(capi.NpairError) as e:
                ev.kmeans_seed(y, 4, 0)
            assert e.value.code == -2
        assert _seed(ev, x, 4, 0, 0) == R.seed_rows(x.cpu().numpy(), 4, 0, 0)   # the evaluator still works
    finally:
        ev.close()


def test_sop_sized_run():
    """60 502 x 512 into k = 11 316 with L = 11 given: distinct rows, the first 64 those of the reference's k = 64 run, repeatable, and
    the device memory the call adds is npair_eval_kmeans_seed_bytes."""
    import time

    import torch
    from npairloss_b200 import capi
    n, k, D, L = 60502, 11316, 512, 11
    rng = np.random.default_rng(20261018)
    centres = rng.standard_normal((k, D)).astype(np.float32)
    x = centres[rng.integers(0, k, size=n)] + 0.6 * rng.standard_normal((n, D)).astype(np.float32) / np.sqrt(D)
    x = (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)
    xt = cuda(x)
    warm = _evaluator(64, D)
    _seed(warm, xt[:64], 4, 0, 1)                                           # loads the kernels
    warm.close()
    ev = capi.Evaluator(n, k, D)
    try:
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        t0 = time.perf_counter()
        rows, phi = _seed(ev, xt, k, 5, L)
        secs = time.perf_counter() - t0
        used = free0 - torch.cuda.mem_get_info()[0]
        want = capi.eval_kmeans_seed_bytes(n, D, L)
        assert want <= used <= want + (2 << 20), (used, want)               # allocation granularity
        assert len(set(rows)) == k and phi > 0
        assert rows[:64] == R.seed_rows(x, 64, 5, L)[0]
        assert _seed(ev, xt, k, 5, L) == (rows, phi)
    finally:
        ev.close()
    print(f"SOP-sized k-means++: {secs:.3f} s, {want / 1e6:.1f} MB")


def _blobs():
    """64 blobs of 5 .. 500 rows around unit centres scaled by 4, noise 0.01 per feature"""
    rng = np.random.default_rng(20261017)
    sizes = np.concatenate([[5, 500], rng.integers(5, 501, size=62)])
    c = rng.standard_normal((64, 48))
    c = c / np.linalg.norm(c, axis=1, keepdims=True) * 4
    lab = np.repeat(np.arange(64), sizes)
    return (c[lab] + 0.01 * rng.standard_normal((len(lab), 48))).astype(np.float32), lab


def test_restarts_keep_the_least_inertia():
    import torch
    from npairloss_b200.torch_api import clustering_metrics
    x, lab = _blobs()
    xt, lt = cuda(x), cuda(lab.astype(np.float32))
    R_ = 4
    for init in ("k-means++", "random"):
        singles = [clustering_metrics(xt, lt, k=40, seed=10 + r, max_iter=6, init=init) for r in range(R_)]
        out, a, c = clustering_metrics(xt, lt, k=40, seed=10, max_iter=6, init=init, n_init=R_)
        inert = [s[0]["inertia"] for s in singles]
        assert out["inertias"] == inert
        r = int(np.argmin(inert))
        assert out["restart"] == r and out["inertia"] == inert[r]
        assert torch.equal(a, singles[r][1]) and torch.equal(c.view(torch.int32), singles[r][2].view(torch.int32))
        assert all(s[0]["restart"] == 0 and len(s[0]["inertias"]) == 1 for s in singles)


def test_random_single_run_is_the_previous_call():
    import torch
    from npairloss_b200 import capi
    from npairloss_b200.torch_api import clustering_metrics
    x, lab = _blobs()
    xt, lt = cuda(x), cuda(lab.astype(np.float32))
    out, a, c = clustering_metrics(xt, lt, seed=3, max_iter=5, init="random", n_init=1)
    init = torch.randperm(x.shape[0], generator=torch.Generator().manual_seed(3))[:64].tolist()
    ev = capi.Evaluator(x.shape[0], 64, x.shape[1])
    try:
        res = ev.kmeans(xt, 64, init, 5)
    finally:
        ev.close()
    assert torch.equal(a, res["assign"]) and torch.equal(c.view(torch.int32), res["centroids"].view(torch.int32))
    assert out["inertia"] == float(res["inertia"]) and out["restart"] == 0


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_planted_blobs_kmeanspp_finds_every_blob(seed):
    """Fixed seeds: k-means++ puts one centre in each of the 64 blobs and Lloyd's iterations recover the labels (NMI = F1 = 1); random
    rows leave some blob without a centre, and a neighbour keeps it."""
    import torch
    from npairloss_b200.torch_api import clustering_metrics
    x, lab = _blobs()
    xt, lt = cuda(x), cuda(lab.astype(np.float32))
    ev = _evaluator(x.shape[0], x.shape[1])
    try:
        rows, _ = ev.kmeans_seed(xt, 64, seed)
    finally:
        ev.close()
    assert len(set(lab[rows])) == 64
    out, _, _ = clustering_metrics(xt, lt, seed=seed, max_iter=20, init="k-means++")
    assert out["nmi"] == 1.0 and out["f1"] == 1.0, out
    rnd = torch.randperm(x.shape[0], generator=torch.Generator().manual_seed(seed))[:64].tolist()
    assert len(set(lab[rnd])) < 64
    out_r, _, _ = clustering_metrics(xt, lt, seed=seed, max_iter=20, init="random")
    assert out_r["nmi"] < 1.0
