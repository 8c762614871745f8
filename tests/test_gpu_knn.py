"""Exact k nearest neighbours on the GPU (npair_eval_knn, DESIGN 8.3): the lists against a numpy lexsort of the layer's own fp32 S and of
exact int64 similarities with planted ties, independence of the block height, the set forms and gallery shards merged two ways,
agreement with the rank and Recall@K of the evaluator, rows past the shared-memory capacity with thousands of tied entries, the NaN rule,
repeatability, argument checks without launches, and an SOP-sized run with its device memory."""
import ctypes as C

import numpy as np
import pytest

from eval_ref import cuda, planted

pytestmark = pytest.mark.gpu

PRECS = (0, 1, 2)          # capi.PREC_FP32_BF16X3, PREC_BF16, PREC_FP32_FP16X2
E_ARG = -1
NPAIR_MAX_K = 1024         # NPAIR_EVAL_KNN_MAX_K


def ref_knn(S, k, self_offset=-1, gallery_row0=0):
    """The call's order over given similarities S [nq, ng] (fp32, or exact int64): s descending, NaN after every number, then column
    ascending; query i's own column self_offset - gallery_row0 + i excluded.  Returns (values [nq, k], global indices [nq, k])."""
    nq, ng = S.shape
    s = S.astype(np.float64)
    nan = np.isnan(s)
    excl = np.zeros((nq, ng), bool)
    if self_offset >= 0:
        i = np.arange(nq)
        c = self_offset - gallery_row0 + i
        ok = (c >= 0) & (c < ng)
        excl[i[ok], c[ok]] = True
    cols = np.broadcast_to(np.arange(ng), (nq, ng))
    order = np.lexsort((cols, np.where(nan, 0.0, -s), nan, excl), axis=-1)[:, :k]
    return np.take_along_axis(S, order, 1), order + gallery_row0


def _knn(ev, q, g, k, **kw):
    sim, idx = ev.knn(q, g, k, **kw)
    return sim.cpu().numpy(), idx.cpu().numpy().astype(np.int64)


def _same(got, want_vals, want_idx):
    sim, idx = got
    np.testing.assert_array_equal(idx, want_idx)
    np.testing.assert_array_equal(np.isnan(sim), np.isnan(want_vals.astype(np.float64)))
    ok = ~np.isnan(sim)
    np.testing.assert_array_equal(sim[ok], np.asarray(want_vals, np.float64)[ok].astype(np.float32))


def _exact(Kq, Kg):
    """int64 similarities of planted rows (entries k/8): s = (Kq Kg^T) / 64, exact in fp32"""
    return (Kq @ Kg.T).astype(np.float64) / 64.0


@pytest.mark.parametrize("prec", PRECS)
def test_bits_of_the_layers_similarities(prec):
    """The lists are the layer's own fp32 S, bit for bit: random unit rows at a ragged D (world 1, S materialised)."""
    from npairloss_b200 import capi
    rng = np.random.default_rng(20261017 + prec)
    n, D = 1000, 100
    x = rng.standard_normal((n, D)).astype(np.float32)
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    lab = rng.integers(0, n // 3, size=n).astype(np.float32)
    xt = cuda(x)
    ctx = capi.Context(capi.make_config(n, D, sim_precision=prec))
    ctx.forward(xt, cuda(lab))
    S = ctx.debug_read(0, n * n).reshape(n, n)
    ctx.close()
    ev = capi.Evaluator(n, n, D, prec)
    try:
        for k in (1, 7, 64, 999):
            sim, idx = _knn(ev, xt, xt, k, self_offset=0)
            v, i = ref_knn(S, k, 0)
            np.testing.assert_array_equal(idx, i, err_msg=f"k={k}")
            np.testing.assert_array_equal(sim.view(np.uint32), v.view(np.uint32), err_msg=f"k={k}")
    finally:
        ev.close()


@pytest.mark.parametrize("prec", PRECS)
def test_ties_lowest_index_wins(prec):
    """Planted entries k/8 (every similarity exact in every format) and a gallery with 600 copies of the all-ones row: for a query of
    all ones they are the row's largest similarity, the k-th boundary falls inside that run of equal values, and the lowest indices win."""
    from npairloss_b200 import capi
    rng = np.random.default_rng(20261018 + prec)
    nq, ng, D = 300, 1500, 64
    Kg, _ = planted(ng, D, 50, rng)
    dup = rng.choice(ng, size=600, replace=False)
    Kg[dup] = 8
    Kq = rng.integers(-8, 9, size=(nq, D)).astype(np.int64)
    Kq[:5] = 8
    q, g = cuda((Kq / 8.0).astype(np.float32)), cuda((Kg / 8.0).astype(np.float32))
    E = _exact(Kq, Kg)
    ev = capi.Evaluator(nq, ng, D, prec)
    try:
        for k in (10, 100, 512):
            v, i = ref_knn(E, k)
            _same(_knn(ev, q, g, k), v, i)
            np.testing.assert_array_equal(i[0], np.sort(dup)[:k])
    finally:
        ev.close()


def test_block_heights_and_ragged_shapes():
    """block_rows 128, 256, 0 (default) and >= nq give the same bits; nq ragged, ng a multiple of neither 32 nor 256."""
    from npairloss_b200 import capi
    rng = np.random.default_rng(20261019)
    nq, ng, D = 601, 1003, 72
    Kq = rng.integers(-8, 9, size=(nq, D)).astype(np.int64)
    Kg, _ = planted(ng, D, 40, rng)
    q, g = cuda((Kq / 8.0).astype(np.float32)), cuda((Kg / 8.0).astype(np.float32))
    v, i = ref_knn(_exact(Kq, Kg), 33)
    ev = capi.Evaluator(nq, ng, D, 2)
    try:
        for br in (128, 256, 0, 640, 4096):
            _same(_knn(ev, q, g, 33, block_rows=br), v, i)
    finally:
        ev.close()


def test_set_forms_and_shards():
    """Disjoint sets, self-retrieval, queries that are gallery rows o, o+1, ... (self_offset > 0), and the gallery split into three
    uneven shards (gallery_row0, shared absmax) merged with knn_merge and with numpy: each equals the one call."""
    import torch
    from npairloss_b200 import capi
    from npairloss_b200.torch_api import knn, knn_merge
    rng = np.random.default_rng(20261020)
    ng, D, k = 1111, 48, 40
    Kg, _ = planted(ng, D, 30, rng)
    g = cuda((Kg / 8.0).astype(np.float32))
    E = _exact(Kg, Kg)
    # self-retrieval through the torch API
    sim, idx = knn(g, k=k)
    assert idx.dtype == torch.int64
    v, i = ref_knn(E, k, 0)
    _same((sim.cpu().numpy(), idx.cpu().numpy()), v, i)
    # queries = gallery rows 300 .. 699
    o, nq = 300, 400
    q = g[o:o + nq].contiguous()
    sim, idx = knn(q, g, k=k, self_offset=o, block_rows=128)
    v, i = ref_knn(E[o:o + nq], k, o)
    _same((sim.cpu().numpy(), idx.cpu().numpy()), v, i)
    # disjoint
    Kq = rng.integers(-8, 9, size=(nq, D)).astype(np.int64)
    qd = cuda((Kq / 8.0).astype(np.float32))
    sim, idx = knn(qd, g, k=k)
    v, i = ref_knn(_exact(Kq, Kg), k)
    _same((sim.cpu().numpy(), idx.cpu().numpy()), v, i)
    # three uneven shards of the gallery against queries = rows o .. o + nq (self columns in two of them)
    absmax = float(g.abs().max())
    ev = capi.Evaluator(nq, ng, D, 2)
    try:
        one = ev.knn(q, g, k, self_offset=o)
        parts = []
        for a, b in ((0, 350), (350, 500), (500, ng)):
            parts.append(ev.knn(q, g[a:b].contiguous(), k, self_offset=o, gallery_row0=a, absmax=absmax))
    finally:
        ev.close()
    ms, mi = knn_merge([p[0] for p in parts], [p[1] for p in parts], k)
    np.testing.assert_array_equal(mi.cpu().numpy(), one[1].cpu().numpy())
    np.testing.assert_array_equal(ms.cpu().numpy().view(np.uint32), one[0].cpu().numpy().view(np.uint32))
    # numpy: concatenate the shard lists and lexsort them by the same order
    s_all = np.concatenate([p[0].cpu().numpy() for p in parts], 1)
    i_all = np.concatenate([p[1].cpu().numpy() for p in parts], 1).astype(np.int64)
    order = np.lexsort((i_all, -s_all.astype(np.float64)), axis=-1)[:, :k]
    np.testing.assert_array_equal(np.take_along_axis(i_all, order, 1), one[1].cpu().numpy())


def test_agrees_with_rank_and_recall():
    """Where a query's list reaches below its best positive p*, #{list entries >= p*} is Evaluator.rank (planted ties); on random unit
    rows Recall@K from knn(k = 8) (a positive among the first K) equals recall_at_k for K <= 8."""
    from npairloss_b200 import capi
    from npairloss_b200.torch_api import knn, recall_at_k
    rng = np.random.default_rng(20261021)
    n, D, k = 1500, 64, 256
    K, lab = planted(n, D, 200, rng)
    x, lt = cuda((K / 8.0).astype(np.float32)), cuda(lab)
    ev = capi.Evaluator(n, n, D, 2)
    try:
        rank = ev.rank(x, lt, x, lt, 0).cpu().numpy()
        best = ev.best_positive(x, lt, x, lt, float(x.abs().max()), 0).cpu().numpy()
        sim, _ = _knn(ev, x, x, k, self_offset=0)
    finally:
        ev.close()
    reach = (best > -np.inf) & (sim[:, -1] < best)
    assert reach.sum() >= n // 4
    np.testing.assert_array_equal((sim[reach] >= best[reach, None]).sum(1), rank[reach])
    # no ties: random unit rows
    xr = rng.standard_normal((n, 128)).astype(np.float32)
    xr /= np.linalg.norm(xr, axis=1, keepdims=True)
    lab2 = rng.integers(0, 300, size=n).astype(np.float32)
    xt, lt2 = cuda(xr), cuda(lab2)
    rec, _ = recall_at_k(xt, lt2, ks=range(1, 9))
    _, idx = knn(xt, k=8)
    hit = lab2[idx.cpu().numpy()] == lab2[:, None]
    for kk in range(1, 9):
        assert hit[:, :kk].any(1).sum() / n == rec[kk], kk


def test_long_rows_with_mass_ties():
    """ng = 20000 columns (past the shared-memory capacity of 8192 keys): a run of 9000 copies of one row (its bin exceeds the capacity:
    every digit is taken from S) and one of 3000 copies of another (compacted), with queries for which each run is the top of the row
    (the k-th value is shared by thousands of entries), one for which a run is the bottom, and random ones."""
    from npairloss_b200 import capi
    rng = np.random.default_rng(20261022)
    nq, ng, D = 260, 20000, 64
    Kg = rng.integers(-8, 9, size=(ng, D)).astype(np.int64)
    perm = rng.permutation(ng)
    run_a, run_b = perm[:9000], perm[9000:12000]
    Kg[run_a] = 8                           # all ones: the largest similarity any row can have with a query of all ones
    Kg[run_b] = -8
    Kq = rng.integers(-8, 9, size=(nq, D)).astype(np.int64)
    Kq[0] = Kg[run_a[0]]
    Kq[1] = Kg[run_b[0]]
    Kq[2] = -Kg[run_a[0]]                   # the run is at the bottom of this row
    q, g = cuda((Kq / 8.0).astype(np.float32)), cuda((Kg / 8.0).astype(np.float32))
    E = _exact(Kq, Kg)
    ev = capi.Evaluator(nq, ng, D, 2)
    try:
        for k in (1, 100, 1024):
            v, i = ref_knn(E, k)
            _same(_knn(ev, q, g, k, block_rows=128), v, i)
            np.testing.assert_array_equal(i[0], np.sort(run_a)[:k])
            np.testing.assert_array_equal(i[1], np.sort(run_b)[:k])
    finally:
        ev.close()


def test_nan_rule():
    """A gallery row of NaN features ranks last for every query; a query of NaN features returns its first k non-self columns, in order,
    with NaN values."""
    from npairloss_b200 import capi
    rng = np.random.default_rng(20261023)
    n, D = 700, 32
    K = rng.integers(-8, 9, size=(n, D)).astype(np.int64)
    x = (K / 8.0).astype(np.float32)
    x[5] = np.nan                           # a NaN query (and gallery row)
    E = _exact(K, K)
    E[5, :] = np.nan
    E[:, 5] = np.nan
    xt = cuda(x)
    ev = capi.Evaluator(n, n, D, 2)
    try:
        sim, idx = _knn(ev, xt, xt, n - 1, self_offset=0, absmax=1.0)
    finally:
        ev.close()
    v, i = ref_knn(E, n - 1, 0)
    _same((sim, idx), v, i)
    others = np.arange(n) != 5
    assert np.all(idx[others, -1] == 5) and np.isnan(sim[others, -1]).all()
    np.testing.assert_array_equal(idx[5], np.delete(np.arange(n), 5))
    assert np.isnan(sim[5]).all()


def test_repeatable_on_fresh_evaluator():
    import torch
    from npairloss_b200 import capi
    rng = np.random.default_rng(20261024)
    nq, ng, D = 500, 9000, 96
    q = cuda(rng.standard_normal((nq, D)).astype(np.float32))
    g = cuda(rng.standard_normal((ng, D)).astype(np.float32))
    runs = []
    for fresh in (False, False, True):
        ev = capi.Evaluator(nq, ng, D, 2)
        try:
            runs.append(_knn(ev, q, g, 200))
            if not fresh:
                s = torch.cuda.Stream()
                with torch.cuda.stream(s):
                    runs.append(_knn(ev, q, g, 200, block_rows=128))
                torch.cuda.synchronize()
        finally:
            ev.close()
    for r in runs[1:]:
        np.testing.assert_array_equal(r[1], runs[0][1])
        np.testing.assert_array_equal(r[0].view(np.uint32), runs[0][0].view(np.uint32))


def test_bad_arguments_launch_nothing():
    import torch
    from npairloss_b200 import capi
    nq, ng, D = 64, 200, 16
    q = torch.randn(nq, D, device="cuda")
    g = torch.randn(ng, D, device="cuda")
    sim = torch.empty(nq, 1024, device="cuda")
    idx = torch.empty(nq, 1024, dtype=torch.int32, device="cuda")
    ev = capi.Evaluator(nq, ng, D, 2)
    L = capi.lib()
    st = torch.cuda.current_stream().cuda_stream
    base = dict(q=q.data_ptr(), nq=nq, g=g.data_ptr(), ng=ng, off=-1, row0=0, absmax=-1.0, k=10, br=0, s=sim.data_ptr(), i=idx.data_ptr())
    bad = [dict(nq=0), dict(ng=0), dict(nq=nq + 1), dict(ng=ng + 1), dict(q=None), dict(g=None), dict(s=None), dict(i=None),
           dict(k=0), dict(k=NPAIR_MAX_K + 1), dict(k=ng + 1), dict(off=0, k=ng), dict(off=-2), dict(row0=-1),
           dict(row0=2 ** 31 - 100), dict(absmax=float("nan")), dict(absmax=float("inf")), dict(br=100), dict(br=-128)]
    try:
        _knn(ev, q, g, 10)                  # loads the kernels
        torch.cuda.synchronize()
        n0 = capi.kernel_launches()
        for b in bad:
            a = {**base, **b}
            rc = L.npair_eval_knn(ev._h, a["q"], a["nq"], a["g"], a["ng"], a["off"], a["row0"], C.c_float(a["absmax"]), a["k"], a["br"],
                                  a["s"], a["i"], st)
            assert rc == E_ARG, b
        assert L.npair_eval_knn(None, None, 0, None, 0, 0, 0, C.c_float(0.0), 0, 0, None, None, None) == E_ARG
        assert capi.kernel_launches() == n0, "a refused call launched kernels"
        # the limits themselves are accepted: k = ng without a self column in the shard, k = ng - 1 with one
        _knn(ev, q, g, ng)
        _knn(ev, q, g, ng - 1, self_offset=0)
        _knn(ev, q, g, ng, self_offset=ng, gallery_row0=0, absmax=1.0)
    finally:
        ev.close()



def test_sop_sized_run():
    """60 502 x 512 self-retrieval (Stanford Online Products' test set), fp16x2, k = 100, default block: the device memory the call adds,
    and on 2048 sampled rows the returned set against fp64 brute force within the format's error bound."""
    import torch
    from npairloss_b200 import capi
    n, D, k, prec = 60502, 512, 100, 2
    rng = np.random.default_rng(20261025)
    centers = rng.standard_normal((11316, D)).astype(np.float32)
    x = centers[rng.integers(0, 11316, size=n)] + 0.8 * rng.standard_normal((n, D)).astype(np.float32)
    x = (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)
    xt = cuda(x)
    ws, kb = capi.eval_workspace_bytes(n, n, D, prec), capi.eval_knn_bytes(n, k, 0)
    ev0 = capi.Evaluator(512, 512, D, prec)                 # loads the kernels
    ev0.knn(xt[:512].contiguous(), xt[:512].contiguous(), 8, self_offset=0)
    ev0.close()
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    ev = capi.Evaluator(n, n, D, prec)
    try:
        sim, idx = ev.knn(xt, xt, k, self_offset=0)
        torch.cuda.synchronize()
        used = free0 - torch.cuda.mem_get_info()[0]
    finally:
        ev.close()
    outputs = n * k * 8
    assert ws + kb <= used <= ws + kb + outputs + (64 << 20), (ws, kb, used)
    rows = torch.from_numpy(rng.choice(n, size=2048, replace=False)).cuda()
    xd = xt.double()
    E = xd[rows] @ xd.T
    E[torch.arange(2048, device="cuda"), rows] = -float("inf")
    M = float(xt.abs().max())
    L1 = float(xt.abs().sum(1).max())
    u = 2.0 ** -24
    eps = 2.0 ** -21 * M * 2 * L1 + D * 2.0 ** -20 * M * M + 3 * D * u * L1 * M + u     # DESIGN 5: fp16x2 operand and accumulation error
    s, ix = sim[rows].double(), idx[rows].long()
    assert bool(((s - E.gather(1, ix)).abs() <= eps).all())
    assert bool((s[:, :-1] >= s[:, 1:]).all())
    omitted = E.clone()
    omitted.scatter_(1, ix, -float("inf"))
    assert bool((omitted.max(1).values <= s[:, -1] + eps).all()), float((omitted.max(1).values - s[:, -1]).max())
    print(f"SOP-sized: workspace {ws / 1e6:.1f} MB + k-NN {kb / 1e6:.1f} MB, allocated {used / 1e6:.1f} MB")
