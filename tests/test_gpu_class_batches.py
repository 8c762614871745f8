"""Hard negative class mining on the GPU (npair_eval_class_batches, DESIGN 8.4): batches and scores against a numpy greedy over the
library's own S (from knn and from a layer context) bit for bit, planted ties decided by pool position, the NaN rule, independence of
the other pools, the stream and the evaluator, the hardness of mined batches on synthetic superclasses, argument checks without
launches, and an SOP-sized run with its device memory."""
import ctypes as C

import numpy as np
import pytest

from eval_ref import cuda

pytestmark = pytest.mark.gpu

PRECS = (0, 1, 2)          # capi.PREC_FP32_BF16X3, PREC_BF16, PREC_FP32_FP16X2
E_ARG = -1
POOL_MAX = 16384           # NPAIR_EVAL_CLASS_POOL_MAX


def ref_greedy(S, pools, n):
    """The header's greedy over given similarities S [C, C] (fp32, or exact float64): seed pools[t][0]; then n - 1 times the unselected
    position with the largest v_j = fmax over the selected classes c of S[c][pool[j]] (NaN below every number), ties to the lowest
    position.  Returns (batches [b, n] int64, scores [b, n] fp32, NaN for the seed)."""
    pools = np.asarray(pools)
    b, P = pools.shape
    out, sc = np.zeros((b, n), np.int64), np.full((b, n), np.nan, np.float32)
    for t in range(b):
        pool = pools[t]
        v = np.full(P, np.nan)
        live = np.ones(P, bool)
        live[0] = False
        c = out[t, 0] = pool[0]
        for s in range(1, n):
            v = np.fmax(v, S[c, pool].astype(np.float64))
            cand = np.flatnonzero(live)
            vv = v[cand]
            j = cand[0] if np.isnan(vv).all() else cand[np.flatnonzero(vv == np.nanmax(vv))[0]]
            live[j] = False
            c = out[t, s] = pool[j]
            sc[t, s] = v[j]
    return out, sc


def _run(ev, x, pools, n):
    b, s = ev.class_batches(x, np.asarray(pools, np.int32), n)
    return b.cpu().numpy().astype(np.int64), s.cpu().numpy()


def _same(got, want):
    """batches equal, scores equal bit for bit (NaN where the reference has NaN)"""
    np.testing.assert_array_equal(got[0], want[0])
    nan = np.isnan(want[1])
    np.testing.assert_array_equal(np.isnan(got[1]), nan)
    np.testing.assert_array_equal(got[1][~nan].view(np.uint32), want[1][~nan].view(np.uint32))


def _pools(rng, C_, P, b):
    return np.stack([rng.permutation(C_)[:P] for _ in range(b)]).astype(np.int32)


def _unit(rng, n, D):
    x = rng.standard_normal((n, D)).astype(np.float32)
    return x / np.linalg.norm(x, axis=1, keepdims=True)


def _exact(K):
    """similarities of planted rows (entries k/8) in float64: (K K^T) / 64, exact in fp32"""
    return (K @ K.T).astype(np.float64) / 64.0


@pytest.mark.parametrize("prec", PRECS)
def test_bits_against_knn_similarities(prec):
    """C = 1000 random unit rows, S taken from knn(E, k = C - 1) scattered back: random pools at n = 2, a middle n and n = P, ragged
    pools, pools covering every class, and b = 133 (no multiple of the SM count), bit for bit; also through hard_class_batches."""
    import torch
    from npairloss_b200 import capi
    from npairloss_b200.torch_api import hard_class_batches, knn
    rng = np.random.default_rng(20261101 + prec)
    C_, D = 1000, 72
    x = cuda(_unit(rng, C_, D))
    sim, idx = knn(x, k=C_ - 1, precision=prec)
    S = np.full((C_, C_), np.nan, np.float32)
    np.put_along_axis(S, idx.cpu().numpy(), sim.cpu().numpy(), 1)
    ev = capi.Evaluator(C_, C_, D, prec)
    try:
        for P, b, n in ((300, 5, 2), (300, 5, 37), (300, 3, 300), (999, 2, 999), (61, 133, 17), (C_, 4, 50)):
            pools = _pools(rng, C_, P, b)
            _same(_run(ev, x, pools, n), ref_greedy(S, pools, n))
    finally:
        ev.close()
    batches, scores = hard_class_batches(x, 24, 7, pool_size=500, seed=5, precision=prec)
    g = torch.Generator().manual_seed(5)
    pools = np.stack([torch.randperm(C_, generator=g)[:500].numpy() for _ in range(7)])
    assert batches.dtype == torch.int64 and batches.is_cuda
    _same((batches.cpu().numpy(), scores.cpu().numpy()), ref_greedy(S, pools, 24))


@pytest.mark.parametrize("prec", PRECS)
def test_bits_against_layer_similarities(prec):
    """C = 3001 random unit rows, S from a world-1 layer context's debug_read(0): pools of every class and a ragged pool at n = P."""
    from npairloss_b200 import capi
    rng = np.random.default_rng(20261102 + prec)
    C_, D = 3001, 100
    xn = _unit(rng, C_, D)
    x = cuda(xn)
    ctx = capi.Context(capi.make_config(C_, D, sim_precision=prec))
    ctx.forward(x, cuda(rng.integers(0, C_ // 3, size=C_).astype(np.float32)))
    S = ctx.debug_read(0, C_ * C_).reshape(C_, C_)
    ctx.close()
    ev = capi.Evaluator(C_, C_, D, prec)
    try:
        for P, b, n in ((C_, 3, 64), (1499, 1, 1499)):
            pools = _pools(rng, C_, P, b)
            _same(_run(ev, x, pools, n), ref_greedy(S, pools, n))
    finally:
        ev.close()


@pytest.mark.parametrize("prec", PRECS)
def test_planted_ties(prec):
    """Entries k/8 make S exact.  The seed and five duplicate classes are all ones, every other row has an entry below one, so the
    duplicates tie at the top of the seed's row and are picked next in pool order; swapping two of them in the pool swaps the picks."""
    from npairloss_b200 import capi
    rng = np.random.default_rng(20261103 + prec)
    C_, D = 400, 64
    K = rng.integers(-8, 9, size=(C_, D)).astype(np.int64)
    K[:, 0] = np.minimum(K[:, 0], 7)
    dup = np.array([3, 50, 77, 120, 300])
    K[dup] = 8
    K[10] = 8                                               # the seed
    x = cuda((K / 8.0).astype(np.float32))
    E = _exact(K)
    others = rng.permutation(np.setdiff1d(np.arange(C_), np.r_[10, dup]))[:245]
    pool = np.r_[10, rng.permutation(np.r_[dup, others])]
    ev = capi.Evaluator(C_, C_, D, prec)
    try:
        pools = np.stack([pool, pool.copy()])
        pos = sorted(np.flatnonzero(np.isin(pool, dup)))
        pools[1, pos[0]], pools[1, pos[3]] = pool[pos[3]], pool[pos[0]]
        got = _run(ev, x, pools, 40)
        _same(got, ref_greedy(E, pools, 40))
        np.testing.assert_array_equal(got[0][0, 1:6], pool[pos])
        np.testing.assert_array_equal(got[0][1, 1:6], pools[1, pos])
        assert (got[1][:, 1:6] == D / 1.0).all()
    finally:
        ev.close()


@pytest.mark.parametrize("prec", PRECS)
def test_nan_class_ranks_last(prec):
    """A class embedding with a NaN: as a candidate it is picked last (n = P), at a NaN score; as the seed every score of the next step
    is NaN, so the next pick is pool position 1, and the batch goes on from there as the numpy greedy does."""
    from npairloss_b200 import capi
    rng = np.random.default_rng(20261104 + prec)
    C_, D = 300, 32
    K = rng.integers(-8, 9, size=(C_, D)).astype(np.int64)
    xn = (K / 8.0).astype(np.float32)
    xn[17, 5] = np.nan
    E = _exact(K)
    E[17, :] = np.nan
    E[:, 17] = np.nan
    x = cuda(xn)
    rest = lambda: rng.permutation(np.setdiff1d(np.arange(C_), [17]))[:119]
    pools = np.stack([np.insert(rest(), 50, 17) for _ in range(5)] + [np.r_[17, rest()]]).astype(np.int32)
    ev = capi.Evaluator(C_, C_, D, prec)
    try:
        got = _run(ev, x, pools, 120)
    finally:
        ev.close()
    _same(got, ref_greedy(E, pools, 120))
    assert (got[0][:5, -1] == 17).all() and np.isnan(got[1][:5, -1]).all()
    assert got[0][5, 1] == pools[5, 1] and np.isnan(got[1][5, :2]).all() and not np.isnan(got[1][5, 2:]).any()


def test_independent_of_other_pools_stream_and_evaluator():
    import torch
    from npairloss_b200 import capi
    rng = np.random.default_rng(20261105)
    C_, D, P, n = 2000, 64, 700, 45
    x = cuda(_unit(rng, C_, D))
    pools = _pools(rng, C_, P, 300)
    runs = []
    ev = capi.Evaluator(C_, C_, D, 2)
    try:
        runs.append(_run(ev, x, pools, n))
        runs.append(_run(ev, x, pools, n))
        sub = _run(ev, x, pools[[7, 150, 299]], n)
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            runs.append(_run(ev, x, pools, n))
        torch.cuda.synchronize()
    finally:
        ev.close()
    ev = capi.Evaluator(C_ + 5, C_ + 9, D, 2)
    try:
        runs.append(_run(ev, x, pools, n))
    finally:
        ev.close()
    for r in runs[1:]:
        _same(r, runs[0])
    _same(sub, (runs[0][0][[7, 150, 299]], runs[0][1][[7, 150, 299]]))


def test_mined_batches_are_hard():
    """64 superclasses of 8 close classes, n = 8 from pools of every class: each mined batch is its seed's superclass, and its mean
    pairwise similarity exceeds that of random batches (the pools' first 8 classes)."""
    from npairloss_b200 import capi
    rng = np.random.default_rng(20261106)
    n_sup, D = 64, 64
    centers = _unit(rng, n_sup, D)
    xn = np.repeat(centers, 8, 0) + 0.15 * rng.standard_normal((n_sup * 8, D)).astype(np.float32) / np.sqrt(D)
    xn = (xn / np.linalg.norm(xn, axis=1, keepdims=True)).astype(np.float32)
    C_ = xn.shape[0]
    pools = _pools(rng, C_, C_, 40)
    for prec in PRECS:
        ev = capi.Evaluator(C_, C_, D, prec)
        try:
            b, _ = _run(ev, cuda(xn), pools, 8)
        finally:
            ev.close()
        for t in range(40):
            np.testing.assert_array_equal(np.sort(b[t]), pools[t, 0] // 8 * 8 + np.arange(8))
    G = xn.astype(np.float64) @ xn.T.astype(np.float64)
    mean = lambda ids: (G[np.ix_(ids, ids)].sum() - len(ids)) / (len(ids) * (len(ids) - 1))
    assert np.mean([mean(r) for r in b]) > np.mean([mean(p[:8]) for p in pools]) + 0.5


def test_bad_arguments_launch_nothing():
    import torch
    from npairloss_b200 import capi
    C_, D = 200, 16
    x = torch.randn(C_, D, device="cuda")
    big = torch.randn(POOL_MAX + 1, 4, device="cuda")
    out = torch.empty(4, POOL_MAX + 1, dtype=torch.int32, device="cuda")
    scores = torch.empty(4, POOL_MAX + 1, device="cuda")
    ev = capi.Evaluator(C_, C_, D, 2)
    ev_big = capi.Evaluator(POOL_MAX + 1, POOL_MAX + 1, 4, 2)
    L = capi.lib()
    st = torch.cuda.current_stream().cuda_stream
    good = np.stack([np.random.default_rng(t).permutation(C_)[:50] for t in range(4)]).astype(np.int32)

    def call(e, xx, Cn, pools, P, b, n, o=out.data_ptr(), s=scores.data_ptr()):
        p = None if pools is None else np.ascontiguousarray(pools, np.int32)
        return L.npair_eval_class_batches(e._h if e else None, xx, Cn, None if p is None else p.ctypes.data, P, b, n, o, s, st)

    dup, neg, over = good.copy(), good.copy(), good.copy()
    dup[2, 40] = dup[2, 3]
    neg[1, 7] = -1
    over[3, 0] = C_
    try:
        _run(ev, x, good, 10)                                # loads the kernels
        ev_big.class_batches(big, np.arange(POOL_MAX, dtype=np.int32)[None], 2)
        torch.cuda.synchronize()
        n0 = capi.kernel_launches()
        bad = [(ev, x.data_ptr(), C_, dup, 50, 4, 10), (ev, x.data_ptr(), C_, neg, 50, 4, 10), (ev, x.data_ptr(), C_, over, 50, 4, 10),
               (ev, x.data_ptr(), C_, good, 50, 4, 1), (ev, x.data_ptr(), C_, good, 50, 4, 51), (ev, x.data_ptr(), C_, good, 1, 4, 1),
               (ev, x.data_ptr(), C_, good, 50, 0, 10), (ev, x.data_ptr(), C_ + 1, good, 50, 4, 10), (ev, x.data_ptr(), 0, good, 50, 4, 2),
               (ev, None, C_, good, 50, 4, 10), (ev, x.data_ptr(), C_, None, 50, 4, 10),
               (ev_big, big.data_ptr(), POOL_MAX + 1, np.arange(POOL_MAX + 1)[None], POOL_MAX + 1, 1, 2)]
        for a in bad:
            assert call(*a) == E_ARG, a[2:]
        assert call(ev, x.data_ptr(), C_, good, 50, 4, 10, o=None) == E_ARG
        assert L.npair_eval_class_batches(None, None, 0, None, 0, 0, 0, None, None, None) == E_ARG
        assert capi.kernel_launches() == n0, "a refused call launched kernels"
        # the limits themselves are accepted: n = P = C, NULL scores, a pool of NPAIR_EVAL_CLASS_POOL_MAX classes
        assert call(ev, x.data_ptr(), C_, good[:, :2], 2, 4, 2, s=None) == 0
        full = np.stack([np.random.default_rng(9).permutation(C_)])
        b, s = _run(ev, x, full, C_)
        assert sorted(b[0]) == list(range(C_))
        b, _ = ev_big.class_batches(big, np.random.default_rng(3).permutation(POOL_MAX + 1)[:POOL_MAX][None], 64, scores=False)
        assert len(set(b.cpu().numpy()[0].tolist())) == 64
        torch.cuda.synchronize()
    finally:
        ev.close()
        ev_big.close()


def test_sop_sized_run():
    """C = 11 318 classes (Stanford Online Products' training classes), D = 512, pools of every class, n = 60, b = 189, fp16x2: the
    device memory the call adds, distinct picks from each pool, and on four batches every pick against an fp64 greedy within the
    format's error bound (each score is the pick's v, and no unpicked class had a larger v)."""
    import torch
    from npairloss_b200 import capi
    C_, D, n, b, prec = 11318, 512, 60, 189, 2
    rng = np.random.default_rng(20261107)
    centers = rng.standard_normal((1500, D)).astype(np.float32)
    xn = centers[rng.integers(0, 1500, size=C_)] + 0.9 * rng.standard_normal((C_, D)).astype(np.float32)
    xn = (xn / np.linalg.norm(xn, axis=1, keepdims=True)).astype(np.float32)
    x = cuda(xn)
    pools = _pools(rng, C_, C_, b)
    ws, cb = capi.eval_workspace_bytes(C_, C_, D, prec), capi.eval_class_batches_bytes(C_, C_, b)
    ev0 = capi.Evaluator(512, 512, D, prec)                 # loads the kernels
    ev0.class_batches(x[:512].contiguous(), _pools(rng, 512, 512, 2), 8)
    ev0.close()
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    ev = capi.Evaluator(C_, C_, D, prec)
    try:
        batches, scores = ev.class_batches(x, pools, n)
        torch.cuda.synchronize()
        used = free0 - torch.cuda.mem_get_info()[0]
    finally:
        ev.close()
    outputs = b * n * 8
    assert ws + cb <= used <= ws + cb + outputs + (64 << 20), (ws, cb, used)
    bt, st = batches.cpu().numpy(), scores.cpu().numpy()
    for t in range(b):
        assert bt[t, 0] == pools[t, 0] and len(set(bt[t].tolist())) == n and np.isin(bt[t], pools[t]).all()
    M, L1, u = float(np.abs(xn).max()), float(np.abs(xn).sum(1).max()), 2.0 ** -24
    eps = 2.0 ** -21 * M * 2 * L1 + D * 2.0 ** -20 * M * M + 3 * D * u * L1 * M + u     # DESIGN 5: fp16x2 operand and accumulation error
    xd = torch.from_numpy(xn).cuda().double()
    for t in (0, 1, 94, 188):
        G = xd[torch.from_numpy(bt[t]).cuda()] @ xd.T                                  # [n, C] fp64
        v = torch.full((C_,), -float("inf"), dtype=torch.float64, device="cuda")
        live = torch.ones(C_, dtype=torch.bool, device="cuda")
        live[bt[t, 0]] = False
        for s in range(1, n):
            v = torch.maximum(v, G[s - 1])
            assert abs(float(v[bt[t, s]]) - float(st[t, s])) <= eps, (t, s)
            assert float(v[live].max()) <= float(st[t, s]) + 2 * eps, (t, s)
            live[bt[t, s]] = False
    print(f"SOP-sized: workspace {ws / 1e6:.1f} MB + class batches {cb / 1e6:.1f} MB, allocated {used / 1e6:.1f} MB")
