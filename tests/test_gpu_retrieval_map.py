"""MAP@R and R-Precision on the GPU (DESIGN 8): per-query values against an fp64 host loop over exact similarities and over the layer's
own similarities, bit for bit; symmetric tiles against full tiles; long positive lists, repeatability and queries without a positive;
agreement with fp64 similarities; and a set whose similarity matrix would not fit in HBM."""
import numpy as np
import pytest

from eval_ref import check_map, cuda, map_ref, planted

pytestmark = pytest.mark.gpu

PRECS = (0, 1, 2)          # capi.PREC_FP32_BF16X3, PREC_BF16, PREC_FP32_FP16X2


@pytest.mark.parametrize("prec", PRECS)
def test_exact_map_with_planted_ties(prec):
    import torch
    from npairloss_b200 import capi
    rng = np.random.default_rng(20171301 + prec)
    n, D = 301, 37
    K, lab = planted(n, D, 40, rng)
    xt, lt = cuda((K / 8.0).astype(np.float32)), cuda(lab)
    ev = capi.Evaluator(n, n, D, prec)
    out = ev.map_at_r(xt, lt, xt, lt, 0)
    ref = map_ref(K @ K.T, lab, lab, 0)
    assert (ref[2] == 0).sum() >= 5 and (ref[2] >= 3).sum() > 50 and (ref[0][ref[2] > 0] < 1).sum() > 20
    check_map(out, ref)
    assert torch.equal(out["rank"], ev.rank(xt, lt, xt, lt, 0))
    ev.close()
    # disjoint sets, and queries that are a subset of the gallery
    nq, ng, D = 157, 389, 61
    Kg, lg = planted(ng, D, 30, rng)
    Kq = rng.integers(-8, 9, size=(nq, D)).astype(np.int64)
    Kq[: nq // 3] = Kg[rng.integers(0, ng, size=nq // 3)]
    lq = rng.integers(0, 30, size=nq).astype(np.float32)
    ev = capi.Evaluator(nq, ng, D, prec)
    qt, qlt, gt, glt = cuda((Kq / 8.0).astype(np.float32)), cuda(lq), cuda((Kg / 8.0).astype(np.float32)), cuda(lg)
    out = ev.map_at_r(qt, qlt, gt, glt, -1)
    check_map(out, map_ref(Kq @ Kg.T, lq, lg, -1))
    assert torch.equal(out["rank"], ev.rank(qt, qlt, gt, glt, -1))
    k = 101
    sub, subl = gt[k:k + nq].contiguous(), glt[k:k + nq].contiguous()
    out = ev.map_at_r(sub, subl, gt, glt, k)
    check_map(out, map_ref(Kg[k:k + nq] @ Kg.T, lg[k:k + nq], lg, k))
    assert torch.equal(out["rank"], ev.rank(sub, subl, gt, glt, k))
    ev.close()


@pytest.mark.parametrize("prec", PRECS)
def test_map_on_the_layers_similarities(prec):
    """Random unit rows at a ragged D: MAP@R from the layer's own fp32 S (world 1, S materialised), bit for bit."""
    from npairloss_b200 import capi
    rng = np.random.default_rng(20171302 + prec)
    n, D = 1000, 100
    x = rng.standard_normal((n, D)).astype(np.float32)
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    lab = rng.integers(0, n // 6, size=n).astype(np.float32)
    xt, lt = cuda(x), cuda(lab)
    ctx = capi.Context(capi.make_config(n, D, sim_precision=prec))
    ctx.forward(xt, lt)
    S = ctx.debug_read(0, n * n).reshape(n, n)
    ctx.close()
    ev = capi.Evaluator(n, n, D, prec)
    out = ev.map_at_r(xt, lt, xt, lt, 0)
    ev.close()
    ref = map_ref(S, lab, lab, 0)
    assert (ref[2] >= 4).sum() > 100
    check_map(out, ref)


@pytest.mark.parametrize("prec", PRECS)
def test_symmetric_tiles_equal_full_tiles(prec):
    import torch
    from npairloss_b200 import capi, synth
    if capi.lib().npair_debug_mma_symmetric(prec) != 1:
        pytest.skip("this device's MMA is not bitwise symmetric in this operand format")
    n, D = 1000, 96
    x, lab = synth.make_inputs(n, D, 20171303, imgs_per_class=7, noise=2.0)
    lab[::97] = -1.0 - np.arange(len(lab[::97]))                     # some queries without a positive
    xt, lt = cuda(x), cuda(lab)
    ev = capi.Evaluator(n, n, D, prec)
    a = ev.map_at_r(xt, lt, xt, lt, 0)
    b = ev.map_at_r(xt, lt, xt.clone(), lt.clone(), 0)                # another buffer: every tile is computed
    torch.cuda.synchronize()
    ev.close()
    for k in a:
        assert a[k].cpu().numpy().tobytes() == b[k].cpu().numpy().tobytes(), k


@pytest.mark.parametrize("prec", PRECS)
def test_long_lists_repeatable_and_no_positive(prec):
    """10 labels x 300 rows (R = 299, a deep search for every negative between a query's extreme positives) plus singletons."""
    from npairloss_b200 import capi
    rng = np.random.default_rng(20171304 + prec)
    n, D = 3010, 48
    K = rng.integers(-8, 9, size=(n, D)).astype(np.int64)
    K[:3000] += 3 * rng.integers(-1, 2, size=(10, D)).astype(np.int64)[np.arange(3000) // 300]   # a weak class structure
    lab = np.concatenate([np.arange(3000) // 300, 100 + np.arange(10)]).astype(np.float32)
    xt, lt = cuda((K / 8.0).astype(np.float32)), cuda(lab)
    ev = capi.Evaluator(n, n, D, prec)
    a = ev.map_at_r(xt, lt, xt, lt, 0)
    b = ev.map_at_r(xt, lt, xt, lt, 0)
    ref = map_ref(K @ K.T, lab, lab, 0)
    ev.close()
    for k in a:
        assert a[k].cpu().numpy().tobytes() == b[k].cpu().numpy().tobytes(), k
    assert (ref[2][:3000] == 299).all() and (ref[2][3000:] == 0).all()
    assert 0.05 < np.nanmean(ref[0]) < 0.95
    check_map(a, ref)
    assert np.isnan(a["map_r"].cpu().numpy()[3000:]).all() and np.isnan(a["r_precision"].cpu().numpy()[3000:]).all()


def _map_fp64(x, lab):
    S = x.astype(np.float64) @ x.astype(np.float64).T
    return map_ref(S, lab, lab, 0)[0]


@pytest.mark.parametrize("prec", (0, 2))
@pytest.mark.parametrize("D", (128, 512))
def test_mean_map_against_fp64(prec, D):
    from npairloss_b200 import capi, synth
    n = 2000
    x, lab = synth.make_inputs(n, D, 20171305 + D, imgs_per_class=8, noise=2.5)
    xt, lt = cuda(x), cuda(lab)
    ev = capi.Evaluator(n, n, D, prec)
    got = ev.map_at_r(xt, lt, xt, lt, 0)["map_r"].cpu().numpy()
    ev.close()
    want = _map_fp64(x, lab)
    assert 0.05 < want.mean() < 0.999
    assert abs(got.mean() - want.mean()) <= 1e-3, (got.mean(), want.mean())


def test_retrieval_metrics_api():
    import torch
    from npairloss_b200 import synth
    from npairloss_b200.torch_api import recall_at_k, retrieval_metrics
    x, lab = synth.make_inputs(600, 64, 20171306, imgs_per_class=3, noise=2.0)
    lab[:4] = [900.0, 901.0, 902.0, 903.0]                             # four queries without a positive
    xt, lt = cuda(x), cuda(lab).long()
    res, per = retrieval_metrics(xt, lt, ks=(1, 5))
    rec, rank = recall_at_k(xt, lt, ks=(1, 5))
    assert torch.equal(per["rank"], rank)
    assert res["recall@1"] == rec[1] and res["recall@5"] == rec[5]
    assert res["no_positive"] == 4
    m = per["map_r"].cpu().numpy()
    assert np.isnan(m[:4]).all() and abs(res["map@r"] - m[4:].mean()) <= 1e-12
    assert 0.0 < res["r_precision"] <= 1.0 and 0.0 < res["map@r"] <= res["r_precision"] + 1e-12
    # disjoint query / gallery sets
    res2, per2 = retrieval_metrics(xt[:300], lt[:300], xt[300:], lt[300:])
    assert per2["map_r"].shape == (300,) and res2["no_positive"] == int((per2["R"] == 0).sum())


def test_batch_beyond_similarity_matrix():
    """Self-retrieval of B = 196608 at D = 128: the fp32 similarity matrix alone would take 155 GB."""
    import torch
    from npairloss_b200 import capi, synth
    B, D, imgs = 196608, 128, 4
    x, lab = synth.make_inputs(B, D, 20171307, imgs_per_class=imgs, noise=1.5)
    xt, lt = cuda(x), cuda(lab)
    del x
    ws = capi.eval_workspace_bytes(B, B, D)
    capi.Evaluator(256, 256, D).close()                                # loads the module
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    ev = capi.Evaluator(B, B, D)
    out = ev.map_at_r(xt, lt, xt, lt, 0)
    torch.cuda.synchronize()
    used = free0 - torch.cuda.mem_get_info()[0]
    extra = capi.eval_map_at_r_bytes(B, B * (imgs - 1))
    outputs = B * (8 + 8 + 4 + 4)
    assert used <= ws + extra + outputs + (256 << 20), (ws, extra, used)
    got = out["map_r"].double().mean().item()
    ev.close()
    del out
    # chunked fp64 brute force: labels are contiguous blocks of `imgs` rows, so the positives of rows [a, a + C) are known columns
    xd = xt.double()
    total = 0.0
    C = 2048
    for a in range(0, B, C):
        S = xd[a:a + C] @ xd.T
        r = torch.arange(C, device=S.device)
        blk = (a + r) // imgs * imgs
        cols = blk[:, None] + torch.arange(imgs, device=S.device)[None, :]
        cols = cols[cols != (a + r)[:, None]].view(C, imgs - 1)
        p = torch.gather(S, 1, cols).sort(dim=1, descending=True).values
        S.scatter_(1, cols, -float("inf"))
        S[r, a + r] = -float("inf")
        R = imgs - 1
        neg_ge = torch.stack([(S >= p[:, k:k + 1]).sum(1) for k in range(R)], 1)
        pos = torch.arange(1, R + 1, device=S.device)[None, :] + neg_ge
        kk = torch.arange(1, R + 1, device=S.device, dtype=torch.float64)[None, :]
        total += float(torch.where(pos <= R, kk / pos.double(), torch.zeros_like(kk)).sum(1).div(R).sum())
        del S
    want = total / B
    print(f"B={B}: MAP@R {got:.6f} (fp64 {want:.6f}), workspace {ws / 1e6:.1f} MB + MAP@R {extra / 1e6:.1f} MB, allocated {used / 1e6:.1f} MB")
    assert abs(got - want) <= 1e-3, (got, want)
