"""The evaluator (DESIGN 8) at the shapes, labels and buffers where its kernels take their less travelled paths, bit for bit against
host loops over exact similarities (entries k/8 with integer |k| <= 8: every similarity, bias and score is exact in every operand
format, so the header's definitions fix every output), in all three formats:
  - self-retrieval with n around the 32-row warp, the 128-row block and the 256-column tile (the symmetric tile list's skipped and
    mirrored chunks, and the label-range skips with their whole-chunk guards) at D = 1 (almost every similarity ties), 3, 64, 65, 130;
  - query / gallery sets: galleries of fewer than 32 rows, more queries than gallery rows, one query, queries at either end of the
    gallery, disjoint sets without a shared label, and arguments the host refuses;
  - labels -0.0 / +0.0 (one label), NaN (equal to nothing), +-inf, negative and large distinct labels, in chunks of one label or only NaN;
  - degenerate lists: one label for all rows, no positive pair at all (no pair buffer) and then one with positives, and query counts
    around eval_seg_scan_kernel's per-thread runs;
  - feature and label buffers 1-3 floats into larger allocations (eval_split_kernel's scalar loads), against aligned copies;
  - one evaluator through a scripted sequence of calls of different sizes and kinds, partly on a side stream, against fresh evaluators;
  - k-means with k = 1, k = n, k around the 256-column tile, D = 1, 3, 65, all-zero points and one init row for every centroid;
  - the sharded two-phase form with one-row shards, shards without a positive, and self rows outside or across the shards."""
import numpy as np
import pytest

from eval_ref import check_map, cuda, map_ref, planted, update_ref

pytestmark = pytest.mark.gpu

PRECS = (0, 1, 2)          # capi.PREC_FP32_BF16X3, PREC_BF16, PREC_FP32_FP16X2
PREC_NAME = {0: "bf16x3", 1: "bf16", 2: "fp16x2"}
E_ARG = -1

_REFS = {}


def _ref(key, fn):
    """Host references depend on the inputs only, not on the format: computed once per case"""
    if key not in _REFS:
        _REFS[key] = fn()
    return _REFS[key]


def _evaluator(nq, ng, D, prec):
    from npairloss_b200 import capi
    return capi.Evaluator(nq, ng, D, prec)


def _bytes(out):
    import torch
    torch.cuda.synchronize()
    if isinstance(out, dict):
        return {k: (v.cpu().numpy().tobytes() if hasattr(v, "cpu") else v) for k, v in out.items()}
    return out.cpu().numpy().tobytes()


# ---------------------------------------------------------------------------------------------------- 1. self-retrieval shape grid
NS = (1, 2, 3, 31, 32, 33, 127, 128, 129, 160, 161, 255, 256, 257, 289, 383, 385, 513)
DS = (1, 3, 64, 65, 130)


def _grid():
    """Every n meets two D and every D meets every residue of the list (not the whole cross product)."""
    return [pytest.param(n, DS[(i + s) % len(DS)], id=f"n{n}-D{DS[(i + s) % len(DS)]}") for i, n in enumerate(NS) for s in (0, 2)]


def _grid_inputs(n, D):
    """planted() rows and labels, with the first half of the rows relabelled in runs of 40: 32-column chunks and 32-row warps of one
    label and of two neighbouring labels, whose label ranges the sweeps skip on"""
    rng = np.random.default_rng(1000 * n + D)
    K, lab = planted(n, D, max(1, n // 5), rng)
    h = n // 2
    lab[:h] = (np.arange(h) // 40).astype(np.float32) + 7000.0
    return K, lab


@pytest.mark.parametrize("prec", PRECS, ids=PREC_NAME.get)
@pytest.mark.parametrize("n,D", _grid())
def test_self_retrieval_shape_grid(prec, n, D):
    """rank and map_at_r against the host loop on the symmetric tile list (one buffer for both sides) and on full tiles (a second
    buffer with the same data): with exact similarities both give the reference bits, whatever the MMA's symmetry."""
    import torch
    K, lab = _grid_inputs(n, D)
    ref = _ref(("grid", n, D), lambda: map_ref(K @ K.T, lab, lab, 0))
    xt, lt = cuda((K / 8.0).astype(np.float32)), cuda(lab)
    ev = _evaluator(n, n, D, prec)
    try:
        for g, gl, kind in ((xt, lt, "symmetric"), (xt.clone(), lt.clone(), "full tiles")):
            rank = ev.rank(xt, lt, g, gl, 0)
            out = ev.map_at_r(xt, lt, g, gl, 0)
            torch.cuda.synchronize()
            np.testing.assert_array_equal(rank.cpu().numpy(), ref[3], err_msg=kind)
            check_map(out, ref)
            assert torch.equal(out["rank"], rank), kind
    finally:
        ev.close()


# ---------------------------------------------------------------------------------------------------- 2. query and gallery sets
def _qg_cases():
    """(nq, ng, self_offset, how the queries are given): 'copy' another buffer, 'prefix' the gallery's own pointer with nq < ng"""
    return [(300, 1, -1, "copy"), (300, 5, -1, "copy"), (300, 31, -1, "copy"), (37, 5, -1, "copy"), (1, 200, -1, "copy"),
            (1, 200, 0, "prefix"), (1, 200, 199, "copy"), (1, 1, 0, "prefix"), (120, 331, 0, "copy"), (120, 331, 0, "prefix"),
            (120, 331, 211, "copy"), (31, 32, 1, "copy"), (255, 257, 2, "copy")]


@pytest.mark.parametrize("prec", PRECS, ids=PREC_NAME.get)
def test_query_gallery_sets(prec):
    import torch
    from npairloss_b200 import capi
    D = 33
    ev = _evaluator(300, 331, D, prec)
    try:
        for ci, (nq, ng, off, how) in enumerate(_qg_cases()):
            rng = np.random.default_rng(ci)
            Kg, lg = planted(ng, D, max(1, ng // 4), rng)
            if off >= 0:
                Kq, lq = Kg[off:off + nq], lg[off:off + nq]
            else:
                Kq = rng.integers(-8, 9, size=(nq, D)).astype(np.int64)
                Kq[: nq // 2] = Kg[rng.integers(0, ng, size=nq // 2)]       # exact duplicates of gallery rows
                lq = rng.integers(0, max(1, ng // 4), size=nq).astype(np.float32)
            gt, glt = cuda((Kg / 8.0).astype(np.float32)), cuda(lg)
            if how == "prefix":
                qt, qlt = gt[off:off + nq], glt[off:off + nq]
                assert off == 0 and qt.data_ptr() == gt.data_ptr()
            else:
                qt, qlt = cuda((Kq / 8.0).astype(np.float32)), cuda(lq)
            ref = map_ref(Kq @ Kg.T, lq, lg, off)
            tag = f"nq {nq} ng {ng} self_offset {off} {how}"
            rank = ev.rank(qt, qlt, gt, glt, off)
            out = ev.map_at_r(qt, qlt, gt, glt, off)
            torch.cuda.synchronize()
            np.testing.assert_array_equal(rank.cpu().numpy(), ref[3], err_msg=tag)
            check_map(out, ref)
        # disjoint sets that share no label: no positive pair at all
        rng = np.random.default_rng(99)
        Kq, Kg = rng.integers(-8, 9, size=(300, D)), rng.integers(-8, 9, size=(331, D))
        lq, lg = (np.arange(300) % 7).astype(np.float32), (100.0 + np.arange(331) % 9).astype(np.float32)
        qt, qlt, gt, glt = cuda((Kq / 8.0).astype(np.float32)), cuda(lq), cuda((Kg / 8.0).astype(np.float32)), cuda(lg)
        out = ev.map_at_r(qt, qlt, gt, glt, -1)
        rank = ev.rank(qt, qlt, gt, glt, -1)
        torch.cuda.synchronize()
        assert not rank.any() and not out["R"].any() and not out["rank"].any()
        assert torch.isnan(out["map_r"]).all() and torch.isnan(out["r_precision"]).all()
        # refused before anything is enqueued, and the evaluator then still computes the right thing
        nq, ng = 120, 331
        Kg, lg = planted(ng, D, 60, np.random.default_rng(7))
        gt, glt = cuda((Kg / 8.0).astype(np.float32)), cuda(lg)
        qt, qlt = gt[100:100 + nq].contiguous(), glt[100:100 + nq].contiguous()
        big, bigl = cuda(np.zeros((301, D), np.float32)), cuda(np.zeros(301, np.float32))
        for call in (lambda: ev.rank(qt, qlt, gt, glt, ng - nq + 1), lambda: ev.map_at_r(qt, qlt, gt, glt, ng - nq + 1),
                     lambda: ev.rank(big, bigl, gt, glt, -1), lambda: ev.map_at_r(big, bigl, gt, glt, -1)):
            with pytest.raises(capi.NpairError) as e:
                call()
            assert e.value.code == E_ARG, str(e.value)
        ref = map_ref(Kg[100:100 + nq] @ Kg.T, lg[100:100 + nq], lg, 100)
        rank = ev.rank(qt, qlt, gt, glt, 100)
        out = ev.map_at_r(qt, qlt, gt, glt, 100)
        torch.cuda.synchronize()
        np.testing.assert_array_equal(rank.cpu().numpy(), ref[3])
        check_map(out, ref)
    finally:
        ev.close()


# ---------------------------------------------------------------------------------------------------- 3. labels
def _odd_labels(n, rng):
    """Labels that compare in surprising ways as floats, placed so that whole 32-row groups hold only NaN (rows 64-95), only -0.0 / +0.0
    (rows 96-127: one label) or one label next to NaN (rows 128-159)"""
    lab = rng.integers(-6, 6, size=n).astype(np.float32)                 # negative labels
    lab[64:96] = np.nan
    lab[96:128] = np.where(np.arange(32) % 2, np.float32(0.0), np.float32(-0.0))
    lab[128:160] = np.where(np.arange(32) % 3, np.float32(3.0), np.float32(np.nan))
    lab[160:176] = np.inf
    lab[176:188] = -np.inf
    lab[188:200] = np.float32(2.0 ** 24) + 2.0 * np.arange(12)           # distinct, 2 ulp apart
    lab[200:206] = np.float32(2.0 ** 24)                                  # one of them again
    lab[rng.integers(206, n, size=20)] = np.nan                           # scattered NaN
    lab[rng.integers(206, n, size=20)] = -0.0
    return lab


@pytest.mark.parametrize("prec", PRECS, ids=PREC_NAME.get)
def test_float_labels(prec):
    """-0.0 == +0.0 (one label); a NaN query has R = 0 and a NaN gallery row is a negative of every query; +-inf and labels >= 2^24
    are labels like any other."""
    import torch
    n, D = 300, 40
    rng = np.random.default_rng(31)
    K = rng.integers(-8, 9, size=(n, D)).astype(np.int64)
    K[rng.integers(0, n, size=60)] = K[rng.integers(0, n, size=60)]     # ties across the odd labels
    lab = _odd_labels(n, rng)
    xt, lt = cuda((K / 8.0).astype(np.float32)), cuda(lab)
    ref = _ref("labels", lambda: map_ref(K @ K.T, lab, lab, 0))
    nan = np.isnan(lab)
    assert (ref[2][nan] == 0).all() and (ref[2][96:128] >= 31).all() and (ref[2][~nan] > 0).sum() > 150
    refq = _ref("labels-disjoint", lambda: map_ref(K[:150] @ K[150:].T, lab[:150], lab[150:], -1))
    ev = _evaluator(n, n, D, prec)
    try:
        for g, gl in ((xt, lt), (xt.clone(), lt.clone())):
            rank = ev.rank(xt, lt, g, gl, 0)
            out = ev.map_at_r(xt, lt, g, gl, 0)
            torch.cuda.synchronize()
            np.testing.assert_array_equal(rank.cpu().numpy(), ref[3])
            check_map(out, ref)
        q, ql, g, gl = xt[:150], lt[:150], xt[150:].clone(), lt[150:].clone()
        check_map(ev.map_at_r(q, ql, g, gl, -1), refq)
        np.testing.assert_array_equal(ev.rank(q, ql, g, gl, -1).cpu().numpy(), refq[3])
    finally:
        ev.close()


# ---------------------------------------------------------------------------------------------------- 4. degenerate lists
@pytest.mark.parametrize("prec", PRECS, ids=PREC_NAME.get)
def test_one_label_for_all_rows(prec):
    """R_i = n - 1 = 1099 (past the sort's 32-wide passes and past 1024) and no negative: MAP@R = R-Precision = 1 exactly"""
    import torch
    n, D = 1100, 24
    rng = np.random.default_rng(41)
    K = rng.integers(-8, 9, size=(n, D)).astype(np.int64)
    K[rng.integers(0, n, size=200)] = K[rng.integers(0, n, size=200)]
    lab = np.full(n, 4.0, np.float32)
    ref = _ref("one-label", lambda: map_ref(K @ K.T, lab, lab, 0))
    assert (ref[0] == 1.0).all() and (ref[1] == 1.0).all() and (ref[2] == n - 1).all()
    xt, lt = cuda((K / 8.0).astype(np.float32)), cuda(lab)
    ev = _evaluator(n, n, D, prec)
    try:
        out = ev.map_at_r(xt, lt, xt, lt, 0)
        rank = ev.rank(xt, lt, xt, lt, 0)
        torch.cuda.synchronize()
        check_map(out, ref)
        np.testing.assert_array_equal(rank.cpu().numpy(), ref[3])
    finally:
        ev.close()


@pytest.mark.parametrize("prec", PRECS, ids=PREC_NAME.get)
def test_no_positive_pair_then_positives(prec):
    """All labels distinct on a fresh evaluator: sum R_i = 0, so the pair buffer is never allocated, and every output is NaN, R = 0 or
    rank = 0.  The same evaluator then grows the buffer from nothing for a set with positives."""
    import torch
    n, D = 500, 65
    rng = np.random.default_rng(43)
    K, lab = planted(n, D, 60, rng)
    xt = cuda((K / 8.0).astype(np.float32))
    distinct = cuda(np.arange(n, dtype=np.float32) * -1.5)
    ev = _evaluator(n, n, D, prec)
    try:
        out = ev.map_at_r(xt, distinct, xt, distinct, 0)
        torch.cuda.synchronize()
        assert torch.isnan(out["map_r"]).all() and torch.isnan(out["r_precision"]).all()
        assert not out["R"].any() and not out["rank"].any() and not ev.rank(xt, distinct, xt, distinct, 0).any()
        ref = _ref("no-positive-then", lambda: map_ref(K @ K.T, lab, lab, 0))
        lt = cuda(lab)
        check_map(ev.map_at_r(xt, lt, xt, lt, 0), ref)
    finally:
        ev.close()


@pytest.mark.parametrize("prec", PRECS, ids=PREC_NAME.get)
@pytest.mark.parametrize("nq", (1023, 1024, 1025, 2049))
def test_segment_scan_runs(prec, nq):
    """eval_seg_scan_kernel gives each of its 1024 threads a run of ceil(nq / 1024) counts: 1, 1, 2 (the last threads' runs empty) and 3"""
    import torch
    D = 16
    rng = np.random.default_rng(nq)
    K, lab = planted(nq, D, nq // 5, rng)
    ref = _ref(("scan", nq), lambda: map_ref(K @ K.T, lab, lab, 0))
    xt, lt = cuda((K / 8.0).astype(np.float32)), cuda(lab)
    ev = _evaluator(nq, nq, D, prec)
    try:
        out = ev.map_at_r(xt, lt, xt, lt, 0)
        torch.cuda.synchronize()
        check_map(out, ref)
    finally:
        ev.close()


# ---------------------------------------------------------------------------------------------------- 5. offset inputs
def _offset_view(torch, src, off):
    from test_gpu_ragged_shapes import _offset_view as view
    return view(torch, src, off)


def _kmeans_bytes(r):
    import torch
    torch.cuda.synchronize()
    return (r["assign"].cpu().numpy().tobytes(), r["centroids"].cpu().numpy().tobytes(), r["inertia"].cpu().numpy().tobytes(),
            r["iterations"], r["changed"], r["empty"])


@pytest.mark.parametrize("prec", PRECS, ids=PREC_NAME.get)
@pytest.mark.parametrize("D", (64, 128))
def test_offset_inputs(prec, D):
    """Queries, gallery and labels 1, 2 and 3 floats into larger allocations: eval_split_kernel takes its scalar loads (D % 4 = 0, so
    only the pointer decides), and every output is bit for bit that of 16-byte aligned copies.  Random data, not exact: any difference
    in how an operand is read would show."""
    import torch
    from npairloss_b200 import capi, synth
    n = 333
    x, lab = synth.make_inputs(n, D, 51 + D, imgs_per_class=3, noise=2.0)
    xt, lt = cuda(x), cuda(lab)
    amax = float(np.abs(x).max())
    init = list(range(0, n, 11))
    ev = _evaluator(n, n, D, prec)

    def run(q, ql, g, gl):
        res = {"rank_self": ev.rank(q, ql, q, ql, 0), "map_self": ev.map_at_r(q, ql, q, ql, 0),
               "rank_disjoint": ev.rank(q[:100], ql[:100], g[100:], gl[100:], -1)}
        best = torch.maximum(ev.best_positive(q, ql, g[:200], gl[:200], amax, 0, 0),
                             ev.best_positive(q, ql, g[200:], gl[200:], amax, 0, 200))
        res["best"] = best
        res["count"] = ev.count(q, g[:200], best, amax, 0, 0) + ev.count(q, g[200:], best, amax, 0, 200)
        return {k: _bytes(v) for k, v in res.items()}, _kmeans_bytes(ev.kmeans(q, len(init), init, 4))

    try:
        want, want_km = run(xt, lt, xt, lt)
        if capi.lib().npair_debug_mma_symmetric(prec) == 1:                # the shards' full tiles against the symmetric one call
            assert np.array_equal(np.frombuffer(want["count"], np.int32), np.frombuffer(want["rank_self"], np.int32))
        for off in (1, 2, 3):
            xv, lv = _offset_view(torch, xt, off), _offset_view(torch, lt, off)
            assert xv.data_ptr() % 16 and lv.data_ptr() % 16
            got, got_km = run(xv, lv, xv, lv)
            assert got == want, (off, [k for k in want if got[k] != want[k]])
            assert got_km == want_km, off
    finally:
        ev.close()


# ---------------------------------------------------------------------------------------------------- 6. one long-lived evaluator
def _script_inputs(D):
    rng = np.random.default_rng(61)
    n = 700
    K, lab = planted(n, D, 120, rng)
    return (K / 8.0).astype(np.float32), lab


def _call(ev, step, x, lab):
    """One scripted call on an evaluator; returns its outputs as bytes"""
    import torch
    kind, a, b, scale = step
    xs = torch.from_numpy(x * np.float32(scale)).cuda() if scale != 1 else torch.from_numpy(x).cuda()
    lt = torch.from_numpy(lab).cuda()
    if kind == "rank":
        out = ev.rank(xs[:a], lt[:a], xs[:a], lt[:a], 0)
    elif kind == "rank_full":
        out = ev.rank(xs[:a], lt[:a], xs[:a].clone(), lt[:a].clone(), 0)
    elif kind == "map":
        out = ev.map_at_r(xs[:a], lt[:a], xs[:a], lt[:a], 0)
    elif kind == "map_full":
        out = ev.map_at_r(xs[:a], lt[:a], xs[:a].clone(), lt[:a].clone(), 0)
    elif kind == "map_disjoint":
        out = ev.map_at_r(xs[:a], lt[:a], xs[a:a + b], lt[a:a + b], -1)
    elif kind == "kmeans":
        return _kmeans_bytes(ev.kmeans(xs[:a], b, list(range(0, 3 * b, 3)), 3))
    elif kind == "shards":
        q, ql, g, gl = xs[:a], lt[:a], xs[:b], lt[:b]
        amax = float(xs[:b].abs().max())
        best = torch.maximum(ev.best_positive(q, ql, g[:b // 2], gl[:b // 2], amax, 0, 0),
                             ev.best_positive(q, ql, g[b // 2:], gl[b // 2:], amax, 0, b // 2))
        out = {"best": best, "count": ev.count(q, g[:b // 2], best, amax, 0, 0) + ev.count(q, g[b // 2:], best, amax, 0, b // 2)}
    return _bytes(out)


SCRIPT = [("rank", 600, 0, 1), ("map", 300, 0, 1), ("map_full", 300, 0, 1), ("rank", 300, 0, 1), ("kmeans", 650, 40, 1),
          ("shards", 200, 500, 1), ("rank", 129, 0, 1), ("map", 700, 0, 2.0 ** 16), ("map_disjoint", 90, 33, 1),
          ("kmeans", 200, 7, 2.0 ** -16), ("rank", 600, 0, 2.0 ** -16), ("rank_full", 600, 0, 1), ("map", 31, 0, 1), ("rank", 600, 0, 1)]


NO_WAIT = 12        # before this step, the device holds the 600-row symmetric tile list (steps 10 and 11)


def _unordered_calls(torch, ev, x, lab, side, fresh):
    """A rank call on the main stream queued behind a sleep, then at once a rank call on `side` with no wait_stream before it.  The
    queued call (600 rows, symmetric tiles) finds its tile list already on the device and does not upload it; the side call (300
    rows) uploads its own, shorter and different, list into the same buffer.  The evaluator must make the side call wait for the
    queued one: otherwise the side call runs during the sleep, and the queued call then sweeps the 300-row list's tiles."""
    assert SCRIPT[NO_WAIT - 2][:2] == ("rank", 600) and SCRIPT[NO_WAIT - 1][:2] == ("rank_full", 600)
    assert SCRIPT[0] == ("rank", 600, 0, 1) and SCRIPT[3] == ("rank", 300, 0, 1)
    xq, lq = torch.from_numpy(x[:600]).cuda(), torch.from_numpy(lab[:600]).cuda()
    xs, ls = torch.from_numpy(x[:300]).cuda(), torch.from_numpy(lab[:300]).cuda()
    torch.cuda.synchronize()
    torch.cuda._sleep(100_000_000)                      # about 50 ms
    queued = ev.rank(xq, lq, xq, lq, 0)
    with torch.cuda.stream(side):
        unwaited = ev.rank(xs, ls, xs, ls, 0)
    torch.cuda.synchronize()
    assert _bytes(queued) == fresh[0], "the rank call queued on the main stream"
    assert _bytes(unwaited) == fresh[3], "the side-stream call issued without a wait"


@pytest.mark.parametrize("prec", PRECS, ids=PREC_NAME.get)
def test_long_lived_evaluator(prec):
    """rank -> map_at_r -> kmeans -> best_positive / count -> rank on one evaluator with spare capacity: shrinking and growing sizes,
    symmetric and full tiles at one n, max|x| changing by 2^16 between calls (the fp16x2 pre-scale), the second half on a side stream,
    and one side-stream call issued without a wait while a call on the main stream is still queued (_unordered_calls).
    Each result is bit for bit that of a fresh evaluator made for exactly that call: nothing the evaluator keeps between calls (the
    symmetric tile list, the absmax word, the error word, the grown MAP@R and k-means buffers) leaks into the next one."""
    import torch
    D = 65
    x, lab = _script_inputs(D)
    fresh = []
    for kind, a, b, scale in SCRIPT:
        nq, ng = {"kmeans": (a, b), "shards": (a, b), "map_disjoint": (a, b)}.get(kind, (a, a))
        ev = _evaluator(nq, ng, D, prec)
        try:
            fresh.append(_call(ev, (kind, a, b, scale), x, lab))
        finally:
            ev.close()
    ev = _evaluator(700, 700, D, prec)
    side = torch.cuda.Stream()
    try:
        for i, step in enumerate(SCRIPT):
            if i == NO_WAIT:
                _unordered_calls(torch, ev, x, lab, side, fresh)
            if i < len(SCRIPT) // 2:
                got = _call(ev, step, x, lab)
            else:
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    got = _call(ev, step, x, lab)
                torch.cuda.current_stream().wait_stream(side)
            assert got == fresh[i], (i, step)
    finally:
        torch.cuda.synchronize()
        ev.close()
    # the first, exact call against the host loop too, so that the fresh evaluators are not merely consistent
    K = np.rint(x * 8).astype(np.int64)
    ref = map_ref(K[:600] @ K[:600].T, lab[:600], lab[:600], 0)
    np.testing.assert_array_equal(np.frombuffer(fresh[0], np.int32), ref[3])


# ---------------------------------------------------------------------------------------------------- 7. k-means edges
def _exact_first_assignment(K, init):
    Kc = K[init]
    return np.argmax(2 * K @ Kc.T - (Kc * Kc).sum(1)[None, :], axis=1)    # 128 * (s - 0.5 ||mu||^2), exact; lowest index on ties


def _kmeans(ev, xt, k, init, max_iter):
    r = ev.kmeans(xt, k, init, max_iter)
    return {"assign": r["assign"].cpu().numpy(), "centroids": r["centroids"].cpu().numpy(), "inertia": float(r["inertia"]),
            "stats": (r["iterations"], r["changed"], r["empty"])}


def _distinct_rows(n, D, rng):
    codes = rng.choice(17 ** D, size=n, replace=False) if 17 ** D < 2 ** 62 else None
    if codes is None:
        K = rng.integers(-8, 9, size=(n, D)).astype(np.int64)
        assert len(np.unique(K, axis=0)) == n
        return K
    return np.stack([(codes // 17 ** d) % 17 - 8 for d in range(D)], 1).astype(np.int64)


def _km_case(name):
    rng = np.random.default_rng(sum(map(ord, name)))
    if name == "k1":
        K = rng.integers(-8, 9, size=(100, 65)).astype(np.int64)
        return K, [37]
    if name.startswith("k=n"):
        n, D = {"k=n-33x3": (33, 3), "k=n-129x65": (129, 65), "k=n-5x1": (5, 1)}[name]
        K = _distinct_rows(n, D, rng)
        return K, list(range(n))
    if name.startswith("n"):
        n, D, k = {"n5-D1": (5, 1, 2), "n33-D3": (33, 3, 7), "n129-D65": (129, 65, 20)}[name]
        K = rng.integers(-8, 9, size=(n, D)).astype(np.int64)
        return K, rng.choice(n, size=k, replace=False).tolist()
    if name.startswith("k25"):
        k = int(name[1:])
        K = rng.integers(-8, 9, size=(600, 24)).astype(np.int64)
        init = rng.choice(600, size=k, replace=False)
        init[k - 1] = init[k - 2]                                           # ties in the last, ragged or full, column tile
        return K, init.tolist()
    if name == "zeros":
        return np.zeros((50, 3), np.int64), [0, 10, 20, 30]
    if name == "one-init-row":
        K = rng.integers(-8, 9, size=(100, 65)).astype(np.int64)
        return K, [7] * 10
    raise KeyError(name)


KM_CASES = ("k1", "k=n-5x1", "k=n-33x3", "k=n-129x65", "n5-D1", "n33-D3", "n129-D65", "k255", "k256", "k257", "zeros", "one-init-row")


@pytest.mark.parametrize("prec", PRECS, ids=PREC_NAME.get)
@pytest.mark.parametrize("case", KM_CASES)
def test_kmeans_edges(prec, case):
    """The first assignment is the exact int64 argmax with the lowest index on ties; C_{t+1} of the run with max_iter = t + 1 is the
    fixed-point update of the run with max_iter = t, for t = 1..3, unless the runs stopped on convergence before."""
    K, init = _km_case(case)
    n, D = K.shape
    k = len(init)
    x = (K / 8.0).astype(np.float32)
    xt = cuda(x)
    want = _exact_first_assignment(K, init)
    ev = _evaluator(n, k, D, prec)
    try:
        prev = _kmeans(ev, xt, k, init, 1)
        np.testing.assert_array_equal(prev["assign"], want)
        np.testing.assert_array_equal(prev["centroids"].view(np.uint32), x[init].view(np.uint32))
        assert prev["stats"] == (1, n, k - len(np.unique(want))), prev["stats"]
        for t in range(1, 4):
            if prev["stats"][0] < t or (prev["stats"][0] > 1 and prev["stats"][1] == 0):
                break                                                        # converged: the later runs are this one
            nxt = _kmeans(ev, xt, k, init, t + 1)
            assert nxt["stats"][0] == t + 1, (t, nxt["stats"])
            np.testing.assert_array_equal(nxt["centroids"].view(np.uint32), update_ref(x, prev["assign"], prev["centroids"]).view(np.uint32),
                                          err_msg=f"t={t}")
            prev = nxt
        final = _kmeans(ev, xt, k, init, 10)
    finally:
        ev.close()
    if case.startswith("k=n"):
        np.testing.assert_array_equal(final["assign"], np.arange(n))
        assert final["stats"] == (2, 0, 0) and final["inertia"] == 0.0, final["stats"]
        np.testing.assert_array_equal(final["centroids"].view(np.uint32), x.view(np.uint32))
    if case == "k1":                                                        # the fixed-point mean of all points
        mean = update_ref(x, np.zeros(n, np.int64), x[init])
        np.testing.assert_array_equal(final["centroids"].view(np.uint32), mean.view(np.uint32))
        assert not final["assign"].any() and final["stats"] == (2, 0, 0)
    if case in ("zeros", "one-init-row"):                                   # k identical centroids: the first takes every point
        assert not want.any()
    if case == "zeros":                                                     # sigma = 1, and nothing ever moves
        assert final["stats"] == (2, 0, k - 1) and final["inertia"] == 0.0 and not final["centroids"].any()
        assert not final["assign"].any()


# ---------------------------------------------------------------------------------------------------- 8. sharded two-phase form
def _shard_cases(ng):
    return {"one-row shards": [(a, a + 1) for a in range(ng)],
            "uneven": [(0, 7), (7, 40), (40, 41), (41, ng)],
            "two": [(0, 20), (20, ng)]}


@pytest.mark.parametrize("prec", PRECS, ids=PREC_NAME.get)
def test_sharded_edges(prec):
    """max over shards of best_positive and the sum over shards of count equal one rank call and the exact p* and rank:
    one-row shards; shards with no positive of any query (-inf, and count 0 where the cut is -inf); shards that start past every
    query's own row (gallery_row0 > self_offset + nq - 1); and queries whose self rows straddle two shards."""
    import torch
    D = 40
    ng = 64
    rng = np.random.default_rng(81)
    Kg = rng.integers(-8, 9, size=(ng, D)).astype(np.int64)
    Kg[40:50] = Kg[rng.integers(0, 40, size=10)]                          # ties across shards
    lg = (np.arange(ng) // 4).astype(np.float32)
    lg[41:ng] = 500.0 + np.arange(ng - 41)                                 # rows 41.. hold no positive of any query
    lg[5] = 900.0                                                           # a query without any positive: cut -inf
    gt, glt = cuda((Kg / 8.0).astype(np.float32)), cuda(lg)
    amax = float(np.abs(Kg).max() / 8.0)
    ev = _evaluator(ng, ng, D, prec)
    try:
        for off, nq in ((-1, 30), (0, 30), (3, 30), (10, 20)):
            q0 = max(off, 0)
            Kq = Kg[q0:q0 + nq] if off >= 0 else rng.integers(-8, 9, size=(nq, D)).astype(np.int64)
            lq = lg[q0:q0 + nq] if off >= 0 else (np.arange(nq) // 3).astype(np.float32)
            qt, qlt = cuda((Kq / 8.0).astype(np.float32)), cuda(lq)
            ref = map_ref(Kq @ Kg.T, lq, lg, off)
            S = (Kq @ Kg.T).astype(np.float64)
            valid = np.ones_like(S, bool)
            if off >= 0:
                valid[np.arange(nq), off + np.arange(nq)] = False
            same = (lq[:, None] == lg[None, :]) & valid
            pstar = np.where(same.any(1), np.where(same, S, -np.inf).max(1) / 64.0, -np.inf).astype(np.float32)
            one = ev.rank(qt, qlt, gt, glt, off)
            np.testing.assert_array_equal(one.cpu().numpy(), ref[3])
            for name, shards in _shard_cases(ng).items():
                tag = f"self_offset {off} nq {nq}: {name}"
                bests = [ev.best_positive(qt, qlt, gt[a:b], glt[a:b], amax, off, a) for a, b in shards]
                best = torch.stack(bests).max(0).values
                counts = [ev.count(qt, gt[a:b], best, amax, off, a) for a, b in shards]
                torch.cuda.synchronize()
                np.testing.assert_array_equal(best.cpu().numpy().view(np.uint32), pstar.view(np.uint32), err_msg=tag)
                total = torch.stack(counts).sum(0).int()
                assert torch.equal(total, one), tag
                for (a, b), bp, c in zip(shards, bests, counts):
                    if a >= 41:                                            # no positive of any query in the shard
                        assert bool(torch.isneginf(bp).all()), (tag, a)
                    assert not c[torch.isneginf(best)].any(), (tag, a)
            assert bool(torch.isneginf(best).any()) == bool((pstar == -np.inf).any())
    finally:
        ev.close()
