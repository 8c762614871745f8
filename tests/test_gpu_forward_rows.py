"""The forward row by row against exact and fp64 references (forward_ref.py), on the GPU's own S.

gpu_harness.check_parity compares the forward with the oracle through aggregates: thresholds bit for bit, the mean loss to 1e-5, the
retrieval counters to one row in 1000.  Here every row's statistics, A and T, log(A/T), hit flags and backward record are checked on
their own: the statistics and the hit flags exactly, A and T componentwise against fp64 sums under the row pass's flush rule, the
records bit for bit or against fp64 of the GPU's own A and T.  The cases reach the paths of the similarity epilogue (symmetric tiles,
mirrored statistics, partial chunks, the SIMT row_stats_ref) and of the row pass (1, 2, 4 and 8 warps per row, the ragged tail, the
unaligned-label path, row blocks with the separate finaliser, cross-batch memory, emulated ranks), and rows whose positives lie
60 .. 110 nats below their maximum, where 2^14 / A overflows fp32 unless the record's exponent offset absorbs it (DESIGN 5)."""
import numpy as np
import pytest

from npairloss_b200 import capi, synth
import forward_ref as fr
import grad_ref
from grad_ref import FP16X2, BF16X3, BF16

pytestmark = pytest.mark.gpu

TC, SIMT = capi.GEMM_TCGEN05, capi.GEMM_SIMT_CHECK
NAME = {FP16X2: "fp16x2", BF16X3: "bf16x3", BF16: "bf16"}
K = {FP16X2: 14, BF16X3: 0, BF16: 0}              # weight_scale_log2
HARD_HARD = dict(synth.DEFAULT_MINING, ap_method=synth.HARD, an_method=synth.HARD, margin_diff=-0.02)
GLOBAL_REL = dict(margin_ident=0.01, margin_diff=-0.02, identsn=-0.4, diffsn=-0.3, ap_region=synth.GLOBAL, ap_method=synth.RELATIVE_HARD,
                  an_region=synth.GLOBAL, an_method=synth.RELATIVE_HARD)
LOCAL_REL = dict(margin_ident=0.01, margin_diff=-0.02, identsn=-0.4, diffsn=-0.3, ap_region=synth.LOCAL, ap_method=synth.RELATIVE_HARD,
                 an_region=synth.LOCAL, an_method=synth.RELATIVE_EASY)
MININGS = {"rand": synth.DEFAULT_MINING, "usage": synth.USAGE_MINING, "hard": HARD_HARD, "global_rel": GLOBAL_REL,
           "local_rel": LOCAL_REL}


@pytest.fixture(scope="module")
def torch():
    import torch
    assert torch.cuda.is_available() and torch.cuda.get_device_capability(0) == (9, 0), "GPU tests need an H100"
    return torch


def lse_wpr(Q, N):
    """Warps per row of the row pass (lse_shape, kernels.cu)."""
    wpr = 1
    while wpr < 8 and Q * wpr < 4096 and N // (2 * wpr) >= 512:
        wpr *= 2
    return 2 if Q >= 1024 and wpr > 2 else wpr


def observe(torch, ctx, Q, tops):
    """Everything the forward left of one context's rows."""
    rd = {k: ctx.debug_read(w, Q) for k, w in (("posi", 1), ("nega", 2), ("min_within", 3), ("max_between", 4), ("max_all", 5),
                                                ("A", 6), ("T", 7), ("cnt_same", 8), ("max_within", 9), ("logv", 11))}
    rd["hits"] = ctx.debug_read(12, 3 * Q)
    rec = torch.zeros((Q, 8), dtype=torch.float32, device="cuda")
    ctx.row_scalars(rec)
    torch.cuda.synchronize()
    rd["rec"] = rec.cpu().numpy()
    rd["tops"] = np.asarray(tops, np.float32)
    return rd


def check_rows(g, S, lab_rows, lab_cols, self_cols, mining, prec, num_tops, world=1, tag="", amb_max=None):
    """Every check of forward_ref on one rank's observed rows.  Returns the reference and the record shifts j."""
    Q, N = S.shape
    ref = fr.reference(S, lab_rows, lab_cols, self_cols, g["posi"], g["nega"], mining, wpr=lse_wpr(Q, N))
    bad = fr.check_stats(ref, g)
    b, meas = fr.check_sums(ref, g["A"], g["T"])
    bad += b
    bad += fr.check_log(ref, g["logv"], g["A"], g["T"])
    bad += fr.check_tops(g["tops"], g["logv"], g["hits"], Q, num_tops)
    b, n_amb = fr.check_hits(ref, S, g["hits"])
    bad += b
    b, j = fr.check_records(ref, g["rec"], g["A"], g["T"], lab_rows, g["posi"], g["nega"], mining, K[prec], world)
    bad += b
    print(f"{tag} {NAME[prec]} Q {Q} N {N}: A {meas['A'][0]:.1f} (tau {meas['A'][1]:.1f}), T {meas['T'][0]:.1f} (tau {meas['T'][1]:.1f}) "
          f"x 2^-24; ambiguous rows {n_amb}; rows with j > 0: {int((j > 0).sum())}")
    if amb_max is not None and n_amb > amb_max:
        bad.append(f"{n_amb} ambiguous rows (at most {amb_max} expected)")
    assert not bad, f"{tag} {NAME[prec]}: " + "; ".join(bad)
    return ref, j


def run_world1(torch, x, lab, mining, prec=FP16X2, backend=TC, num_tops=5, tag="", amb_max=0, lab_offset=False, **cfg):
    Q, D = x.shape
    xt = torch.from_numpy(x).cuda()
    if lab_offset:                              # the labels one float past a 16-byte boundary: every row through the tail loop
        buf = torch.zeros(Q + 1, dtype=torch.float32, device="cuda")
        buf[1:] = torch.from_numpy(lab).cuda()
        lt = buf[1:]
    else:
        lt = torch.from_numpy(lab).cuda()
    ctx = capi.Context(capi.make_config(Q, D, num_tops=num_tops, sim_precision=prec, gemm_backend=backend, **mining, **cfg))
    try:
        g = observe(torch, ctx, Q, ctx.forward(xt, lt))
        S = ctx.debug_read(0, Q * Q).reshape(Q, Q)
    finally:
        ctx.close()
    check_rows(g, S, lab, lab, np.arange(Q), mining, prec, num_tops, tag=tag, amb_max=amb_max)
    return g, S


# ------------------------------------------------------------------------------------------------- world 1: shapes and minings
@pytest.mark.parametrize("mining", ["rand", "usage"])
@pytest.mark.parametrize("Q", [2, 3, 33, 129, 255, 1000, 4097])
def test_world1_shapes(torch, Q, mining):
    """Symmetric tiles with mirrored statistics, partial chunks and ragged D; at Q = 2 and 3 the counters use the N - 2 clamp."""
    x, lab = synth.make_inputs(Q, 72 if Q < 1000 else 200, 100 + Q, noise=2.5)
    run_world1(torch, x, lab, MININGS[mining], num_tops=3 + Q % 3 if Q < 4 else 5, tag=f"{mining}")


@pytest.mark.parametrize("mining", list(MININGS))
def test_every_mining(torch, mining):
    x, lab = synth.make_inputs(1000, 128, 7, noise=2.5)
    run_world1(torch, x, lab, MININGS[mining], tag=mining)


def test_all_negative_rows(torch):
    """Row 0 is u and every other row lies in the -u hemisphere: a padding column counted as a similarity of 0 would show in row 0's
    max_between and max_all.  Ragged N = 301."""
    Q, D = 301, 40
    x, lab = synth.make_inputs(Q, D, 21, noise=2.5)
    u = x[0].copy()
    d = x[1:] @ u
    x[1:] -= np.where(d >= 0, 2 * d + 1e-2, 0.0)[:, None] * u[None, :]
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    lab[0] = -1.0
    g, S = run_world1(torch, x, lab, MININGS["rand"], tag="all-negative")
    assert g["max_all"][0] < 0 and g["max_between"][0] < 0


def test_singletons_and_ties(torch):
    """Singleton labels (no same-label column: no hit, A = 0, log 0), groups of four equal rows (exact ties, which count against the
    positive) and a cosine-0.9996 cone."""
    Q, D = 260, 64
    x, _ = synth.make_inputs(Q, D, 22)
    g, _ = run_world1(torch, x, np.arange(Q, dtype=np.float32), MININGS["rand"], tag="singletons")
    assert (g["A"] == 0).all() and (g["logv"] == 0).all() and not g["hits"].any() and (g["cnt_same"] == 0).all()
    x, lab = grad_ref.cone_inputs(Q, D, 0.1, 23, dup=4)
    run_world1(torch, x, lab, MININGS["usage"], tag="dup ties")
    x, lab = grad_ref.cone_inputs(Q, D, 0.02, 24)
    run_world1(torch, x, lab, MININGS["rand"], tag="cone 0.9996", amb_max=None)


def test_unaligned_labels(torch):
    """The label pointer one float off 16-byte alignment sends every row through the tail loop, which adds the same terms in the same
    order per lane as the 16-byte path: every per-row result is bit for bit that of the aligned run."""
    x, lab = synth.make_inputs(1000, 96, 25, noise=2.5)
    a, _ = run_world1(torch, x, lab, MININGS["usage"], tag="aligned")
    b, _ = run_world1(torch, x, lab, MININGS["usage"], tag="offset labels", lab_offset=True)
    for k in ("A", "T", "logv", "hits", "rec", "tops"):
        np.testing.assert_array_equal(a[k].view(np.uint32), b[k].view(np.uint32), err_msg=k)


@pytest.mark.parametrize("prec,backend", [(FP16X2, SIMT), (BF16X3, TC), (BF16, TC), (BF16X3, SIMT)],
                         ids=["simt-fp16x2", "bf16x3", "bf16", "simt-bf16x3"])
def test_other_producers(torch, prec, backend):
    x, lab = synth.make_inputs(384, 72, 26, noise=2.5)
    run_world1(torch, x, lab, MININGS["usage"], prec=prec, backend=backend, tag="producer")


def test_headline_shape(torch):
    """Q = N = 8192, D = 512, usage mining: every row's hit flags exact, no ambiguous row."""
    x, lab = synth.make_inputs(8192, 512, 20171230, noise=2.5)
    run_world1(torch, x, lab, MININGS["usage"], tag="headline")


# ------------------------------------------------------------------------------------------------- other producers of the state
def test_row_blocks(torch):
    """Three blocks of 384 rows and the separate finaliser, against the S of a materialised twin (the same bits)."""
    Q, D = 1024, 96
    x, lab = synth.make_inputs(Q, D, 27, noise=2.5)
    mining = MININGS["usage"]
    xt, lt = torch.from_numpy(x).cuda(), torch.from_numpy(lab).cuda()
    out = {}
    for rows in (0, 384):
        ctx = capi.Context(capi.make_config(Q, D, num_tops=5, sim_block_rows=rows, **mining))
        try:
            out[rows] = observe(torch, ctx, Q, ctx.forward(xt, lt))
            if rows == 0:
                S = ctx.debug_read(0, Q * Q).reshape(Q, Q)
        finally:
            ctx.close()
    check_rows(out[384], S, lab, lab, np.arange(Q), mining, FP16X2, 5, tag="row blocks", amb_max=0)


@pytest.mark.parametrize("world,Q", [(2, 333), (3, 333), (8, 256)])
def test_emulated_world(torch, world, Q):
    """Every rank of a world on one GPU: self columns at rank * Q + i, m2c carries log2(world).  Ragged Q = 333; at world 8, Q = 256
    the row pass runs 4 warps per row over 512-column segments, and rank r's self columns lie in segment r / 2."""
    D = 80
    x, lab = synth.make_inputs(Q * world, D, 28 + world, noise=2.5)
    mining = MININGS["usage"]
    xt, lt = torch.from_numpy(x).cuda(), torch.from_numpy(lab).cuda()
    for r in range(world):
        ctx = capi.Context(capi.make_config(Q, D, world=world, rank=r, num_tops=5, **mining))
        try:
            g = observe(torch, ctx, Q, ctx.forward_gathered(xt, lt))
            S = ctx.debug_read(0, Q * Q * world).reshape(Q, Q * world)
        finally:
            ctx.close()
        check_rows(g, S, lab[r * Q:(r + 1) * Q], lab, np.arange(Q) + r * Q, mining, FP16X2, 5, world=world, tag=f"world {world} rank {r}",
                   amb_max=0)


@pytest.mark.parametrize("Q,m", [(256, 8192), (256, 3000), (1024, 4096)])
def test_memory_rows(torch, Q, m):
    """Cross-batch memory: N = Q + m columns; Q = 256 with m = 8192 runs 8 warps per row, m = 3000 runs 4, Q = 1024 runs 2."""
    D = 64
    x, lab = synth.make_inputs(Q + m, D, 30, noise=2.5)
    lab = np.concatenate([lab[:Q], lab[Q:] % (Q // 2)]).astype(np.float32)
    mining = MININGS["usage"]
    xt, lt, xm, lm = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (x[:Q], lab[:Q], x[Q:], lab[Q:]))
    ctx = capi.Context(capi.make_config(Q, D, num_tops=5, **mining), memory_rows=m)
    try:
        g = observe(torch, ctx, Q, ctx.forward_memory(xt, lt, xm, lm, m))
        S = ctx.debug_read(0, Q * (Q + m)).reshape(Q, Q + m)
    finally:
        ctx.close()
    print(f"memory Q {Q} m {m}: {lse_wpr(Q, Q + m)} warps per row")
    check_rows(g, S, lab[:Q], lab, np.arange(Q), mining, FP16X2, 5, tag=f"memory m {m}", amb_max=0)


# ------------------------------------------------------------------------------------------------- dynamic range
GAPS = (60.0, 78.0, 79.5, 83.0, 86.0, 88.0, 95.0, 102.0, 110.0)
R2 = 128.0                                       # squared norm of the planted rows: every other column lies R2 nats below them


def planted_inputs(Q, D, seed):
    """Un-normalised rows.  Group g (four rows, two dimensions of its own) holds a = b = r u and p, q in the (u, w) plane, labels
    (a, p) and (b, q): row a's maximum is b (gap 0) and its only positive p lies GAPS[g] nats below it; q lies 5 nats further.  Every
    other row (norms 0.5 .. 4, labels in pairs) lives in the remaining dimensions, R2 nats below the planted rows' maxima."""
    rng = np.random.default_rng(seed)
    G = len(GAPS)
    x = np.zeros((Q, D), np.float64)
    lab = np.zeros(Q, np.float32)
    r = np.sqrt(R2)
    for gi, gap in enumerate(GAPS):
        u, w = np.zeros(D), np.zeros(D)
        u[2 * gi], w[2 * gi + 1] = 1.0, 1.0
        cp, cq = 1 - gap / R2, 1 - (gap + 5) / R2
        x[4 * gi] = r * u
        x[4 * gi + 1] = r * (cp * u + np.sqrt(1 - cp * cp) * w)
        x[4 * gi + 2] = r * u
        x[4 * gi + 3] = r * (cq * u - np.sqrt(1 - cq * cq) * w)
        lab[4 * gi:4 * gi + 4] = [1000 + 2 * gi, 1000 + 2 * gi, 1001 + 2 * gi, 1001 + 2 * gi]
    n = Q - 4 * G
    bulk = rng.standard_normal((n, D - 2 * G))
    bulk *= (rng.uniform(0.5, 4.0, n) / np.linalg.norm(bulk, axis=1))[:, None]
    x[4 * G:, 2 * G:] = bulk
    lab[4 * G:] = np.arange(n) // 2
    return np.ascontiguousarray(x, dtype=np.float32), lab


def flushed_step(x, S, ref, Q):
    """grad_ref's world-1 step (R, B, R32) with the weights built from the flushed sums: the terms the row pass drops weigh nothing."""
    E = np.exp(S.astype(np.float64) - ref["max_all"].astype(np.float64)[:, None])
    state = dict(A=ref["A64"], T=ref["T64"], temp1=np.where(ref["kept"] & ref["same"], E, 0.0),
                 temp2=np.where(ref["kept"] & ref["diff"], E, 0.0))
    G, Gabs = grad_ref.weights(state, Q)
    return grad_ref._products(x, [(G, Gabs, slice(0, Q), 0.5, 0.5)])


@pytest.mark.parametrize("path", ["fused", "split"])
@pytest.mark.parametrize("prec", [FP16X2, BF16X3])
def test_dynamic_range(torch, prec, path):
    """Positives 60 .. 110 nats below the row maximum.  Records finite (with j > 0 on the fp16x2 rows past 79 nats), A = 0 and no
    positive weight past 87.3 nats, p* subnormal (95, 102 nats) and zero (110 nats) in retrieval_cut, and the gradient against fp64
    weights built from the flushed A and T."""
    Q, D = 512, 64
    x, lab = planted_inputs(Q, D, 31)
    mining = MININGS["rand"]
    flags = capi.FLAG_NO_FUSED_GRAD if path == "split" else 0
    xt, lt = torch.from_numpy(x).cuda(), torch.from_numpy(lab).cuda()
    ctx = capi.Context(capi.make_config(Q, D, num_tops=5, sim_precision=prec, flags=flags, **mining))
    try:
        tops = ctx.forward(xt, lt)
        dx = torch.full_like(xt, float("nan"))
        ctx.backward(1.0, dx)
        torch.cuda.synchronize()
        dx = dx.cpu().numpy()
        S = ctx.debug_read(0, Q * Q).reshape(Q, Q)
        # the gradient first: it needs nothing but S and the thresholds
        ref = fr.reference(S, lab, lab, np.arange(Q), ctx.debug_read(1, Q), ctx.debug_read(2, Q), mining, wpr=lse_wpr(Q, Q))
        # Two allowances that rows of unit norm never need.  Every weight carries the exponent's relative error, (|m2| + 2 |arg|) ln 2
        # 2^-24 with |m2| up to 185 here (forward_ref.tau_rows; the reference's expf(s - max) has no |m2| term), which the rows' own
        # norm does not bound where weights cancel (a = b): each row may also be off by 4 tau_i ||B_i||.  An fp16x2 weight below 2^-24 of
        # the 2^k scale has no piece at all (fp16's smallest subnormal): the componentwise floor is 2^-(23 + k) (lw / Q) sum_j |x_jd|.
        step = flushed_step(x, S, ref, Q)
        row_extra = 4 * ref["tau"] * np.linalg.norm(step["B"], axis=1)
        floor = 2.0 ** -(23 + K[prec]) / Q * np.abs(x.astype(np.float64)).sum(axis=0)[None, :] if prec == FP16X2 else grad_ref.TINY
        bad, m = grad_ref.violations(dx, step, grad_ref.tau(prec, path, Q), k_sgemm=256.0, floor=floor, row_extra=row_extra)
        print(f"dynamic range {NAME[prec]} {path}: normwise {m['normwise']:.2e} worst row {m['row']:.3f} componentwise "
              f"{m['comp']:.1f} x 2^-24")
        assert not bad, f"dynamic range {NAME[prec]} {path}: " + "; ".join(bad)
        g = observe(torch, ctx, Q, tops)
    finally:
        ctx.close()
    ref, j = check_rows(g, S, lab, lab, np.arange(Q), mining, prec, 5, tag=f"dynamic range {path}", amb_max=None)
    a_rows = 4 * np.arange(len(GAPS))
    gap = (g["max_all"][a_rows] - S[a_rows, a_rows + 1]).astype(np.float64)
    print("gap, A, j of the planted rows:", [(round(float(t), 2), float(g["A"][i]), int(j[i])) for t, i in zip(gap, a_rows)])
    flushed = gap > 126 * np.log(2) + 0.01
    assert (g["A"][a_rows][flushed] == 0).all() and (g["logv"][a_rows][flushed] == 0).all()
    assert (g["A"][a_rows][~flushed] > 0).all()
    if prec == FP16X2:
        assert ((j[a_rows] > 0) == ((gap > np.log(2.0) * 114) & ~flushed)).all(), j[a_rows]
    else:
        assert (j == 0).all()
    hits = g["hits"].reshape(3, Q)[:, a_rows]
    pstar = np.exp(-gap).astype(np.float32)                  # expf(max_within - max_all)
    print("hits k = 1, 5, 10 of the planted rows:", hits.T.astype(int).tolist())
    assert not hits[:, pstar == 0].any()                     # p* underflows: every column ties with the positive
    assert hits[1:, (pstar > 0) & (pstar < 2.0 ** -126)].all()   # p* subnormal: the positive is second, after b
