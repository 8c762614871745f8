"""The similarity sweep's S against sim_ref's exact model and fp64 (rules (i) - (iii)) on every path that computes it: the layer at
world 1 (symmetric tiles, mirrored stores), emulated worlds 2 and 3, the cross-batch memory step with memory rows far larger and
smaller than the batch, the SIMT check backend, the evaluator's k-NN with k = every column (its q != g S rows, full tiles) and its
best positive with labels in pairs (S[i][partner] through EPI_STATS | EPI_SYM); at ragged D and row counts, the HL shape, every
operand format, and inputs whose cross terms matter: one-chunk probes, mixed norms, spikes, cones, duplicates and both ends of the
fp32 range.  Every case prints its largest |S - M| / B in units of 2^-24 (SIMRATIO lines, pytest -s)."""
import numpy as np
import pytest

from npairloss_b200 import capi
import gpu_harness
import sim_ref
from sim_ref import BF16, BF16X3, FP16X2, KINDS, PRECS

pytestmark = pytest.mark.gpu
RAND = dict(ap_region=1, ap_method=2, an_region=1, an_method=2)
PNAME = {FP16X2: "fp16x2", BF16X3: "bf16x3", BF16: "bf16"}


@pytest.fixture(scope="module")
def torch():
    import torch
    assert torch.cuda.is_available() and torch.cuda.get_device_capability(0) == (9, 0), "GPU tests need an H100"
    return torch


def _check(S, xa, xb, prec, path, tag, absmax=None):
    bad, m = sim_ref.check(S, xa, xb, prec, "simt" if path == "simt" else "tc", absmax=absmax)
    print(f"SIMRATIO {PNAME[prec]:7s} {path:8s} {tag:32s} ratio {m['ratio']:9.2f}  of tau {m['worst']:.3f}")
    assert not bad, f"{PNAME[prec]} {path} {tag}: {bad}"


def _labels(n):
    return (np.arange(n) // 2).astype(np.float32)


def _layer_S(torch, x, prec, backend=capi.GEMM_TCGEN05):
    """The world-1 layer's S (debug_read(0)); a forward that stops on a device error (S with infinities) still leaves S."""
    Q, D = x.shape
    ctx = capi.Context(capi.make_config(Q, D, sim_precision=prec, gemm_backend=backend, num_tops=2, **RAND))
    try:
        try:
            ctx.forward(torch.from_numpy(x).cuda(), torch.from_numpy(_labels(Q)).cuda())
        except capi.NpairError:
            pass
        torch.cuda.synchronize()
        return ctx.debug_read(0, Q * Q).reshape(Q, Q)
    finally:
        ctx.close()


def _knn_S(torch, q, g, prec, absmax=-1.0, ev=None):
    """S[q, g] from the evaluator's k-NN with k = every column, sorted back by index; galleries above 1024 rows in shards of 1024
    with the shared absmax of both sets."""
    nq, ng = q.shape[0], g.shape[0]
    own = ev is None
    ev = ev or capi.Evaluator(nq, min(ng, 1024), q.shape[1], prec)
    if ng > 1024 and absmax < 0:
        absmax = float(max(np.abs(q).max(), np.abs(g).max()))
    S = np.empty((nq, ng), np.float32)
    try:
        qt = torch.from_numpy(q).cuda()
        for c0 in range(0, ng, 1024):
            gs = np.ascontiguousarray(g[c0:c0 + 1024])
            sim, idx = ev.knn(qt, torch.from_numpy(gs).cuda(), gs.shape[0], gallery_row0=c0, absmax=absmax)
            torch.cuda.synchronize()
            sim, idx = sim.cpu().numpy(), idx.cpu().numpy()
            assert (np.sort(idx, 1) == np.arange(c0, c0 + gs.shape[0])[None, :]).all()
            np.put_along_axis(S[:, c0:c0 + gs.shape[0]], idx - c0, sim, 1)
    finally:
        if own:
            ev.close()
    return S


# ------------------------------------------------------------------------------------------------------------- the layer at world 1
D_LIST = [1, 8, 15, 16, 17, 31, 32, 33, 64, 65, 100, 128, 129, 512, 1024, 2048, 4096]
ROWS = [1, 7, 8, 9, 127, 128, 129, 255, 256, 257, 1000]
KIND_CYCLE = ["probe", "dense", "mixed", "cone0.99", "spike"]


@pytest.mark.parametrize("prec", PRECS)
def test_layer_every_D(torch, prec):
    for i, D in enumerate(D_LIST):
        rows = 160 if D <= 1024 else 72
        for kind in ("probe", KIND_CYCLE[1 + i % 4]):
            x = KINDS[kind](rows, D, 100 + i)
            _check(_layer_S(torch, x, prec), x, x, prec, "layer", f"{kind} {rows}x{D}")


@pytest.mark.parametrize("prec", PRECS)
def test_layer_every_row_count(torch, prec):
    for i, rows in enumerate(ROWS):
        for D in (33, 129):
            kind = KIND_CYCLE[i % len(KIND_CYCLE)]
            x = KINDS[kind](rows, D, 200 + i)
            _check(_layer_S(torch, x, prec), x, x, prec, "layer", f"{kind} {rows}x{D}")


@pytest.mark.parametrize("kind", sorted(KINDS))
@pytest.mark.parametrize("prec", PRECS)
def test_layer_every_kind(torch, prec, kind):
    """Every input kind at a shape with ragged tiles and a ragged last chunk; tiny and huge are the ends of the fp32 range, where the
    fp16x2 pre-scale's exponent is clamped"""
    x = KINDS[kind](300, 130, 7)
    _check(_layer_S(torch, x, prec), x, x, prec, "layer", f"{kind} 300x130")


@pytest.mark.parametrize("prec", [FP16X2, BF16X3])
def test_layer_hl(torch, prec):
    x = KINDS["cone0.99"](8192, 512, 11)
    _check(_layer_S(torch, x, prec), x, x, prec, "layer", "cone0.99 8192x512 (HL)")


# --------------------------------------------------------------------------------------------- emulated worlds, SIMT check, memory step
@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("prec", PRECS)
def test_emulated_worlds(torch, prec, world):
    for kind in ("probe", "mixed", "cone0.9996", "dup"):
        Q = 136
        x = KINDS[kind](Q * world, 100, 30 + world)
        g = gpu_harness.gpu_step_world(x, _labels(Q * world), Q, world, RAND, prec, capi.GEMM_TCGEN05, want_grad=False)
        _check(g["S"], x, x, prec, f"world{world}", f"{kind} {Q}x{world}x100")


@pytest.mark.parametrize("prec", PRECS)
def test_simt_check_backend(torch, prec):
    for kind in ("probe", "mixed", "spike", "cone0.99", "tiny", "huge"):
        x = KINDS[kind](130, 200, 41)
        _check(_layer_S(torch, x, prec, capi.GEMM_SIMT_CHECK), x, x, prec, "simt", f"{kind} 130x200")


@pytest.mark.parametrize("mem_scale", [2.0 ** 6, 2.0 ** -6])
@pytest.mark.parametrize("prec", PRECS)
def test_memory_step(torch, prec, mem_scale):
    """The pre-scale covers the batch and the memory rows: memory rows 2^6 times larger or smaller than the batch's"""
    Q, m, D = 192, 520, 129
    for kind in ("dense", "probe", "cone0.99"):
        xa = KINDS[kind](Q + m, D, 51)
        x, xm = np.ascontiguousarray(xa[:Q]), np.ascontiguousarray(xa[Q:] * np.float32(mem_scale))
        lab = _labels(Q + m)
        ctx = capi.Context(capi.make_config(Q, D, sim_precision=prec, num_tops=2, **RAND), memory_rows=m)
        try:
            t = [torch.from_numpy(a).cuda() for a in (x, lab[:Q], xm, lab[Q:])]
            ctx.forward_memory(*t, m)
            torch.cuda.synchronize()
            S = ctx.debug_read(0, Q * (Q + m)).reshape(Q, Q + m)
        finally:
            ctx.close()
        _check(S, x, np.concatenate([x, xm]), prec, "memory", f"{kind} x{mem_scale:g} {Q}+{m}x{D}")


# --------------------------------------------------------------------------------------------------------------------- the evaluator
@pytest.mark.parametrize("prec", PRECS)
def test_knn_queries_not_gallery(torch, prec):
    """q != g with values that exercise the cross terms, full tiles, ragged D; a 2500-row gallery in shards with the shared absmax"""
    for i, (kind, nq, ng, D) in enumerate([("probe", 200, 700, 100), ("mixed", 129, 1000, 65), ("spike", 64, 300, 512),
                                           ("cone0.9996", 130, 257, 33), ("dense", 96, 2500, 129), ("tiny", 40, 50, 17),
                                           ("huge", 40, 50, 17)]):
        x = KINDS[kind](nq + ng, D, 60 + i)
        q, g = np.ascontiguousarray(x[:nq]), np.ascontiguousarray(x[nq:])
        if kind == "huge":
            q, g = np.ascontiguousarray(x[::-1][:nq]), np.ascontiguousarray(x[::-1][nq:])     # the huge row among the gallery's
        _check(_knn_S(torch, q, g, prec), q, g, prec, "knn", f"{kind} {nq}x{ng}x{D}")


@pytest.mark.parametrize("prec", PRECS)
def test_best_positive_partner(torch, prec):
    """Labels in pairs across the query and gallery sets: each query's best positive is S[i][partner(i)], produced by the statistics
    sweep (EPI_STATS; EPI_SYM when the gallery is the query set)"""
    for i, (kind, n, D) in enumerate([("probe", 300, 100), ("mixed", 257, 129), ("cone0.99", 130, 512)]):
        x = KINDS[kind](2 * n, D, 70 + i)
        rng = np.random.default_rng(i)
        perm = rng.permutation(n)
        q, g = np.ascontiguousarray(x[:n]), np.ascontiguousarray(x[n:])
        ql = np.arange(n, dtype=np.float32)
        gl = np.empty(n, np.float32)
        gl[perm] = ql                          # gallery row perm[i] is query i's partner
        ev = capi.Evaluator(n, n, D, prec)
        try:
            amax = float(max(np.abs(q).max(), np.abs(g).max()))
            best = ev.best_positive(*[torch.from_numpy(a).cuda() for a in (q, ql, g, gl)], amax).cpu().numpy()
            # the same labels within one set: pairs (2j, 2j + 1), the self pair excluded, through EPI_SYM
            lp = (np.arange(n) // 2).astype(np.float32)
            qt, lt = torch.from_numpy(q).cuda(), torch.from_numpy(lp).cuda()
            best_sym = ev.best_positive(qt, lt, qt, lt, float(np.abs(q).max()), self_offset=0).cpu().numpy()
            torch.cuda.synchronize()
        finally:
            ev.close()
        ref = sim_ref.model(q, g[perm], prec, amax)
        diag = {k: v.diagonal()[:, None] for k, v in ref.items()}
        bad, m = sim_ref.violations(best[:, None], diag, sim_ref.tau(prec, "tc", diag["L"]))
        print(f"SIMRATIO {PNAME[prec]:7s} best     {kind} {n}x{D} ratio {m['ratio']:9.2f}  of tau {m['worst']:.3f}")
        assert not bad, (kind, bad)
        even = (n // 2) * 2
        partner = np.arange(even) ^ 1
        ref = sim_ref.model(q[:even], q[partner], prec)
        diag = {k: v.diagonal()[:, None] for k, v in ref.items()}
        bad, m = sim_ref.violations(best_sym[:even, None], diag, sim_ref.tau(prec, "tc", diag["L"]))
        print(f"SIMRATIO {PNAME[prec]:7s} best_sym {kind} {n}x{D} ratio {m['ratio']:9.2f}  of tau {m['worst']:.3f}")
        assert not bad, (kind, "sym", bad)
