"""The fused gradient kernel's two weight builders (DESIGN 4): a warp's K step without a same-label pair, a self pair or a column past
N takes the different-label builder, every other step the general one.  NPAIR_FLAG_GRAD_GENERAL sends every step through the general
builder; the gradient must keep every bit.  Shuffled labels with 8 images per class put same-label pairs in many steps and leave many
without, so both builders run side by side in the same tiles; ragged N leaves a partial last K step."""
import numpy as np
import pytest

from npairloss_b200 import capi, synth
from gpu_harness import gpu_step_world

pytestmark = pytest.mark.gpu

FP16X2, BF16X3, BF16 = capi.PREC_FP32_FP16X2, capi.PREC_FP32_BF16X3, capi.PREC_BF16
GENERAL = capi.FLAG_GRAD_GENERAL
# an_method HARD / RELATIVE_HARD compare -s (the different-label builder's folded sign), the others +s
MININGS = {"usage": dict(synth.USAGE_MINING), "rand": dict(synth.DEFAULT_MINING),
           "easy": dict(synth.USAGE_MINING, an_method=synth.RELATIVE_EASY, diffsn=-0.4),
           "relative": dict(ap_region=1, ap_method=3, an_region=1, an_method=3, identsn=-0.4, diffsn=-0.3)}


@pytest.fixture(scope="module")
def torch():
    import torch
    assert torch.cuda.is_available() and torch.cuda.get_device_capability(0) == (9, 0), "GPU tests need an H100"
    return torch


def _shuffled(n, D, seed, imgs=8, noise=2.0):
    x, lab = synth.make_inputs(n, D, seed=seed, imgs_per_class=imgs, noise=noise)
    p = np.random.default_rng(seed).permutation(n)
    return np.ascontiguousarray(x[p]), np.ascontiguousarray(lab[p])


def _step(torch, x, lab, flags, prec, mining, **extra):
    Q, D = x.shape
    ctx = capi.Context(capi.make_config(Q, D, sim_precision=prec, flags=flags, **mining, **extra))
    try:
        xt, lt = torch.from_numpy(x).cuda(), torch.from_numpy(lab).cuda()
        tops = np.array(ctx.forward(xt, lt), dtype=np.float32)
        dx = torch.full_like(xt, float("nan"))
        ctx.backward(0.7, dx)
        torch.cuda.synchronize()
        return tops, dx.cpu().numpy()
    finally:
        ctx.close()


def _same_bits(a, b, tag):
    assert np.isfinite(a).all(), f"{tag}: non-finite gradient"
    np.testing.assert_array_equal(a.view(np.uint32), b.view(np.uint32), err_msg=tag)


@pytest.mark.parametrize("prec", [FP16X2, BF16X3, BF16])
@pytest.mark.parametrize("mining", sorted(MININGS))
@pytest.mark.parametrize("Q,D", [(1000, 128), (2053, 64)])
def test_builders_match(torch, prec, mining, Q, D):
    x, lab = _shuffled(Q, D, seed=Q + D)
    t0, g0 = _step(torch, x, lab, 0, prec, MININGS[mining])
    t1, g1 = _step(torch, x, lab, GENERAL, prec, MININGS[mining])
    np.testing.assert_array_equal(t0, t1)
    assert np.abs(g0).max() > 0, "no pair selected: the comparison says nothing"
    _same_bits(g0, g1, f"prec {prec} {mining} Q {Q} D {D}")


def test_builders_match_nan_labels(torch):
    """NaN labels equal nothing, their own included: a NaN row's pairs are all different-label"""
    x, lab = _shuffled(777, 64, seed=5)
    lab[::7] = np.nan
    t0, g0 = _step(torch, x, lab, 0, FP16X2, MININGS["usage"])
    t1, g1 = _step(torch, x, lab, GENERAL, FP16X2, MININGS["usage"])
    np.testing.assert_array_equal(t0, t1)
    _same_bits(g0, g1, "NaN labels")


@pytest.mark.parametrize("mining", ["usage", "rand"])
def test_builders_match_row_blocks(torch, mining):
    """row-block mode: each block's launch starts at a later row, so its self columns move with it"""
    x, lab = _shuffled(1100, 128, seed=11)
    t0, g0 = _step(torch, x, lab, 0, FP16X2, MININGS[mining], sim_block_rows=256)
    t1, g1 = _step(torch, x, lab, GENERAL, FP16X2, MININGS[mining], sim_block_rows=256)
    t2, g2 = _step(torch, x, lab, 0, FP16X2, MININGS[mining])
    np.testing.assert_array_equal(t0, t1)
    _same_bits(g0, g1, f"row blocks {mining}")
    _same_bits(g0, g2, f"row blocks against S whole {mining}")


@pytest.mark.parametrize("prec", [FP16X2, BF16X3])
def test_builders_match_memory_step(torch, prec):
    """cross-batch memory: the memory rows' columns lie past Q, their records weigh nothing in the transposed term"""
    Q, m, D = 600, 1000, 128
    x, lab = _shuffled(Q + m, D, seed=3)
    xt, lt = torch.from_numpy(x).cuda(), torch.from_numpy(lab).cuda()
    out = []
    for flags in (0, GENERAL):
        ctx = capi.Context(capi.make_config(Q, D, sim_precision=prec, flags=flags, **MININGS["usage"]), memory_rows=m)
        try:
            tops = np.array(ctx.forward_memory(xt[:Q], lt[:Q], xt[Q:], lt[Q:], m), dtype=np.float32)
            dx = torch.full_like(xt[:Q], float("nan"))
            ctx.backward(0.7, dx)
            torch.cuda.synchronize()
            out.append((tops, dx.cpu().numpy()))
        finally:
            ctx.close()
    np.testing.assert_array_equal(out[0][0], out[1][0])
    assert np.abs(out[0][1]).max() > 0
    _same_bits(out[0][1], out[1][1], f"memory step prec {prec}")


@pytest.mark.parametrize("bwd_exchange", [0, 1])
def test_builders_match_emulated_world2(torch, bwd_exchange):
    """world 2: rank r's self columns start at r Q, and its column records are the world's"""
    Q, world, D = 520, 2, 128
    x, lab = _shuffled(Q * world, D, seed=7)
    r0 = gpu_step_world(x, lab, Q, world, MININGS["usage"], FP16X2, capi.GEMM_TCGEN05, bwd_exchange=bwd_exchange)
    r1 = gpu_step_world(x, lab, Q, world, MININGS["usage"], FP16X2, capi.GEMM_TCGEN05, bwd_exchange=bwd_exchange, flags=GENERAL)
    np.testing.assert_array_equal(r0["tops"], r1["tops"])
    assert np.abs(r0["dx"]).max() > 0
    _same_bits(r0["dx"], r1["dx"], f"world 2 exchange {bwd_exchange}")
