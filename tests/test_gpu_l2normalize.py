"""SURVEY 8f-1: the L2Normalize producer layer (usage/def.prototxt:115-120) -- stand-alone ABI calls and fused into the loss
layer (npair_config.normalize_input) -- against the oracle's statement of the layer composed with the oracle of the loss."""
import numpy as np
import pytest

from npairloss_b200 import capi, synth

pytestmark = pytest.mark.gpu


def _raw_inputs(B, D, seed, noise=2.5):
    x, lab = synth.make_inputs(B, D, seed, noise=noise)
    scale = np.random.default_rng(seed + 1).uniform(0.3, 30.0, size=(B, 1)).astype(np.float32)
    return np.ascontiguousarray(x * scale), lab


def test_standalone_forward_backward(oracle):
    import torch
    for (R, D) in [(64, 128), (1000, 200), (7, 3), (4096, 512)]:
        x, _ = _raw_inputs(R, D, 3 + R)
        x[R // 2] = 0.0                                              # a zero row stays zero, its gradient is zero
        dy = np.random.default_rng(R).standard_normal((R, D)).astype(np.float32)
        y, inv = capi.l2normalize_forward(torch.from_numpy(x).cuda())
        dx = capi.l2normalize_backward(y, inv, torch.from_numpy(dy).cuda())
        y_o, inv_o = oracle.l2normalize_forward(x)
        dx_o = oracle.l2normalize_backward(y_o, inv_o, dy)
        np.testing.assert_allclose(y.cpu().numpy(), y_o, rtol=3e-7, atol=1e-30)
        np.testing.assert_allclose(inv.cpu().numpy(), inv_o, rtol=3e-7)
        assert np.linalg.norm(dx.cpu().numpy() - dx_o) <= 2e-6 * np.linalg.norm(dx_o)
        assert not y.cpu().numpy()[R // 2].any() and not dx.cpu().numpy()[R // 2].any()


@pytest.mark.parametrize("R,D", [(64, 128), (1000, 200), (7, 3)])
def test_standalone_buffers_at_any_offset(R, D):
    """Every buffer 1, 2 or 3 floats into a larger allocation: the 4-byte-load fallback keeps the summation order of the 16-byte
    path, so y, 1/||x|| and dx are bit for bit those of aligned buffers."""
    import torch
    x, _ = _raw_inputs(R, D, 5 + R)
    dy = np.random.default_rng(R + 1).standard_normal((R, D)).astype(np.float32)
    xt, dyt = torch.from_numpy(x).cuda(), torch.from_numpy(dy).cuda()
    y0, inv0 = capi.l2normalize_forward(xt)
    dx0 = capi.l2normalize_backward(y0, inv0, dyt)
    L, st = capi.lib(), torch.cuda.current_stream().cuda_stream
    for off in (1, 2, 3):
        def at(t):
            buf = torch.full((t.numel() + off,), float("nan"), dtype=torch.float32, device="cuda")
            v = buf[off:].view(t.shape)
            v.copy_(t)
            return v
        xv, dyv, y, dx = at(xt), at(dyt), at(torch.empty_like(xt)), at(torch.empty_like(xt))
        inv = at(torch.empty_like(inv0))
        assert L.npair_l2normalize_forward(xv.data_ptr(), R, D, y.data_ptr(), inv.data_ptr(), st) == 0
        assert L.npair_l2normalize_backward(y.data_ptr(), inv.data_ptr(), dyv.data_ptr(), R, D, dx.data_ptr(), st) == 0
        torch.cuda.synchronize()
        for got, want, what in ((y, y0, "y"), (inv, inv0, "1/||x||"), (dx, dx0, "dx")):
            assert torch.equal(got.view(torch.int32), want.view(torch.int32)), f"R{R} D{D} offset {off}: {what}"


@pytest.mark.parametrize("B,D,mining", [(512, 128, "usage"), (1000, 200, "default"), (2048, 512, "usage")])
def test_fused_normalize_input_world1(oracle, B, D, mining):
    import torch
    m = {"usage": synth.USAGE_MINING, "default": synth.DEFAULT_MINING}[mining]
    x, lab = _raw_inputs(B, D, 11 + B)
    ctx = capi.Context(capi.make_config(B, D, normalize_input=1, **m))
    dx_t, dl_t = torch.from_numpy(x).cuda(), torch.from_numpy(lab).cuda()
    g = torch.full_like(dx_t, float("nan"))
    tops = ctx.forward(dx_t, dl_t)
    ctx.backward(0.7, g)
    torch.cuda.synchronize()
    S = ctx.debug_read(0, B * B).reshape(B, B)
    ctx.close()
    y_o, inv_o = oracle.l2normalize_forward(x)
    assert np.abs(S - (y_o.astype(np.float64) @ y_o.astype(np.float64).T)).max() <= 1e-6 + 1.5e-5
    tops_o, dy_o = oracle.step_world(y_o, lab, oracle.make_config(B, D, faithful_sorts=0, **m), 0.7, S_inject_all=S)
    dx_o = oracle.l2normalize_backward(y_o, inv_o, dy_o)
    assert abs(tops[0] - tops_o[0, 0]) <= 1e-5 * abs(tops_o[0, 0]) + 1e-6
    assert abs(tops[4] - tops_o[0, 4]) <= 2e-6 * abs(tops_o[0, 4])          # feature_asum is taken on the normalised bottom
    gd = g.cpu().numpy()
    assert np.isfinite(gd).all()
    assert np.linalg.norm(gd - dx_o) <= 1e-5 * np.linalg.norm(dx_o)
    # the fused layer equals the two stand-alone layers chained
    y, inv = capi.l2normalize_forward(dx_t)
    ctx2 = capi.Context(capi.make_config(B, D, **m))
    g2 = torch.empty_like(dx_t)
    tops2 = ctx2.forward(y, dl_t)
    ctx2.backward(0.7, g2)
    dx2 = capi.l2normalize_backward(y, inv, g2)
    torch.cuda.synchronize()
    ctx2.close()
    assert tops2 == tops and torch.equal(dx2, g)


def test_fused_normalize_input_two_ranks(oracle):
    """world = 2 through the external-collectives ABI: the gathered bottoms are raw embeddings."""
    import torch
    Q, D, world = 160, 96, 2
    x, lab = _raw_inputs(Q * world, D, 5)
    dev = torch.device("cuda:0")
    xt, lt = torch.from_numpy(x).to(dev), torch.from_numpy(lab).to(dev)
    N = Q * world
    ctxs, S, tops = [], np.zeros((N, N), np.float32), np.zeros((world, 5), np.float32)
    rs = torch.empty((world, Q, 8), dtype=torch.float32, device=dev)
    for r in range(world):
        c = capi.Context(capi.make_config(Q, D, world=world, rank=r, normalize_input=1, **synth.USAGE_MINING))
        tops[r] = c.forward_gathered(xt, lt)
        c.row_scalars(rs[r])
        S[r * Q:(r + 1) * Q] = c.debug_read(0, Q * N).reshape(Q, N)
        ctxs.append(c)
    gd = np.zeros((N, D), np.float32)
    for r in range(world):
        g = torch.full((Q, D), float("nan"), dtype=torch.float32, device=dev)
        ctxs[r].backward_gathered(1.0, rs, g)
        gd[r * Q:(r + 1) * Q] = g.cpu().numpy()
        ctxs[r].close()
    y_o, inv_o = oracle.l2normalize_forward(x)
    tops_o, dy_o = oracle.step_world(y_o, lab, oracle.make_config(Q, D, world=world, faithful_sorts=0, **synth.USAGE_MINING), 1.0, S_inject_all=S)
    dx_o = oracle.l2normalize_backward(y_o, inv_o, dy_o)
    np.testing.assert_allclose(tops[:, 0], tops_o[:, 0], rtol=1e-5, atol=1e-6)
    assert np.linalg.norm(gd - dx_o) <= 1e-5 * np.linalg.norm(dx_o)
