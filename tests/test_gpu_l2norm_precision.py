"""The L2Normalize producer (l2norm_fwd_kernel / l2norm_bwd_kernel) against fp64 by l2norm_ref, componentwise, at both ends of the
fp32 range and on all three load paths (aligned 16-byte vec, unaligned quad, scalar); power-of-two invariance bit for bit; a row
offset past 2^31 elements; and the layer with normalize_input = 1 bit for bit against the layer without it on rows normalised by the
stand-alone call, on every forward path."""
import numpy as np
import pytest

import l2norm_ref as ref
from npairloss_b200 import capi, synth

pytestmark = pytest.mark.gpu

F32 = np.float32
D_LIST = [1, 2, 3, 4, 5, 31, 32, 33, 127, 128, 129, 200, 512, 1024, 4095, 4096, 8192]
ROWS = [1, 7, 8, 9, 1000, 8193]


@pytest.fixture(scope="module")
def torch():
    import torch
    assert torch.cuda.is_available() and torch.cuda.get_device_capability(0) == (9, 0), "GPU tests need an H100"
    return torch


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _same(a, b):
    """Bit for bit, except that any NaN matches any NaN (the device's canonical NaN differs from a NaN numpy propagates)."""
    na, nb = np.isnan(a), np.isnan(b)
    return bool((na == nb).all()) and np.array_equal(_bits(np.where(na, 0, a).astype(F32)), _bits(np.where(nb, 0, b).astype(F32)))


def _special_rows(D, seed):
    """Rows at the ends of the range: spikes at every exponent 2^-149 .. 2^127, norms > FLT_MAX, subnormal elements, +-0, NaN, inf."""
    rng = np.random.default_rng(seed)
    rows = []
    for e in range(-149, 128):
        s = np.zeros(D, F32); s[(e * 7) % D] = np.ldexp(F32(rng.uniform(1, 2)) if e < 127 else F32(1.0), e); rows.append(s)
    rows.append(np.full(D, np.ldexp(F32(1.0), 127), F32))                  # ||x|| = sqrt(D) 2^127 > FLT_MAX for D >= 2
    rows.append(np.full(D, F32(3.0e38), F32))
    rows.append(np.ldexp(rng.uniform(-1, 1, D), -140).astype(F32))          # subnormal elements
    rows.append((rng.uniform(-1, 1, D) * 1e-40).astype(F32))
    rows.append(np.zeros(D, F32))
    rows.append(-np.zeros(D, F32))
    for bad in (np.nan, np.inf, -np.inf):
        s = rng.standard_normal(D).astype(F32); s[rng.integers(D)] = bad; rows.append(s)
    return np.stack(rows)


def _inputs(R, D, seed):
    """R rows: Gaussian rows at norms spread over 2^-140 .. 2^127, the special rows mixed in (as many as fit)."""
    rng = np.random.default_rng(seed)
    g = rng.standard_normal((R, D)).astype(F32)
    k = rng.integers(-140, 124, size=R)
    k[: R // 4] = 0
    x = np.ldexp(g, k[:, None]).astype(F32)
    sp = _special_rows(D, seed + 1)
    pick = rng.permutation(R)[: min(R, sp.shape[0])]
    x[pick] = sp[rng.permutation(sp.shape[0])[: pick.size]]
    return x


def _at(torch, a, off):
    """a on the device, `off` floats into a larger allocation (off = 0: the allocation itself, 16-byte aligned)."""
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    if off == 0:
        return t
    buf = torch.full((t.numel() + off,), float("nan"), dtype=torch.float32, device="cuda")
    v = buf[off:].view(t.shape)
    v.copy_(t)
    return v


def _run(torch, x, dy, off=0):
    """(y, inv, dx) of the stand-alone calls with every buffer `off` floats off alignment."""
    R, D = x.shape
    L, st = capi.lib(), torch.cuda.current_stream().cuda_stream
    xv, dyv = _at(torch, x, off), _at(torch, dy, off)
    y, dx = _at(torch, np.zeros_like(x), off), _at(torch, np.zeros_like(x), off)
    inv = _at(torch, np.zeros(R, F32), off)
    assert L.npair_l2normalize_forward(xv.data_ptr(), R, D, y.data_ptr(), inv.data_ptr(), st) == 0
    assert L.npair_l2normalize_backward(y.data_ptr(), inv.data_ptr(), dyv.data_ptr(), R, D, dx.data_ptr(), st) == 0
    torch.cuda.synchronize()
    return y.cpu().numpy(), inv.cpu().numpy(), dx.cpu().numpy()


MAX = {"y": 0.0, "inv": 0.0, "dx": 0.0, "chain": 0.0}


@pytest.mark.parametrize("D", D_LIST)
def test_componentwise_every_path(torch, D):
    """Every row count, both alignments (vec / quad when D % 4 == 0, scalar otherwise), against the rules of l2norm_ref and bit for
    bit against its fp32 emulation of the kernels' order."""
    for R in ROWS:
        if R * D > 1 << 23:
            continue
        x = _inputs(R, D, 1000 * D + R)
        dy = np.random.default_rng(R + D).standard_normal((R, D)).astype(F32)
        outs = []
        ye, ie = ref.emulate_forward(x)
        for off in (0, 1):
            y, inv, dx = _run(torch, x, dy, off)
            assert _same(y, ye) and _same(inv, ie), f"R{R} D{D} off{off}: forward differs from the fp32 emulation of its order"
            assert _same(dx, ref.emulate_backward(y, inv, dy)), f"R{R} D{D} off{off}: backward differs from the emulation"
            v, m = ref.check_forward(x, y, inv)
            assert not v, f"R{R} D{D} off{off}: {v}"
            vb, mb = ref.check_backward(y, inv, dy, dx)
            assert not vb, f"R{R} D{D} off{off}: {vb}"
            fin = np.isfinite(x).all(axis=1)
            vc, mc = ref.check_chain(x[fin], dy[fin], dx[fin])
            assert not vc, f"R{R} D{D} off{off}: {vc}"
            for k, val in (("y", m["y"]), ("inv", m["inv"]), ("dx", mb), ("chain", mc)):
                MAX[k] = max(MAX[k], val)
            outs.append((y, inv, dx))
        for a, b in zip(outs[0], outs[1]):                      # the load path does not change the summation order
            assert np.array_equal(_bits(a), _bits(b)), f"R{R} D{D}: aligned and unaligned buffers differ"
    print(f"L2NORM_RATIO D={D} max ratios of the bounds so far: {MAX}")


@pytest.mark.parametrize("D", [1, 3, 4, 33, 128, 200, 4096])
def test_power_of_two_invariance(torch, D):
    """x with elements in [2^-20, 2^4] or exactly 0: y(x 2^k) == y(x), inv(x 2^k) == inv(x) 2^-k and dx(x 2^k) == dx(x) 2^-k bit for
    bit, where those values are normal floats.  The unscaled kernel fails this at |k| >~ 62."""
    rng = np.random.default_rng(D)
    R = 24
    x = np.ldexp(rng.uniform(1, 2, (R, D)) * rng.choice([-1, 1], (R, D)), rng.integers(-20, 4, (R, D))).astype(F32)
    x[rng.random((R, D)) < 0.2] = 0
    x[0] = 0; x[0, 0] = 1.0
    dy = rng.standard_normal((R, D)).astype(F32)
    y0, i0, dx0 = _run(torch, x, dy)
    for k in (-106, -90, -75, -64, -63, 0, 60, 63, 64, 100, 123):
        for off in (0, 1):
            y, inv, dx = _run(torch, np.ldexp(x, k).astype(F32), dy, off)
            assert np.array_equal(_bits(y), _bits(y0)), f"D{D} k{k} off{off}: y"
            want = np.ldexp(i0.astype(np.float64), -k)
            n = (np.abs(want) >= 2.0 ** -126) & (np.abs(want) <= ref.FLT_MAX)
            assert np.array_equal(_bits(inv[n]), _bits(want[n].astype(F32))), f"D{D} k{k} off{off}: inv"
            want = np.ldexp(dx0.astype(np.float64), -k)       # exact where dx and the row's 1/||x 2^k|| are normal floats
            n = (np.abs(want) >= 2.0 ** -126) & (np.abs(want) <= ref.FLT_MAX) & (inv >= 2.0 ** -126)[:, None]
            assert np.array_equal(_bits(dx[n]), _bits(want[n].astype(F32))), f"D{D} k{k} off{off}: dx"


def test_nonfinite_rows_leave_the_others_unchanged(torch):
    x = synth.make_inputs(64, 129, 5)[0]
    dy = np.random.default_rng(6).standard_normal(x.shape).astype(F32)
    y0, i0, dx0 = _run(torch, x, dy)
    bad = [3, 8, 40, 63]
    x[3, 7], x[8, 0], x[40, 128] = np.nan, np.inf, -np.inf
    x[63] = np.nan
    y, inv, dx = _run(torch, x, dy)
    keep = np.setdiff1d(np.arange(64), bad)
    for a, b in ((y, y0), (inv, i0), (dx, dx0)):
        assert np.array_equal(_bits(a[keep]), _bits(b[keep]))
    assert np.isnan(y[bad]).all() and np.isnan(inv[bad]).all() and np.isnan(dx[bad]).all()


def test_inf_inv_norm_gives_no_nan_gradient(torch):
    """||x|| < 2^-128: inv = +inf, and dx is +-inf or exactly 0 (0 where dy - y (y . dy) is 0), never NaN."""
    D = 64
    x = np.zeros((3, D), F32)
    x[0, :3] = np.ldexp(F32(1.0), -140)
    x[1, 5] = np.ldexp(F32(1.0), -149)
    x[2, ::2] = np.ldexp(F32(1.5), -133)
    dy = np.zeros_like(x); dy[:, 1] = 1.0; dy[0, 0] = 1.0; dy[2, 4] = -2.0
    y, inv, dx = _run(torch, x, dy)
    assert (inv == np.inf).all(), inv
    assert not np.isnan(dx).any() and ((dx == 0) | np.isinf(dx)).all()
    assert not ref.check_backward(y, inv, dy, dx)[0]


def test_nan_inv_norm_gives_a_nan_gradient(torch):
    """The stand-alone backward with a caller's NaN 1/||x|| beside a finite y: the row's gradient is NaN, also where dy - y (y . dy)
    is 0; +inf keeps those components 0."""
    D = 8
    y = np.zeros((2, D), F32); y[:, 0] = 1.0
    dy = np.zeros((2, D), F32); dy[:, 3] = 1.0
    inv = np.array([np.nan, np.inf], F32)
    L, st = capi.lib(), torch.cuda.current_stream().cuda_stream
    yt, it, gt = (torch.from_numpy(a).cuda() for a in (y, inv, dy))
    dx = torch.empty_like(yt)
    assert L.npair_l2normalize_backward(yt.data_ptr(), it.data_ptr(), gt.data_ptr(), 2, D, dx.data_ptr(), st) == 0
    dx = dx.cpu().numpy()
    assert np.isnan(dx[0]).all(), dx[0]
    assert dx[1, 3] == np.inf and (np.delete(dx[1], 3) == 0).all(), dx[1]


def test_row_offset_past_2_31_elements(torch):
    """rows * D > 2^31: D = 4096, 2^19 + 3 rows made on the device; the tail rows (and a few rescued ones) against fp64."""
    free = torch.cuda.mem_get_info()[0]
    if free < 40 * 2 ** 30:
        pytest.skip(f"needs 40 GB free on the device for a 26 GB peak, {free / 2 ** 30:.1f} GB free")
    R, D = 2 ** 19 + 3, 4096
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn(R, D, device="cuda", generator=g)
    x[-8:] *= torch.tensor([1.0, 2.0 ** 100, 2.0 ** -100, 2.0 ** 70, 2.0 ** -70, 0.5, 2.0 ** 120, 2.0 ** -130], device="cuda")[:, None]
    y, inv = capi.l2normalize_forward(x)
    tail = slice(R - 64, R)
    xt = x[tail].cpu().numpy()
    del x
    dy = torch.randn(R, D, device="cuda", generator=g)
    dx = capi.l2normalize_backward(y, inv, dy)
    torch.cuda.synchronize()
    yt, it, dyt, dxt = y[tail].cpu().numpy(), inv[tail].cpu().numpy(), dy[tail].cpu().numpy(), dx[tail].cpu().numpy()
    del y, dy, dx
    assert not ref.check_forward(xt, yt, it)[0]
    assert not ref.check_backward(yt, it, dyt, dxt)[0]


# ------------------------------------------------------------------------------------------- every path of the layer that runs it
RAND = dict(ap_region=capi.LOCAL, ap_method=capi.RAND, an_region=capi.LOCAL, an_method=capi.RAND)


def _layer_rows(N, D, seed):
    """Rows at norms 2^-140 .. 2^120 (a Gaussian row at 2^k) and spikes, no non-finite element."""
    rng = np.random.default_rng(seed)
    x = np.ldexp(rng.standard_normal((N, D)), rng.integers(-140, 120, (N, 1))).astype(F32)
    x[1] = 0; x[1, D // 2] = np.ldexp(F32(1.0), -149)
    x[2] = 0; x[2, 0] = np.ldexp(F32(1.5), 127)
    return x


def _labels(n):
    return (np.arange(n) // 2).astype(F32)


def _step(torch, path, x, lab, norm, **cfg):
    """(tops, S, dx) of one step on `path`; norm = 1: the layer normalises x itself, 0: x is the normalised rows."""
    N, D = x.shape
    xt, lt = torch.from_numpy(x).cuda(), torch.from_numpy(lab).cuda()
    if path.startswith("world"):
        W = int(path[5:])
        Q = N // W
        ctxs, S, tops = [], [], []
        rs = torch.empty((W, Q, 8), dtype=torch.float32, device="cuda")
        for r in range(W):
            c = capi.Context(capi.make_config(Q, D, world=W, rank=r, normalize_input=norm, **RAND, **cfg))
            tops.append(c.forward_gathered(xt, lt))
            c.row_scalars(rs[r])
            S.append(c.debug_read(0, Q * N))
            ctxs.append(c)
        g = []
        for r in range(W):
            gr = torch.full((Q, D), float("nan"), dtype=torch.float32, device="cuda")
            if W == 1:
                ctxs[r].backward(1.0, gr)
            else:
                ctxs[r].backward_gathered(1.0, rs, gr)
            torch.cuda.synchronize()
            g.append(gr.cpu().numpy())
            ctxs[r].close()
        return np.array(tops, F32), np.concatenate(S), np.concatenate(g)
    if path == "memory":
        m = N // 3
        Q = N - m
        mem = capi.l2normalize_forward(xt[Q:])[0] if norm else xt[Q:].contiguous()   # the memory holds normalised rows either way
        c = capi.Context(capi.make_config(Q, D, normalize_input=norm, **RAND, **cfg), memory_rows=m)
        tops = c.forward_memory(xt[:Q].contiguous(), lt[:Q].contiguous(), mem, lt[Q:].contiguous(), m)
        g = torch.full((Q, D), float("nan"), dtype=torch.float32, device="cuda")
        c.backward(0.7, g)
        torch.cuda.synchronize()
        S = c.debug_read(0, Q * N)
        c.close()
        return np.array(tops, F32), S, g.cpu().numpy()
    c = capi.Context(capi.make_config(N, D, normalize_input=norm, **RAND, **cfg))
    g = torch.full((N, D), float("nan"), dtype=torch.float32, device="cuda")
    if path == "async":
        tops_d = torch.zeros(5, device="cuda")
        lw = torch.tensor([0.7], dtype=torch.float32, device="cuda")
        graph = torch.cuda.CUDAGraph()
        c.forward_async(xt, lt, tops_d)                            # eager warm-up step, then the captured one replayed
        c.backward_device_weight(lw, g)
        torch.cuda.synchronize()
        with torch.cuda.graph(graph):
            c.forward_async(xt, lt, tops_d)
            c.backward_device_weight(lw, g)
        g.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        tops = tops_d.cpu().numpy()
    else:
        tops = np.array(c.forward(xt, lt), F32)
        c.backward(0.7, g)
    torch.cuda.synchronize()
    S = c.debug_read(0, N * N) if path != "blocks" else np.zeros(0, F32)
    c.close()
    return np.asarray(tops, F32), S, g.cpu().numpy()


def _layers_agree(torch, path, x, lab, **cfg):
    """Layer A (normalize_input = 1 on x) against layer B (normalize_input = 0 on the stand-alone y, then the stand-alone backward)."""
    tA, SA, gA = _step(torch, path, x, lab, 1, **cfg)
    xt = torch.from_numpy(x).cuda()
    y, inv = capi.l2normalize_forward(xt)
    tB, SB, gB = _step(torch, path, y.cpu().numpy(), lab, 0, **cfg)
    Q = gB.shape[0]
    dxB = capi.l2normalize_backward(y[:Q].contiguous(), inv[:Q].contiguous(), torch.from_numpy(gB).cuda()).cpu().numpy()
    assert np.array_equal(_bits(tA), _bits(tB)), f"{path}: tops {tA} vs {tB}"
    assert np.array_equal(_bits(SA), _bits(SB)), f"{path}: S"
    assert np.array_equal(_bits(gA), _bits(dxB)), f"{path}: dx"
    return tA, gA


@pytest.mark.parametrize("path", ["step", "world1", "world2", "world3", "memory", "async", "blocks"])
@pytest.mark.parametrize("D", [33, 128, 129, 512])
def test_layer_normalises_as_the_standalone_call(torch, path, D):
    N = 384 if path != "world3" else 408
    x = _layer_rows(N, D, D)
    cfg = {"sim_block_rows": 128} if path == "blocks" else {}
    _layers_agree(torch, path, x, _labels(N), **cfg)


@pytest.mark.parametrize("k", [-70, 70])
def test_layer_scale_invariance(torch, k):
    """x 2^k gives the tops of x and the gradient dx 2^-k, bit for bit (the rescue path and the fast path)."""
    x = synth.make_inputs(256, 129, 9)[0] * F32(3.0)
    lab = _labels(256)
    t0, S0, g0 = _step(torch, "step", x, lab, 1)
    t1, S1, g1 = _step(torch, "step", np.ldexp(x, k).astype(F32), lab, 1)
    assert np.array_equal(_bits(t0), _bits(t1)) and np.array_equal(_bits(S0), _bits(S1))
    want = np.ldexp(g0.astype(np.float64), -k)
    n = (np.abs(want) >= 2.0 ** -126) | (want == 0)
    assert np.array_equal(_bits(g1[n]), _bits(want[n].astype(F32)))


def test_layer_nan_feature_row(torch):
    """One NaN feature row at world 1: layers A and B agree bit for bit (NaNs compared as integers)."""
    x = synth.make_inputs(128, 64, 3)[0]
    x[5, 9] = np.nan
    lab = _labels(128)
    tA, SA, gA = _step(torch, "step", x, lab, 1)
    xt = torch.from_numpy(x).cuda()
    y, inv = capi.l2normalize_forward(xt)
    tB, SB, gB = _step(torch, "step", y.cpu().numpy(), lab, 0)
    dxB = capi.l2normalize_backward(y, inv, torch.from_numpy(gB).cuda()).cpu().numpy()
    assert np.array_equal(_bits(tA), _bits(tB)) and np.array_equal(_bits(SA), _bits(SB)) and np.array_equal(_bits(gA), _bits(dxB))


def test_torch_memory_ring_stores_the_rows_the_layer_used(torch):
    from npairloss_b200 import torch_api
    M, Q, D = 96, 64, 129
    loss = torch_api.NPairLoss(normalize_input=1, memory_rows=M, **RAND)
    for step in range(2):
        x = _layer_rows(Q, D, 50 + step)
        xt = torch.from_numpy(x).cuda().requires_grad_(True)
        loss(xt, torch.from_numpy(_labels(Q)).cuda())
        torch.cuda.synchronize()
    rows, _ = loss.memory()
    y0 = capi.l2normalize_forward(torch.from_numpy(_layer_rows(Q, D, 50)).cuda())[0]
    y1 = capi.l2normalize_forward(torch.from_numpy(_layer_rows(Q, D, 51)).cuda())[0]
    want = torch.cat([y1[32:], y0[32:], y1[:32]])          # slots 0..63 took batch 0; batch 1 filled 64..95 and wrapped to 0..31
    assert torch.equal(rows.view(torch.int32), want.view(torch.int32))


def test_class_embeddings_of_extreme_scale(torch):
    from npairloss_b200 import torch_api
    rng = np.random.default_rng(4)
    for k in (-130, -70, 0, 70, 120):
        x = np.ldexp(rng.standard_normal((60, 33)), k).astype(F32)
        lab = torch.from_numpy((np.arange(60) % 6).astype(F32)).cuda()
        cl, emb = torch_api.class_embeddings(torch.from_numpy(x).cuda(), lab, normalize=True)
        _, mean = torch_api.class_embeddings(torch.from_numpy(x).cuda(), lab, normalize=False)
        e = emb.cpu().numpy()
        v, _ = ref.check_forward(mean.cpu().numpy(), e, capi.l2normalize_forward(mean)[1].cpu().numpy())
        assert not v, f"k{k}: {v}"
        np.testing.assert_allclose(np.linalg.norm(e.astype(np.float64), axis=1), 1.0, rtol=1e-6)
