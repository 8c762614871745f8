"""Row-block similarity mode on the GPU: the context keeps one block of rows of S and recomputes it, so tops, gradient and every
per-row array must be bit for bit those of the materialised path; and a batch whose S would not fit in HBM trains."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROWS = (1, 2, 3, 4, 5, 6, 7, 8, 9)        # npair_debug_read selectors of the per-row arrays


def _bits(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float32)).view(np.uint32)


def _assert_bitwise(a, b, what):
    assert np.array_equal(_bits(a), _bits(b)), f"{what}: not bitwise equal (max abs diff {np.abs(np.asarray(a) - np.asarray(b)).max():.3e})"


def _step(x, lab, Q, world, prec=2, sim_block_rows=0, loss_weight=0.7, **cfg):
    """Every rank emulated on one GPU through the external-collectives calls (as tests/gpu_harness.gpu_step_world, without S)."""
    import torch
    from npairloss_b200 import capi
    N, D = x.shape
    dev = torch.device("cuda:0")
    xt, lt = torch.from_numpy(x).to(dev), torch.from_numpy(lab).to(dev)
    tops = np.zeros((world, 5), np.float32)
    rows = np.zeros((len(ROWS), N), np.float32)
    dx = torch.full((N, D), float("nan"), dtype=torch.float32, device=dev)
    ctxs = []
    try:
        for r in range(world):
            c = capi.Context(capi.make_config(Q, D, world=world, rank=r, sim_precision=prec, sim_block_rows=sim_block_rows, **cfg))
            ctxs.append(c)
            tops[r] = c.forward_gathered(xt, lt)
            for k, w in enumerate(ROWS):
                rows[k, r * Q:(r + 1) * Q] = c.debug_read(w, Q)
        if world > 1:
            assert ctxs[0].bwd_exchange_mode() == 2
            rs = torch.empty((world, Q, 8), dtype=torch.float32, device=dev)
            for r in range(world):
                ctxs[r].row_scalars(rs[r])
            for r in range(world):
                ctxs[r].backward_gathered(loss_weight, rs, dx[r * Q:(r + 1) * Q])
        else:
            ctxs[0].backward_partial(loss_weight, dx, None)
        torch.cuda.synchronize()
    finally:
        for c in ctxs:
            c.close()
    return tops, dx.cpu().numpy(), rows


def _compare(x, lab, Q, world, height, tag, **cfg):
    t0, g0, r0 = _step(x, lab, Q, world, **cfg)
    t1, g1, r1 = _step(x, lab, Q, world, sim_block_rows=height, **cfg)
    _assert_bitwise(t1, t0, f"{tag} tops")
    _assert_bitwise(g1, g0, f"{tag} gradient")
    for k, w in enumerate(ROWS):
        _assert_bitwise(r1[k], r0[k], f"{tag} debug_read({w})")
    assert np.isfinite(g1).all() and np.abs(g1).max() > 0, tag


def _inputs(N, D=128, seed=11, noise=2.5):
    from npairloss_b200 import synth
    return synth.make_inputs(N, D, seed, noise=noise)


@pytest.mark.parametrize("world", [1, 2, 3])
@pytest.mark.parametrize("height", [128, 384])
def test_blocks_match_materialised(world, height):
    """Q = 1000 is no multiple of the height: the last block is short."""
    from npairloss_b200 import synth
    Q = 1000
    x, lab = _inputs(Q * world, seed=world)
    _compare(x, lab, Q, world, height, f"w{world} h{height}", **synth.USAGE_MINING)


@pytest.mark.parametrize("prec", [0, 1, 2], ids=["bf16x3", "bf16", "fp16x2"])
@pytest.mark.parametrize("world", [1, 2])
def test_blocks_every_precision(prec, world):
    from npairloss_b200 import synth
    Q = 700
    x, lab = _inputs(Q * world, D=96, seed=20 + prec)
    _compare(x, lab, Q, world, 256, f"prec {prec} w{world}", prec=prec, **synth.USAGE_MINING)


def _minings():
    from npairloss_b200 import synth
    out = []
    for region in (synth.LOCAL, synth.GLOBAL):
        for method in (synth.HARD, synth.EASY, synth.RAND, synth.RELATIVE_HARD, synth.RELATIVE_EASY):
            rel = method in (synth.RELATIVE_HARD, synth.RELATIVE_EASY)
            sns = ([-0.3, -0.0] if region == synth.LOCAL else [-0.0]) if rel else [-1.0]
            for sn in sns:
                out.append(pytest.param(dict(ap_region=region, ap_method=method, an_region=region, an_method=method, identsn=sn, diffsn=sn,
                                             margin_ident=0.02, margin_diff=-0.05),
                                        id=f"{'LG'[region == synth.GLOBAL]}{method}_sn{sn}"))
    # mixed regions: the usage block's GLOBAL closed form with a LOCAL general-SN select
    out.append(pytest.param(dict(ap_region=synth.GLOBAL, ap_method=synth.RELATIVE_EASY, identsn=-0.0,
                                 an_region=synth.LOCAL, an_method=synth.RELATIVE_HARD, diffsn=-0.7, margin_diff=-0.05), id="mixed"))
    return out


@pytest.mark.parametrize("mining", _minings())
def test_blocks_every_accepted_mining(mining):
    Q = 900
    x, lab = _inputs(Q, seed=5)
    _compare(x, lab, Q, 1, 256, f"{mining}", **mining)


@pytest.mark.parametrize("Q,D,height,chunk", [(999, 101, 256, 0), (999, 101, 384, 0), (1001, 130, 256, 64)])
def test_blocks_ragged_shapes(Q, D, height, chunk):
    """Q*D % 4 != 0 and a short last block (231 or 233 rows): every block's split-K reduce sums slices that are not 16-byte
    aligned, and D = 101 takes the gradient drain's scalar stores.  grad_chunk_cols = 64 puts the chunk key's m_blk0 term (the
    block's first 128-row tile) into the first chunk of every tile."""
    from npairloss_b200 import synth
    x, lab = _inputs(Q, D=D, seed=Q + D)
    lab[-1] = lab[-2]                   # an odd batch's last image joins the class before it: every row has a positive
    _compare(x, lab, Q, 1, height, f"Q{Q} D{D} h{height} chunk{chunk}", grad_chunk_cols=chunk, **synth.USAGE_MINING)


def test_blocks_every_accepted_mining_world2():
    from npairloss_b200 import synth
    Q = 600
    x, lab = _inputs(2 * Q, seed=6)
    for m in (dict(synth.USAGE_MINING, an_method=synth.RELATIVE_EASY, diffsn=-0.4), dict(synth.DEFAULT_MINING, ap_method=synth.HARD)):
        _compare(x, lab, Q, 2, 128, f"w2 {m}", **m)


def test_blocks_normalize_input():
    from npairloss_b200 import synth
    Q = 800
    x, lab = _inputs(Q, seed=9)
    x = x * np.linspace(0.5, 3.0, Q, dtype=np.float32)[:, None]       # raw embeddings of varied norm
    _compare(np.ascontiguousarray(x), lab, Q, 1, 256, "normalize_input", normalize_input=1, **synth.USAGE_MINING)


def test_blocks_forward_backward_and_torch_module():
    import torch
    from npairloss_b200 import capi, synth, torch_api
    Q, D = 1100, 128
    x, lab = _inputs(Q, D, seed=13)
    dx, dl = torch.from_numpy(x).cuda(), torch.from_numpy(lab).cuda()
    outs = []
    for h in (0, 256):
        c = capi.Context(capi.make_config(Q, D, sim_block_rows=h, **synth.USAGE_MINING))
        g = torch.empty_like(dx)
        t = c.forward_backward(dx, dl, 0.5, g)
        torch.cuda.synchronize()
        t2 = c.forward(dx, dl)                 # the separate calls agree with the fused one
        g2 = torch.empty_like(dx)
        c.backward(0.5, g2)
        torch.cuda.synchronize()
        if h:
            with pytest.raises(capi.NpairError) as e:
                c.debug_read(0, Q * Q)
            assert e.value.code == -6
        c.close()
        _assert_bitwise(t2, t, f"h{h} forward vs forward_backward")
        _assert_bitwise(g2.cpu().numpy(), g.cpu().numpy(), f"h{h} backward vs forward_backward")
        outs.append((t, g.cpu().numpy()))
    _assert_bitwise(outs[1][0], outs[0][0], "forward_backward tops")
    _assert_bitwise(outs[1][1], outs[0][1], "forward_backward gradient")
    grads = []
    for kw in (dict(), dict(sim_block_rows=256)):
        m = torch_api.NPairLoss(**synth.USAGE_MINING, **kw)
        xr = dx.clone().requires_grad_(True)
        loss, tops = m(xr, dl)
        loss.backward()
        grads.append((tops.cpu().numpy(), xr.grad.cpu().numpy()))
    _assert_bitwise(grads[1][0], grads[0][0], "NPairLoss tops")
    _assert_bitwise(grads[1][1], grads[0][1], "NPairLoss gradient")


def _fp64_reference(xt, lt, chunk=1024):
    """RAND/RAND at world 1 in fp64 on the GPU, S recomputed in row chunks: every non-self pair is selected, so
    A_i = sum_same exp(S_ij - max_i), T_i = sum_all exp(S_ij - max_i), loss = -mean log(A/T), G_ij = exp(S_ij - max_i) (1/T_i - [same] / A_i),
    dX = (G + G^T) X / (2 Q); top-1 = share of rows whose best positive is not tied or beaten by any other column."""
    import torch
    B = xt.shape[0]
    X = xt.double()
    mx = torch.empty(B, dtype=torch.float64, device=X.device)
    A, T = torch.empty_like(mx), torch.empty_like(mx)
    hit = torch.empty(B, dtype=torch.bool, device=X.device)
    for j0 in range(0, B, chunk):
        j1 = min(B, j0 + chunk)
        S = X[j0:j1] @ X.T
        idx = torch.arange(j0, j1, device=X.device)
        S[idx - j0, idx] = -torch.inf
        same = lt[j0:j1, None] == lt[None, :]
        m = S.max(dim=1).values
        E = torch.exp(S - m[:, None])
        mx[j0:j1], T[j0:j1], A[j0:j1] = m, E.sum(dim=1), torch.where(same, E, 0.0).sum(dim=1)
        best = torch.where(same, S, -torch.inf).max(dim=1).values
        hit[j0:j1] = (S >= best[:, None]).sum(dim=1) <= 1
        del S, E, same
    loss = -torch.log(A / T).mean().item()
    dX = torch.zeros_like(X)
    for j0 in range(0, B, chunk):
        j1 = min(B, j0 + chunk)
        S = X[j0:j1] @ X.T
        idx = torch.arange(j0, j1, device=X.device)
        same = lt[j0:j1, None] == lt[None, :]
        G = torch.exp(S - mx[j0:j1, None]) * (1.0 / T[j0:j1, None] - torch.where(same, 1.0 / A[j0:j1, None], 0.0))
        G[idx - j0, idx] = 0.0
        dX[j0:j1] += G @ X
        dX += G.T @ X[j0:j1]
        del S, G, same
    dX /= 2.0 * B
    return loss, hit.double().mean().item(), dX


def test_batch_beyond_materialised_s():
    """B = 196608, D = 256 on one GPU: the materialised S alone would take 155 GB."""
    import torch
    import ctypes as C
    from npairloss_b200 import capi, synth
    B, D = 196608, 256
    assert 4 * B * B > 150e9
    mining = dict(synth.DEFAULT_MINING)
    x, lab = synth.make_inputs(B, D, 20171230, noise=1.0)
    cfg = capi.make_config(B, D, sim_block_rows=2048, **mining)
    ws = capi.lib().npair_workspace_bytes(C.byref(cfg))
    assert 0 < ws < 8e9, ws
    capi.Context(capi.make_config(1024, D, sim_block_rows=256)).close()    # loads the module and caches the symmetry check
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    ctx = capi.Context(cfg)
    torch.cuda.synchronize()
    used = free0 - torch.cuda.mem_get_info()[0]
    assert ws <= used <= ws + (256 << 20), (ws, used)
    xt, lt = torch.from_numpy(x).cuda(), torch.from_numpy(lab).cuda()
    del x
    g = torch.empty_like(xt)
    tops = ctx.forward(xt, lt)
    ctx.backward(1.0, g)
    torch.cuda.synchronize()
    ctx.close()
    ctx2 = capi.Context(capi.make_config(B, D, sim_block_rows=1536, **mining))
    g2 = torch.empty_like(xt)
    tops2 = ctx2.forward(xt, lt)
    ctx2.backward(1.0, g2)
    torch.cuda.synchronize()
    ctx2.close()
    _assert_bitwise(tops2, tops, "tops, heights 2048 vs 1536")
    assert torch.equal(g.view(torch.int32), g2.view(torch.int32)), "gradient, heights 2048 vs 1536"
    del g2
    loss_ref, top1_ref, dX = _fp64_reference(xt, lt)
    assert abs(tops[0] - loss_ref) <= 1e-5 * abs(loss_ref), (tops[0], loss_ref)
    assert abs(tops[1] - top1_ref) * B <= B / 1000, (tops[1], top1_ref)
    err = (g.double() - dX).norm().item() / dX.norm().item()
    print(f"B={B}: loss {tops[0]:.7f} (fp64 {loss_ref:.7f}), top1 {tops[1]:.5f} (fp64 {top1_ref:.5f}), gradient normwise error {err:.3e}")
    assert err <= 1e-5, err
