"""The cross-batch memory ring kept by the context (DESIGN 4.3.1) on the GPU: npair_forward_ring against npair_forward_memory over a
Python ring laid out as NPairLoss's own, bit for bit, step after step; the ring tiles each step re-splits, through pre-scale changes;
checkpoints (read / load), the reset and the refusals; the asynchronous forward, capture once the ring is full and replays; and
NPairLoss(library_memory=True) against the module's own ring, eager and in a captured training step."""
import ctypes as C

import numpy as np
import pytest

from npairloss_b200 import capi, synth, torch_api

pytestmark = pytest.mark.gpu

FP16X2, BF16X3, BF16 = capi.PREC_FP32_FP16X2, capi.PREC_FP32_BF16X3, capi.PREC_BF16
E_ARG, E_STATE = -1, -6
USAGE = dict(synth.USAGE_MINING)
RAND = dict(synth.DEFAULT_MINING)
LOCAL_SN = dict(ap_region=capi.LOCAL, ap_method=capi.RELATIVE_HARD, an_region=capi.LOCAL, an_method=capi.RELATIVE_HARD, identsn=-0.4,
                diffsn=-0.3, margin_diff=-0.02)
DEBUG = [1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12]
TILE = 32


@pytest.fixture(scope="module")
def torch():
    import torch
    assert torch.cuda.is_available() and torch.cuda.get_device_capability(0) == (9, 0), "GPU tests need an H100"
    return torch


def _bits(a):
    a = a.detach().cpu().numpy() if hasattr(a, "detach") else np.asarray(a, dtype=np.float32)
    return np.ascontiguousarray(a).view(np.uint32)


def _batch(torch, Q, D, seed, scale=1.0):
    x, lab = synth.make_inputs(Q, D, seed=seed, imgs_per_class=2, noise=0.7)
    return torch.from_numpy(x * np.float32(scale)).cuda(), torch.from_numpy(lab).cuda()


class PyRing:
    """NPairLoss._forward_memory's ring: head = count mod M, a batch larger than M leaves its last M rows."""

    def __init__(self, torch, M, D):
        self.M, self.count = M, 0
        self.x = torch.zeros(max(M, 1), D, dtype=torch.float32, device="cuda")
        self.l = torch.zeros(max(M, 1), dtype=torch.float32, device="cuda")

    @property
    def m(self):
        return min(self.count, self.M)

    def push(self, rows, lab):
        """The slots written, in order."""
        q, M = rows.shape[0], self.M
        if M == 0:
            self.count += q
            return []
        slots = [(self.count + r) % M for r in range(max(0, q - M), q)]
        if q > M:
            rows, lab, self.count, q = rows[q - M:], lab[q - M:], self.count + q - M, M
        head = self.count % M
        first = min(q, M - head)
        self.x[head:head + first] = rows[:first]
        self.l[head:head + first] = lab[:first]
        if first < q:
            self.x[:q - first] = rows[first:]
            self.l[:q - first] = lab[first:]
        self.count += q
        return slots


class TileModel:
    """The ring tiles a step re-splits (npair_debug_read 13): all of [bt, nt) when the pre-scale differs from the one the pieces were
    split at (or none were), else the tiles of the slots pushed since, and the tile of row Q + m - 1 when m changed."""

    def __init__(self, Q):
        self.Q, self.valid, self.scale, self.m, self.dirty = Q, False, None, 0, set()

    def step(self, m, scale):
        Q = self.Q
        bt, nt = -(-Q // TILE), -(-(Q + m) // TILE)
        full = not self.valid or scale != self.scale
        bnd = (Q + m - 1) // TILE if m != self.m else -1
        out = [t for t in range(bt, nt) if full or t in self.dirty or t == bnd]
        self.dirty = {t for t in self.dirty if t >= nt}
        self.valid, self.scale, self.m = True, scale, m
        return out, full

    def push(self, slots):
        self.dirty |= {(self.Q + s) // TILE for s in slots}

    def load(self):
        self.valid, self.m, self.dirty = False, 0, set()


def _cfg(Q, D, prec, mining, **extra):
    return capi.make_config(Q, D, sim_precision=prec, **mining, **extra)


def _outputs(torch, ctx, Q, m, tops, weights=None, rl=None):
    dx = torch.full((Q, ctx.cfg.D), float("nan"), device="cuda")
    ctx.backward(1.0, dx)
    rec = torch.empty(8 * Q, device="cuda")
    ctx.row_scalars(rec)
    torch.cuda.synchronize()
    out = dict(tops=_bits(np.asarray(tops, dtype=np.float32)), dx=_bits(dx), rec=_bits(rec),
               S=ctx.debug_read(0, Q * (Q + m)).view(np.uint32))
    for w in DEBUG:
        out[f"dbg{w}"] = ctx.debug_read(w, 3 * Q if w == 12 else (1 if w == 10 else Q)).view(np.uint32)
    if rl is not None:
        out["row_loss"] = _bits(rl)
    return out


def _same(a, b, tag):
    assert a.keys() == b.keys(), tag
    for k in a:
        np.testing.assert_array_equal(a[k], b[k], err_msg=f"{tag}: {k}")


def _step_pair(torch, ring, ref, pyr, x, l, weights=None, asyn=False):
    """One step of the ring context and of the memory context over pyr: both outputs, then pyr takes the batch's rows."""
    Q, m = x.shape[0], pyr.m
    outs = []
    for ctx in (ref, ring):
        rl = torch.full((Q,), float("nan"), device="cuda") if weights is not None else None
        if weights is not None:
            ctx.set_anchor_io(weights, rl)
        if ctx is ref:
            tops = ctx.forward_memory(x, l, pyr.x, pyr.l, m)
        elif asyn:
            t = torch.full((5,), float("nan"), device="cuda")
            ctx.forward_ring_async(x, l, t)
            tops = t.cpu().numpy()
        else:
            tops = ctx.forward_ring(x, l)
        if weights is not None:
            ctx.set_anchor_io(None, None)
        outs.append(_outputs(torch, ctx, Q, m, tops, weights, rl))
    rows = capi.l2normalize_forward(x)[0] if ref.cfg.normalize_input else x
    slots = pyr.push(rows, l)
    return outs[0], outs[1], slots


def _check_ring(torch, ring, pyr, tag):
    M, D = ring.memory_rows, ring.cfg.D
    rows, labs = torch.full((max(M, 1), D), float("nan"), device="cuda"), torch.full((max(M, 1),), float("nan"), device="cuda")
    count = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    ring.ring_read(rows, labs, count)
    torch.cuda.synchronize()
    assert int(count.item()) == pyr.count, tag
    np.testing.assert_array_equal(_bits(rows[:pyr.m]), _bits(pyr.x[:pyr.m]), err_msg=f"{tag}: ring rows")
    np.testing.assert_array_equal(_bits(labs[:pyr.m]), _bits(pyr.l[:pyr.m]), err_msg=f"{tag}: ring labels")


def _tiles(ring):
    t = ring.debug_read(13, 1 + 4096)
    return [int(v) for v in t[1:1 + int(t[0])]]


# ------------------------------------------------------------------------------------------------ 1. bitwise over a run of steps
CASES = [
    # prec, Q, M, D, mining, extra config, anchor weights, asynchronous ring forward
    (FP16X2, 200, 700, 101, USAGE, {}, False, False),
    (BF16X3, 200, 700, 101, USAGE, {}, False, False),
    (BF16, 200, 700, 101, USAGE, {}, False, False),
    (FP16X2, 256, 100, 64, RAND, {}, False, False),                        # Q > M
    (BF16X3, 96, 333, 128, LOCAL_SN, dict(normalize_input=1), False, True),
    (FP16X2, 120, 500, 72, USAGE, dict(flags=capi.FLAG_NO_FUSED_GRAD), False, False),
    (BF16, 200, 700, 101, RAND, dict(normalize_input=1), True, False),     # anchor weights and row losses
    (FP16X2, 64, 256, 64, LOCAL_SN, {}, True, True),                       # Q | M, whole tiles
]


@pytest.mark.parametrize("prec,Q,M,D,mining,extra,weighted,asyn", CASES)
def test_ring_matches_memory_forward_over_a_run(torch, prec, Q, M, D, mining, extra, weighted, asyn):
    steps = 2 * -(-M // Q) + 3
    ring = capi.Context(_cfg(Q, D, prec, mining, **extra), memory_rows=M, ring=True)
    ref = capi.Context(_cfg(Q, D, prec, mining, **extra), memory_rows=M)
    pyr, model = PyRing(torch, M, D), TileModel(Q)
    try:
        for s in range(steps):
            x, l = _batch(torch, Q, D, 1000 * s + Q + M)
            w = torch.rand(Q, generator=torch.Generator().manual_seed(s)).cuda() if weighted else None
            if w is not None:
                w[::7] = 0.0
            m = pyr.m
            a, b, slots = _step_pair(torch, ring, ref, pyr, x, l, w, asyn)
            tag = f"step {s} (m = {m})"
            _same(a, b, tag)
            expect, _ = model.step(m, a["dbg10"][0])
            assert _tiles(ring) == expect, tag
            model.push(slots)
            _check_ring(torch, ring, pyr, tag)
    finally:
        ring.close(); ref.close()


# ------------------------------------------------------------------------------------------------ 2. pre-scale changes
def test_prescale_changes_resplit_every_tile(torch):
    """Un-normalised fp16x2 batches whose max |x| crosses powers of two up and back down (the ring's rows carry theirs until pushed
    out): outputs stay bit for bit, every ring tile is re-split on the steps whose pre-scale changed and only the pushed tiles and the
    boundary tile on the others."""
    Q, M, D = 100, 450, 96
    scales = [1, 1, 5, 1, 1, 1, 1, 1, 0.1, 0.1, 0.1, 0.1, 0.1, 0.1, 1, 9, 1, 1, 1, 1, 1, 1]
    ring = capi.Context(_cfg(Q, D, FP16X2, USAGE), memory_rows=M, ring=True)
    ref = capi.Context(_cfg(Q, D, FP16X2, USAGE), memory_rows=M)
    pyr, model = PyRing(torch, M, D), TileModel(Q)
    changed = partial = 0
    try:
        for s, f in enumerate(scales):
            x, l = _batch(torch, Q, D, 77 + s, scale=f)
            m = pyr.m
            a, b, slots = _step_pair(torch, ring, ref, pyr, x, l)
            _same(a, b, f"step {s}")
            expect, full = model.step(m, a["dbg10"][0])
            got = _tiles(ring)
            assert got == expect, f"step {s}"
            nt, bt = -(-(Q + m) // TILE), -(-Q // TILE)
            if full and s > 0:
                changed += 1
                assert got == list(range(bt, nt)), f"step {s}"
            elif s > 0 and m == M:
                partial += 1
                assert len(got) < nt - bt, f"step {s}: a step whose pre-scale held re-split every tile"
            model.push(slots)
        assert changed >= 3 and partial >= 3, (changed, partial)
    finally:
        ring.close(); ref.close()


# ------------------------------------------------------------------------------------------------ 3. checkpoints and refusals
def test_checkpoint_load_continues_bit_for_bit(torch):
    Q, M, D = 200, 700, 101
    cfg = _cfg(Q, D, FP16X2, USAGE, normalize_input=1)
    a, b, ref = (capi.Context(cfg, memory_rows=M, ring=True), capi.Context(cfg, memory_rows=M, ring=True),
                 capi.Context(cfg, memory_rows=M))
    pyr = PyRing(torch, M, D)
    try:
        for s in range(10):
            x, l = _batch(torch, Q, D, 500 + s)
            if s == 5:                                 # the checkpoint: a's ring into the fresh context b
                rows, labs = torch.empty(M, D, device="cuda"), torch.empty(M, device="cuda")
                count = torch.zeros(1, dtype=torch.int64, device="cuda")
                a.ring_read(rows, labs, count)
                b.ring_load(rows, labs, int(count.item()))
            o_ref, o_a, slots = _step_pair(torch, a, ref, pyr, x, l)
            _same(o_ref, o_a, f"step {s}")
            if s >= 5:
                o_b = _outputs(torch, b, Q, min(pyr.count - Q, M), b.forward_ring(x, l))
                _same(o_a, o_b, f"continued step {s}")
        _check_ring(torch, b, pyr, "continued ring")
    finally:
        a.close(); b.close(); ref.close()


@pytest.mark.parametrize("count", [0, 1, 333, 699, 700, 1234, 5000])
def test_load_any_count_then_step(torch, count):
    """A load with count < M, = M and > M, and the reset (0): the next steps equal the memory forward over the Python ring loaded the
    same way."""
    Q, M, D = 200, 700, 101
    cfg = _cfg(Q, D, BF16X3, USAGE)
    ring, ref = capi.Context(cfg, memory_rows=M, ring=True), capi.Context(cfg, memory_rows=M)
    pyr = PyRing(torch, M, D)
    try:
        for s in range(3):                             # something to overwrite
            x, l = _batch(torch, Q, D, 900 + s)
            _step_pair(torch, ring, ref, pyr, x, l)
        g = torch.Generator().manual_seed(count)
        m = min(count, M)
        rows = torch.randn(max(m, 1), D, generator=g).cuda()
        rows = rows / rows.norm(dim=1, keepdim=True)
        labs = torch.randint(0, Q // 2, (max(m, 1),), generator=g).float().cuda()
        if count == 0:
            ring.ring_load(None, None, 0)
        else:
            ring.ring_load(rows, labs, count)
        pyr.count = count
        pyr.x[:m] = rows[:m]
        pyr.l[:m] = labs[:m]
        _check_ring(torch, ring, pyr, "loaded")
        model = TileModel(Q)
        model.load()
        for s in range(4):
            x, l = _batch(torch, Q, D, 950 + s)
            mm = pyr.m
            o_ref, o_ring, slots = _step_pair(torch, ring, ref, pyr, x, l)
            _same(o_ref, o_ring, f"step {s} after load({count})")
            expect, _ = model.step(mm, o_ref["dbg10"][0])
            assert _tiles(ring) == expect
            model.push(slots)
        _check_ring(torch, ring, pyr, "after the steps")
    finally:
        ring.close(); ref.close()


def test_refusals(torch):
    L = capi.lib()
    Q, M, D = 64, 100, 32
    cfg = _cfg(Q, D, FP16X2, USAGE)
    ring, plain, mem = capi.Context(cfg, memory_rows=M, ring=True), capi.Context(cfg), capi.Context(cfg, memory_rows=M)
    x, l = _batch(torch, Q, D, 3)
    tops = torch.zeros(5, device="cuda")
    dx = torch.zeros(Q, D, device="cuda")
    host = (C.c_float * 5)()
    try:
        ring.forward_ring(x, l)                        # one row set in the ring
        torch.cuda.synchronize()
        n0 = capi.kernel_launches()
        st = torch.cuda.current_stream().cuda_stream
        h = ring._h
        for rc in (L.npair_forward(h, x.data_ptr(), l.data_ptr(), host, st),
                   L.npair_forward_async(h, x.data_ptr(), l.data_ptr(), tops.data_ptr(), st),
                   L.npair_forward_memory(h, x.data_ptr(), l.data_ptr(), x.data_ptr(), l.data_ptr(), 4, host, st),
                   L.npair_forward_memory_async(h, x.data_ptr(), l.data_ptr(), x.data_ptr(), l.data_ptr(), 0, tops.data_ptr(), st),
                   L.npair_forward_backward(h, x.data_ptr(), l.data_ptr(), C.c_float(1.0), dx.data_ptr(), host, st)):
            assert rc == E_STATE
            assert b"npair_forward_ring" in L.npair_last_error(h)
        for ctx in (plain, mem):
            assert L.npair_forward_ring(ctx._h, x.data_ptr(), l.data_ptr(), host, st) == E_STATE
            assert L.npair_forward_ring_async(ctx._h, x.data_ptr(), l.data_ptr(), tops.data_ptr(), st) == E_STATE
            assert L.npair_memory_ring_read(ctx._h, x.data_ptr(), l.data_ptr(), tops.data_ptr(), st) == E_STATE
            assert L.npair_memory_ring_load(ctx._h, x.data_ptr(), l.data_ptr(), 3, st) == E_STATE
        assert L.npair_memory_ring_load(h, x.data_ptr(), l.data_ptr(), -1, st) == E_ARG
        assert L.npair_memory_ring_load(h, None, l.data_ptr(), 5, st) == E_ARG
        assert L.npair_memory_ring_load(h, x.data_ptr(), None, 5, st) == E_ARG
        assert L.npair_memory_ring_read(h, None, l.data_ptr(), tops.data_ptr(), st) == E_ARG
        assert L.npair_memory_ring_read(h, x.data_ptr(), l.data_ptr(), None, st) == E_ARG
        assert L.npair_forward_ring(h, None, l.data_ptr(), host, st) == E_ARG
        assert L.npair_forward_ring_async(h, x.data_ptr(), l.data_ptr(), None, st) == E_ARG
        assert capi.kernel_launches() == n0
        # what npair_create_memory refuses, npair_create_memory_ring refuses, and its workspace is 0
        for bad, m in ((dict(world=2, rank=0), M), (dict(gemm_backend=capi.GEMM_SIMT_CHECK), M), (dict(global_scope=1), M),
                       (dict(sim_block_rows=128, Q=512), M), ({}, -1)):
            q = bad.pop("Q", Q)
            c = capi.make_config(q, D, **bad)
            out = C.c_void_p()
            assert L.npair_create_memory_ring(C.byref(c), m, C.byref(out)) == E_ARG, bad
            assert L.npair_memory_ring_workspace_bytes(C.byref(c), m) == 0, bad
            assert L.npair_create_memory(C.byref(c), m, C.byref(out)) == E_ARG, bad
        # the ring still holds the one batch
        rows, labs = torch.empty(M, D, device="cuda"), torch.empty(M, device="cuda")
        count = torch.zeros(1, dtype=torch.int64, device="cuda")
        ring.ring_read(rows, labs, count)
        torch.cuda.synchronize()
        assert int(count.item()) == Q
        np.testing.assert_array_equal(_bits(rows[:Q]), _bits(x))
    finally:
        ring.close(); plain.close(); mem.close()


def test_workspace_is_what_the_context_allocates(torch):
    Q, M, D = 300, 5000, 256
    cfg = _cfg(Q, D, FP16X2, USAGE)
    want = capi.memory_workspace_bytes(cfg, M, ring=True)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    ring = capi.Context(cfg, memory_rows=M, ring=True)
    torch.cuda.synchronize()
    used = free0 - torch.cuda.mem_get_info()[0]
    ring.close()
    # every buffer is a cudaMalloc of its own: the driver rounds each up to its pages, and sub-allocates small ones
    assert want - (8 << 20) <= used <= want + 40 * (2 << 20), (want, used)
    assert want - capi.memory_workspace_bytes(cfg, M) == 4 * M * D + 8 * M + 8 * -(-(Q + M) // TILE) + 32


# ------------------------------------------------------------------------------------------------ 4. asynchronous forward and capture
def test_capture_once_full_and_replays(torch):
    Q, M, D = 128, 300, 64
    cfg = _cfg(Q, D, FP16X2, USAGE)
    cap, eager = capi.Context(cfg, memory_rows=M, ring=True), capi.Context(cfg, memory_rows=M, ring=True)
    sx, sl = _batch(torch, Q, D, 1)
    tops = torch.zeros(5, device="cuda")
    lw = torch.ones(1, device="cuda")
    dx = torch.zeros(Q, D, device="cuda")

    def ring_state(ctx):
        rows, labs = torch.empty(M, D, device="cuda"), torch.empty(M, device="cuda")
        count = torch.zeros(1, dtype=torch.int64, device="cuda")
        ctx.ring_read(rows, labs, count)
        torch.cuda.synchronize()
        return _bits(rows), _bits(labs), int(count.item())

    def eager_step(ctx, x, l):
        t = ctx.forward_ring(x, l)
        d = torch.zeros(Q, D, device="cuda")
        ctx.backward(1.0, d)
        torch.cuda.synchronize()
        return _bits(np.asarray(t, dtype=np.float32)), _bits(d)

    try:
        b = 0
        while True:
            x, l = _batch(torch, Q, D, 100 + b)
            full = b * Q >= M
            if not full:                               # capture before the ring is full: refused, nothing enqueued
                before = ring_state(cap)
                n0 = capi.kernel_launches()
                g = torch.cuda.CUDAGraph()
                with pytest.raises(capi.NpairError) as e:
                    with torch.cuda.graph(g):
                        cap.forward_ring_async(sx, sl, tops)
                assert e.value.code == E_STATE and f"{M - b * Q} more" in str(e.value)
                assert capi.kernel_launches() == n0
                after = ring_state(cap)
                assert all(np.array_equal(u, v) for u, v in zip(before[:2], after[:2])) and before[2] == after[2]
            else:
                break
            sx.copy_(x); sl.copy_(l)                   # eager asynchronous steps against the synchronous ones
            cap.forward_ring_async(sx, sl, tops)
            cap.backward_device_weight(lw, dx)
            torch.cuda.synchronize()
            ta, da = _bits(tops), _bits(dx)
            te, de = eager_step(eager, x, l)
            np.testing.assert_array_equal(ta, te, err_msg=f"async tops {b}")
            np.testing.assert_array_equal(da, de, err_msg=f"async gradient {b}")
            b += 1
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            cap.forward_ring_async(sx, sl, tops)
            cap.backward_device_weight(lw, dx)
        for k in range(6):                             # replays over new batches, more than M rows: the ring wraps on the device
            x, l = _batch(torch, Q, D, 200 + k)
            sx.copy_(x); sl.copy_(l)
            g.replay()
            torch.cuda.synchronize()
            te, de = eager_step(eager, x, l)
            np.testing.assert_array_equal(_bits(tops), te, err_msg=f"replay {k} tops")
            np.testing.assert_array_equal(_bits(dx), de, err_msg=f"replay {k} gradient")
        cap.async_status()
        for k in range(2):                             # eager steps continue from the device count
            x, l = _batch(torch, Q, D, 300 + k)
            (tc, dc), (te, de) = eager_step(cap, x, l), eager_step(eager, x, l)
            np.testing.assert_array_equal(tc, te, err_msg=f"eager tops {k} after the replays")
            np.testing.assert_array_equal(dc, de, err_msg=f"eager gradient {k} after the replays")
        rc, re_ = ring_state(cap), ring_state(eager)
        assert rc[2] == re_[2] == (b + 8) * Q
        assert np.array_equal(rc[0], re_[0]) and np.array_equal(rc[1], re_[1])
        # a load that leaves the ring not full, then a replay: NaN tops, the error for async_status, the ring untouched
        rows, labs = torch.randn(M, D, device="cuda"), torch.zeros(M, device="cuda")
        cap.ring_load(rows, labs, M - 5)
        before = ring_state(cap)
        g.replay()
        torch.cuda.synchronize()
        assert np.isnan(tops.cpu().numpy()).all()
        with pytest.raises(capi.NpairError) as e:
            cap.async_status()
        assert e.value.code == E_STATE and "not full" in str(e.value)
        after = ring_state(cap)
        assert after[2] == M - 5 and np.array_equal(before[0], after[0]) and np.array_equal(before[1], after[1])
        cap.async_status()                             # the bit was cleared
        del g
    finally:
        cap.close(); eager.close()


# ------------------------------------------------------------------------------------------------ 5. NPairLoss(library_memory=True)
def test_module_library_memory_matches_module_ring(torch):
    """Over batch-size changes (the context is re-created and the ring carried over), with normalize_input."""
    M, D = 300, 64
    lib_fn = torch_api.NPairLoss(memory_rows=M, library_memory=True, normalize_input=1, **USAGE)
    ref_fn = torch_api.NPairLoss(memory_rows=M, normalize_input=1, **USAGE)
    for s, Q in enumerate([128, 128, 96, 96, 96, 128, 400, 128, 128]):
        x, l = _batch(torch, Q, D, 40 + s)
        xa, xb = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
        la, ta = lib_fn(xa, l)
        lb, tb = ref_fn(xb, l)
        la.backward(); lb.backward()
        np.testing.assert_array_equal(_bits(ta), _bits(tb), err_msg=f"tops of step {s}")
        np.testing.assert_array_equal(_bits(xa.grad), _bits(xb.grad), err_msg=f"gradient of step {s}")
        ma, mb = lib_fn.memory(), ref_fn.memory()
        np.testing.assert_array_equal(_bits(ma[0]), _bits(mb[0]), err_msg=f"memory rows after step {s}")
        np.testing.assert_array_equal(_bits(ma[1]), _bits(mb[1]), err_msg=f"memory labels after step {s}")
    lib_fn.reset_memory(); ref_fn.reset_memory()
    assert lib_fn.memory()[0].shape[0] == 0
    x, l = _batch(torch, 128, D, 99)
    np.testing.assert_array_equal(_bits(lib_fn(x, l)[1]), _bits(ref_fn(x, l)[1]), err_msg="after the reset")


def _trunk(torch, D_in, D):
    torch.manual_seed(1234)
    return torch.nn.Sequential(torch.nn.Linear(D_in, 256), torch.nn.ReLU(), torch.nn.Linear(256, D)).cuda()


def test_module_capture_before_full_raises(torch):
    Q, D, M = 128, 64, 300
    loss_fn = torch_api.NPairLoss(memory_rows=M, library_memory=True, blocking=False, **USAGE)
    x, l = _batch(torch, Q, D, 5)
    loss_fn(x, l)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match="2 more eager step"):
        with torch.cuda.graph(g):
            loss_fn(x, l)


def test_whole_torch_step_captured_with_library_memory(torch):
    """Linear trunk -> NPairLoss(memory_rows=M, library_memory=True, blocking=False) -> backward -> SGD captured with torch.cuda.graph
    once the ring is full, replayed over new batches: the parameters equal, bit for bit, eager steps of the module's own ring."""
    Q, D_in, D, M = 256, 64, 512, 600
    warm = -(-M // Q)
    data = []
    for b in range(warm + 5):
        x, lab = synth.make_inputs(Q, D_in, seed=60 + b, imgs_per_class=2, noise=0.5)
        data.append((torch.from_numpy(x).cuda(), torch.from_numpy(lab).cuda()))
    net, net_ref = _trunk(torch, D_in, D), _trunk(torch, D_in, D)
    loss_fn = torch_api.NPairLoss(memory_rows=M, library_memory=True, blocking=False, normalize_input=1, **USAGE)
    loss_ref = torch_api.NPairLoss(memory_rows=M, normalize_input=1, **USAGE)
    opt, opt_ref = torch.optim.SGD(net.parameters(), lr=0.5), torch.optim.SGD(net_ref.parameters(), lr=0.5)

    def step(n, f, o, x, l):
        o.zero_grad(set_to_none=True)
        loss, _ = f(n(x), l)
        loss.backward()
        o.step()
        return loss

    sx, sl = data[0][0].clone(), data[0][1].clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):                            # eager steps until the ring is full
        for b in range(warm):
            sx.copy_(data[b][0]); sl.copy_(data[b][1])
            step(net, loss_fn, opt, sx, sl)
    torch.cuda.current_stream().wait_stream(side)
    for b in range(warm):
        step(net_ref, loss_ref, opt_ref, *data[b])
    g = torch.cuda.CUDAGraph()
    opt.zero_grad(set_to_none=True)
    with torch.cuda.graph(g):
        sloss, _ = loss_fn(net(sx), sl)
        sloss.backward()
        opt.step()
    for b in range(warm, warm + 5):
        sx.copy_(data[b][0]); sl.copy_(data[b][1])
        g.replay()
        lr = step(net_ref, loss_ref, opt_ref, *data[b])
        torch.cuda.synchronize()
        np.testing.assert_array_equal(_bits(sloss), _bits(lr), err_msg=f"loss of batch {b}")
    for (n, p), p_ref in zip(net.named_parameters(), net_ref.parameters()):
        np.testing.assert_array_equal(_bits(p), _bits(p_ref), err_msg=n)
    loss_fn.async_status()
    ma, mb = loss_fn.memory(), loss_ref.memory()
    np.testing.assert_array_equal(_bits(ma[0]), _bits(mb[0]), err_msg="memory rows")
