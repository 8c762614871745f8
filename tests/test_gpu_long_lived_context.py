"""One layer context through a run of training steps, bit for bit against a fresh context per step.

A training job creates one context and calls it thousands of times, and the context carries state from one call to the next: the
BlockScalars (tickets, error bits, select counters, the pre-scale), the GLOBAL select's histogram and candidates, the host-side step
state (the published tops and their sequence number, whether a forward succeeded), the row block S holds in row-block mode, and
buffers every step rewrites (the normalised rows, the split-K partial products, the row records).  The layer is bitwise deterministic
(its atomics are integer counts or ordered-uint min / max), so a script of steps on one context must give exactly the bits that a new
context gives for each step on its own; any difference is state that leaked from an earlier step.  Each step changes something a
stale value would hide: the pre-scale's binade, the select paths (collapsed rows), an error, two forwards before one backward, two
backwards after one forward, inputs written in place, inputs off the 16-byte grid, a zero loss weight, and a switch of stream while
the previous backward is still queued behind a sleep (the context must order its own work across streams).

The fresh results are checked against the oracle (gpu_harness.check_parity) on the script's first batch; the first step after the
error runs that batch again and must equal the first step bit for bit."""
import numpy as np
import pytest

from npairloss_b200 import capi, synth

pytestmark = pytest.mark.gpu

Q, D = 333, 72
FP16X2, BF16X3, BF16 = capi.PREC_FP32_FP16X2, capi.PREC_FP32_BF16X3, capi.PREC_BF16
REL_H, REL_E = synth.RELATIVE_HARD, synth.RELATIVE_EASY
E_EMPTY_LIST, E_POS_RANGE, E_STATE = (next(c for c, n in capi.ERRORS.items() if n == name) for name in ("E_EMPTY_LIST", "E_POS_RANGE", "E_STATE"))
# about 50 ms of GPU time at the H100's clocks: long enough for a whole step issued behind it on another stream to finish first
SLEEP_CYCLES = 100_000_000


@pytest.fixture(scope="module")
def cuda():
    import torch
    assert torch.cuda.is_available(), "GPU tests need an H100"
    assert torch.cuda.get_device_capability(0) == (9, 0)
    return torch


def _mining(region, identsn, diffsn, ap_method=REL_H, an_method=REL_H):
    return dict(margin_ident=0.01, margin_diff=-0.02, identsn=identsn, diffsn=diffsn, ap_region=region, ap_method=ap_method,
                an_region=region, an_method=an_method)


GLOBAL_REL = _mining(synth.GLOBAL, -0.3, -0.45, REL_H, REL_E)
LOCAL_REL = _mining(synth.LOCAL, -0.3, -0.4, REL_E, REL_H)

# name -> (world, mining, make_config extras)
CONFIGS = {
    "usage_fp16x2": (1, synth.USAGE_MINING, dict(sim_precision=FP16X2)),
    "global_rel_bf16x3": (1, GLOBAL_REL, dict(sim_precision=BF16X3)),
    "local_rel": (1, LOCAL_REL, dict(sim_precision=FP16X2)),
    "local_rel_warp": (1, LOCAL_REL, dict(sim_precision=FP16X2, flags=capi.FLAG_LSEL_WARP)),
    "row_blocks": (1, LOCAL_REL, dict(sim_precision=BF16X3, sim_block_rows=128)),       # three blocks at Q = 333
    "normalize_input": (1, synth.USAGE_MINING, dict(sim_precision=FP16X2, normalize_input=1)),
    "bf16": (1, synth.USAGE_MINING, dict(sim_precision=BF16)),
    "no_fused_grad": (1, synth.USAGE_MINING, dict(sim_precision=FP16X2, flags=capi.FLAG_NO_FUSED_GRAD, grad_chunk_cols=64)),
    # bwd_exchange 0 (AUTO) gives the row-record exchange (mode 2) on a device whose MMA is bitwise symmetric, 1 forces reduce-scatter
    "world2_row_records": (2, GLOBAL_REL, dict(sim_precision=FP16X2, bwd_exchange=0)),
    "world2_reduce_scatter": (2, GLOBAL_REL, dict(sim_precision=FP16X2, bwd_exchange=1)),
}


def _bits(a):
    return np.ascontiguousarray(np.asarray(a, np.float32)).view(np.uint32)


def _unit(x):
    return np.ascontiguousarray(x / np.linalg.norm(x.astype(np.float64), axis=1, keepdims=True).astype(np.float32), np.float32)


def _collapsed(B, seed, eps=0.03):
    """Rows normalize(e0 + eps g): every similarity close to one value, which sends the relative selects to their fallbacks."""
    rng = np.random.default_rng(seed)
    e = np.zeros(D, np.float32)
    e[0] = 1.0
    return _unit(e[None, :] + np.float32(eps) * rng.standard_normal((B, D)).astype(np.float32))


def _labels(n, per_class):
    """Classes of per_class rows, the rows left over joining the last class: every row has a same-label partner, which LOCAL
    relative mining needs (a row alone in its class is refused with E_EMPTY_LIST)."""
    return np.minimum(np.arange(n) // per_class, n // per_class - 1).astype(np.float32)


def _batch(n, seed, per_class=4, scale=1.0, zero_row=None):
    x, _ = synth.make_inputs(n, D, seed=seed, imgs_per_class=per_class, noise=2.5)
    lab = _labels(n, per_class)
    x = np.ascontiguousarray(x * np.float32(scale))
    if zero_row is not None:
        x[zero_row] = 0.0
    return x, lab


class Runner:
    """All ranks of one configuration (world 2: emulated on one GPU through the external-collectives calls, as
    gpu_harness.gpu_step_world does, but with contexts that live until close())."""

    def __init__(self, spec):
        self.world, self.mining, extra = spec
        self.N = self.world * Q
        self.blocks = extra.get("sim_block_rows", 0) > 0
        self.ctxs = []
        try:
            for r in range(self.world):
                self.ctxs.append(capi.Context(capi.make_config(Q, D, world=self.world, rank=r, **self.mining, **extra)))
        except Exception:
            self.close()
            raise
        if self.world > 1:
            assert self.ctxs[0].bwd_exchange_mode() == (1 if extra.get("bwd_exchange") else 2)

    def close(self):
        for c in self.ctxs:
            c.close()

    def forward(self, xt, lt, lw=None, dx=None):
        """The step's forward (with the backward in the same call when lw is given, world 1); returns its observation."""
        try:
            if self.world == 1 and lw is not None:
                tops = [self.ctxs[0].forward_backward(xt, lt, lw, dx)]
            elif self.world == 1:
                tops = [self.ctxs[0].forward(xt, lt)]
            else:
                tops, errs = [], []
                for c in self.ctxs:             # every rank runs its forward, as on separate GPUs, before an error is reported
                    try:
                        tops.append(c.forward_gathered(xt, lt))
                    except capi.NpairError as e:
                        errs.append(e)
                if errs:
                    raise errs[0]
        except capi.NpairError as e:
            return {"rc": e.code, "dbg": self._debug(error=True)}
        return {"rc": 0, "tops": _bits(tops).tobytes(), "dbg": self._debug(error=False)}

    def _debug(self, error):
        # after a refused forward only what precedes the selects is compared: the thresholds and weights of rows whose lists are
        # empty are unspecified (the reference's behaviour there is undefined)
        which = (3, 4, 5, 8, 9) if error else tuple(range(1, 10))
        out = {w: b"".join(_bits(c.debug_read(w, Q)).tobytes() for c in self.ctxs) for w in which}
        out[10] = b"".join(_bits(c.debug_read(10, 1)).tobytes() for c in self.ctxs)
        if not self.blocks:
            out[0] = b"".join(_bits(c.debug_read(0, Q * self.N)).tobytes() for c in self.ctxs)
        return out

    def backward(self, lw):
        """Enqueues the backward on the current stream; returns the gradient tensor (N x D), or the error code."""
        import torch
        try:
            if self.world == 1:
                g = torch.full((Q, D), float("nan"), dtype=torch.float32, device="cuda")
                self.ctxs[0].backward(lw, g)
                return g
            mode = self.ctxs[0].bwd_exchange_mode()
            if mode == 2:
                rs = torch.empty((self.world, Q, 8), dtype=torch.float32, device="cuda")
                for r, c in enumerate(self.ctxs):
                    c.row_scalars(rs[r])
                g = torch.full((self.N, D), float("nan"), dtype=torch.float32, device="cuda")
                for r, c in enumerate(self.ctxs):
                    c.backward_gathered(lw, rs, g[r * Q:(r + 1) * Q])
                return g
            local = torch.full((self.N, D), float("nan"), dtype=torch.float32, device="cuda")
            total = torch.zeros((self.N, D), dtype=torch.float32, device="cuda")
            for r, c in enumerate(self.ctxs):
                th = torch.full((self.N, D), float("nan"), dtype=torch.float32, device="cuda")
                c.backward_partial(lw, local[r * Q:(r + 1) * Q], th)
                total += th
            return local + total
        except capi.NpairError as e:
            return e.code


def _grad(g):
    """Observation of a backward's result (after a synchronisation)."""
    return {"rc": g} if isinstance(g, int) else {"rc": 0, "grad": _bits(g.cpu().numpy()).tobytes()}


def _offset_view(torch, src, off):
    buf = torch.empty(src.numel() + 4, dtype=src.dtype, device=src.device)
    v = buf[off:off + src.numel()].view(src.shape)
    v.copy_(src)
    return v


# ------------------------------------------------------------------------------------------------------------------------- the script
# Each step: (name, live(run, state) -> observations, fresh ops).  `fresh` lists the calls a new context makes for the same step's
# observations, one new context per entry; None = the live calls.  `state` carries tensors from one step to the next.
def _tensors(torch, x, lab):
    return torch.from_numpy(x).cuda(), torch.from_numpy(lab).cuda()


def _plain(data, lw):
    def run(torch, rn, st):
        xt, lt = _tensors(torch, *data)
        obs = [rn.forward(xt, lt)]
        g = rn.backward(lw)
        torch.cuda.synchronize()
        return obs + [_grad(g)]
    return run


def _fused(data, lw):
    def run(torch, rn, st):
        xt, lt = _tensors(torch, *data)
        if rn.world > 1:                # no npair_forward_backward for external collectives
            return _plain(data, lw)(torch, rn, st)
        g = torch.full((Q, D), float("nan"), dtype=torch.float32, device="cuda")
        obs = rn.forward(xt, lt, lw, g)
        torch.cuda.synchronize()
        return [obs, _grad(g)]
    return run


def _two_forwards(first, second, lw):
    def run(torch, rn, st):
        xt, lt = _tensors(torch, *first)
        assert rn.forward(xt, lt)["rc"] == 0
        return _plain(second, lw)(torch, rn, st)
    return run


def _two_backwards(data, lw):
    def run(torch, rn, st):
        xt, lt = _tensors(torch, *data)
        obs = [rn.forward(xt, lt)]
        g1 = rn.backward(lw)
        g2 = rn.backward(lw)
        torch.cuda.synchronize()
        obs += [_grad(g1), _grad(g2)]
        assert obs[1] == obs[2], "two backwards of one forward differ"
        return obs
    return run


def _keep_inputs(data, lw):
    def run(torch, rn, st):
        st["x"], st["lab"] = _tensors(torch, *data)
        obs = [rn.forward(st["x"], st["lab"])]
        g = rn.backward(lw)
        torch.cuda.synchronize()
        return obs + [_grad(g)]
    return run


def _in_place(data, lw):
    def run(torch, rn, st):
        x, lab = data
        if "x" not in st:               # a fresh context's step: new tensors
            st["x"], st["lab"] = _tensors(torch, x, lab)
        else:                           # after the previous step has finished
            st["x"].copy_(torch.from_numpy(x))
            st["lab"].copy_(torch.from_numpy(lab))
        obs = [rn.forward(st["x"], st["lab"])]
        g = rn.backward(lw)
        torch.cuda.synchronize()
        st.clear()
        return obs + [_grad(g)]
    return run


def _offsets(data, lw):
    def run(torch, rn, st):
        xt, lt = _tensors(torch, *data)
        xv, lv = _offset_view(torch, xt, 1), _offset_view(torch, lt, 3)
        assert xv.data_ptr() % 16 and lv.data_ptr() % 16
        obs = [rn.forward(xv, lv)]
        g = rn.backward(lw)
        torch.cuda.synchronize()
        return obs + [_grad(g)]
    return run


def _stream_switch(first, second, lw):
    """On stream A: the first batch's forward, a sleep, its backward; then at once, on stream B, the second batch's forward and
    backward.  The context must make B wait for A's backward: without that, B's forward runs during the sleep and A's backward reads
    the second batch's scratch."""
    def run(torch, rn, st):
        xa, la = _tensors(torch, *first)
        xb, lb = _tensors(torch, *second)
        torch.cuda.synchronize()
        sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
        with torch.cuda.stream(sa):
            obs = [rn.forward(xa, la)]
            torch.cuda._sleep(SLEEP_CYCLES)
            ga = rn.backward(lw)
        with torch.cuda.stream(sb):
            obs_b = rn.forward(xb, lb)
            gb = rn.backward(lw)
        torch.cuda.synchronize()
        return obs + [_grad(ga), obs_b, _grad(gb)]

    def fresh_first(torch, rn, st):
        return _plain(first, lw)(torch, rn, st)

    def fresh_second(torch, rn, st):
        return _plain(second, lw)(torch, rn, st)
    return run, [fresh_first, fresh_second]


def _error_step(data):
    def run(torch, rn, st):
        xt, lt = _tensors(torch, *data)
        obs = [rn.forward(xt, lt)]
        assert obs[0]["rc"] in (E_EMPTY_LIST, E_POS_RANGE), f"the forward returned {obs[0]['rc']}, not E_EMPTY_LIST / E_POS_RANGE"
        g = rn.backward(1.0)
        torch.cuda.synchronize()
        assert g == E_STATE, f"a backward after a refused forward returned {g}, not E_STATE"
        return obs + [_grad(g)]
    return run


def _script(world):
    n = world * Q
    b1 = _batch(n, 1)
    collapsed = (_collapsed(n, 3), _labels(n, 4))
    distinct = (_batch(n, 4)[0], np.arange(n, dtype=np.float32))        # no same-label pair: every mining index is refused
    steps = [
        ("1 plain", _plain(b1, 1.0), None),
        ("2 rows x4, forward_backward", _fused(_batch(n, 2, per_class=3, scale=4.0), 0.7), None),
        ("3 collapsed", _plain(collapsed, -0.5), None),
        ("4 refused forward", _error_step(distinct), None),
        ("5 step 1 again", _plain(b1, 1.0), None),
        ("6 forward, forward, backward", _two_forwards(_batch(n, 6), _batch(n, 7, per_class=5), 1.0),
         [_plain(_batch(n, 7, per_class=5), 1.0)]),
        ("7 forward, backward, backward", _two_backwards(_batch(n, 8, per_class=2), 0.9), None),
        ("8 rows x2^-5, a zero row", _keep_inputs(_batch(n, 9, scale=2.0 ** -5, zero_row=7), 1.0), None),
        ("9 inputs in place", _in_place(_batch(n, 10, per_class=3), 1.0), None),
        ("10 inputs off the 16-byte grid", _offsets(_batch(n, 11), 1.0), None),
        ("11 loss weight 0", _plain(_batch(n, 12), 0.0), None),
    ]
    live12, fresh12 = _stream_switch(_batch(n, 13), _batch(n, 14, per_class=6, scale=3.0), 1.0)
    steps.append(("12 stream switch behind a queued backward", live12, fresh12))
    steps.append(("13 step 1 again", _plain(b1, 1.0), None))
    return steps, b1


def _fresh(torch, spec, step):
    _, live, fresh = step
    obs, st = [], {}
    for op in fresh or [live]:
        rn = Runner(spec)
        try:
            obs += op(torch, rn, st)
        finally:
            rn.close()
    return obs


def _diff(a, b):
    """Names of the fields two observations differ in."""
    keys = sorted(set(a) | set(b), key=str)
    out = [k for k in keys if k != "dbg" and a.get(k) != b.get(k)]
    da, db = a.get("dbg", {}), b.get("dbg", {})
    out += [f"debug {w}" for w in sorted(set(da) | set(db)) if da.get(w) != db.get(w)]
    return out


@pytest.mark.parametrize("name", list(CONFIGS))
def test_long_lived_context(cuda, oracle, name):
    torch = cuda
    world, mining, extra = CONFIGS[name]
    steps, b1 = _script(world)
    fresh = [_fresh(torch, CONFIGS[name], s) for s in steps]
    rn = Runner(CONFIGS[name])
    try:
        st = {}
        for i, step in enumerate(steps):
            got = step[1](torch, rn, st)
            assert len(got) == len(fresh[i]), step[0]
            for k, (a, b) in enumerate(zip(got, fresh[i])):
                assert a == b, f"{name}, step {step[0]}, observation {k}: {_diff(a, b)} differ from a fresh context's"
    finally:
        torch.cuda.synchronize()
        rn.close()
    assert fresh[4] == fresh[0] and fresh[12] == fresh[0], "the same batch gave different bits on fresh contexts"
    _check_first_step(torch, oracle, name, b1, fresh[0])


def _check_first_step(torch, oracle, name, b1, obs):
    """The fresh results are right, not just consistent: the first step's observations `obs` are bit for bit those of
    gpu_harness.gpu_step_world (the external-collectives calls), whose result then goes through the oracle check.  Row-block mode: its
    materialised twin, whose bits it must have, stands in.  normalize_input: the step is the L2Normalize of the rows, the layer
    without normalize_input on those rows, and the L2Normalize backward of its gradient."""
    import gpu_harness
    world, mining, extra = CONFIGS[name]
    prec = extra["sim_precision"]
    cfg = {k: v for k, v in extra.items() if k != "sim_precision"}
    if cfg.pop("sim_block_rows", 0):
        twin = _fresh(torch, (world, mining, dict(cfg, sim_precision=prec)), ("1 plain", _plain(b1, 1.0), None))
        for a, b in zip(obs, twin):
            b = dict(b, dbg={w: v for w, v in b.get("dbg", {}).items() if w != 0}) if "dbg" in b else b
            assert a == b, f"{name}: row-block step 1 vs the materialised path: {_diff(a, b)}"
        obs = twin
    x, lab = b1
    y = inv = None
    if cfg.pop("normalize_input", 0):
        y, inv = capi.l2normalize_forward(torch.from_numpy(x).cuda())
        x = y.cpu().numpy()
    g = gpu_harness.gpu_step_world(x, lab, Q, world, mining, prec, capi.GEMM_TCGEN05, loss_weight=1.0, **cfg)
    fwd, bwd = obs
    assert fwd["tops"] == _bits(g["tops"]).tobytes(), f"{name}: tops"
    for w, key in ((0, "S"), (1, "posi"), (2, "nega")):
        assert fwd["dbg"][w] == _bits(g[key]).tobytes(), f"{name}: {key}"
    dx = g["dx"]
    if y is not None:
        dx = capi.l2normalize_backward(y, inv, torch.from_numpy(dx).cuda()).cpu().numpy()
    # gpu_step_world adds a zero transposed term at world 1, which turns -0.0 into +0.0: compare values, not bits
    assert np.array_equal(np.frombuffer(bwd["grad"], np.float32).reshape(dx.shape), dx), f"{name}: gradient"
    gpu_harness.check_parity(oracle, x, lab, Q, world, mining, prec, capi.GEMM_TCGEN05, loss_weight=1.0, tag=f"{name} step 1", gpu=g,
                             **cfg)


# ------------------------------------------------------------------------------------------------------- two contexts, interleaved
def test_two_contexts_interleaved(cuda):
    """fp16x2 Q = 512 materialised and bf16x3 Q = 333 in row-block mode, alternating forward_backward steps on two streams (each
    context switching stream every step): each equals its own fresh results, so nothing in the library is shared between them."""
    torch = cuda
    specs = [(512, dict(synth.USAGE_MINING, sim_precision=FP16X2)), (333, dict(LOCAL_REL, sim_precision=BF16X3, sim_block_rows=128))]

    def step(ctx, q, i):
        x, _ = synth.make_inputs(q, D, seed=900 + 10 * i + q, imgs_per_class=2 + i % 3, noise=2.5)
        lab = _labels(q, 2 + i % 3)
        xt, lt = _tensors(torch, np.ascontiguousarray(x * np.float32(2.0 ** (3 * (i % 3) - 3))), lab)
        g = torch.full((q, D), float("nan"), dtype=torch.float32, device="cuda")
        tops = ctx.forward_backward(xt, lt, 0.8, g)
        return tops, g

    n_steps = 6
    want = []
    for i in range(n_steps):
        row = []
        for q, kw in specs:
            ctx = capi.Context(capi.make_config(q, D, **kw))
            try:
                tops, g = step(ctx, q, i)
                torch.cuda.synchronize()
                row.append((_bits(tops).tobytes(), _bits(g.cpu().numpy()).tobytes()))
            finally:
                ctx.close()
        want.append(row)
    ctxs = [capi.Context(capi.make_config(q, D, **kw)) for q, kw in specs]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    try:
        torch.cuda.synchronize()
        for i in range(n_steps):
            outs = []
            for k, (q, _) in enumerate(specs):
                with torch.cuda.stream(streams[(i + k) % 2]):
                    outs.append(step(ctxs[k], q, i))
            torch.cuda.synchronize()
            for k, (tops, g) in enumerate(outs):
                got = (_bits(tops).tobytes(), _bits(g.cpu().numpy()).tobytes())
                assert got[0] == want[i][k][0], f"context {k}, step {i}: tops"
                assert got[1] == want[i][k][1], f"context {k}, step {i}: gradient"
    finally:
        torch.cuda.synchronize()
        for c in ctxs:
            c.close()


# --------------------------------------------------------------------------------------------------------------- torch_api.NPairLoss
def test_npairloss_module_across_batch_sizes(cuda):
    """One NPairLoss module over batches of 333, 333, 200 and 333 rows (the context is re-created for 200 and again for 333): every
    gradient and loss equals a fresh module's bit for bit, and a backward through an older forward is still refused."""
    torch = cuda
    from npairloss_b200.torch_api import NPairLoss
    kw = dict(LOCAL_REL, sim_precision=FP16X2)

    def batch(n, i):
        x, _ = synth.make_inputs(n, D, seed=950 + i, imgs_per_class=3, noise=2.5)
        return torch.from_numpy(x * np.float32(1.5 ** i)).cuda().requires_grad_(True), torch.from_numpy(_labels(n, 3)).cuda()

    def run(mod, n, i):
        x, lab = batch(n, i)
        loss, tops = mod(x, lab)
        (0.6 * loss).backward()
        torch.cuda.synchronize()
        return _bits(tops.cpu().numpy()).tobytes(), _bits(x.grad.cpu().numpy()).tobytes()

    sizes = [333, 333, 200, 333]
    want = [run(NPairLoss(**kw), n, i) for i, n in enumerate(sizes)]
    mod = NPairLoss(**kw)
    for i, n in enumerate(sizes):
        assert run(mod, n, i) == want[i], f"step {i} (batch {n})"
    x1, l1 = batch(333, 0)
    x2, l2 = batch(333, 1)
    loss1, _ = mod(x1, l1)
    loss2, _ = mod(x2, l2)
    with pytest.raises(RuntimeError, match="another forward ran through this module"):
        loss1.backward()
    (0.6 * loss2).backward()
    torch.cuda.synchronize()
    assert _bits(x2.grad.cpu().numpy()).tobytes() == want[1][1], "the newer forward's backward"
