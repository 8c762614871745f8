"""Per-anchor loss weights (DESIGN 4.5) without a GPU: the weighted statement over both oracle restatements, its identities (w = 1 is
the unweighted oracle bit for bit, linearity in w, finite differences), the weighted record model, and the torch API's plumbing."""
import itertools

import numpy as np
import pytest
import torch

import forward_ref
import grad_ref
from npairloss_b200 import capi, synth, torch_api
from oracle import npair_oracle_np as onp

METHODS = [0, 1, 2, 3, 4]
REGIONS = [0, 1]


@pytest.mark.parametrize("world", [1, 2, 4])
def test_restatements_agree_weighted_all_modes(oracle, world):
    """The C++ oracle's weighted step (its own fp32 backward on weighted state) and the NumPy oracle's (fp64 G scaled by w) agree for
    every (region, method) combination, weights with 0, 1 and 2^-j."""
    Q, D = 24, 16
    N = Q * world
    x, lab = synth.make_inputs(N, D, seed=70 + world, imgs_per_class=3, noise=0.7)
    w = grad_ref.make_weights(N, np.random.default_rng(world))
    n = 0
    for apR, apM, anR, anM in itertools.product(REGIONS, METHODS, REGIONS, METHODS):
        kw = dict(margin_ident=0.02, margin_diff=-0.03, identsn=-0.4, diffsn=-0.3,
                  ap_region=apR, ap_method=apM, an_region=anR, an_method=anM)
        tc, dc = oracle.step_world(x, lab, oracle.make_config(Q, D, world=world, **kw), 0.7, anchor_weight=w)
        tn, dn = onp.step_world(x, lab, Q, world, 0.7, anchor_weight=w, **kw)
        np.testing.assert_allclose(tc, tn, rtol=2e-6, atol=1e-7, err_msg=str(kw))
        assert np.linalg.norm(dc - dn) <= 2e-6 * max(np.linalg.norm(dn), 1e-12), kw
        n += 1
    assert n == 100


@pytest.mark.parametrize("world", [1, 3])
def test_unit_weights_are_the_unweighted_oracle_bit_for_bit(oracle, world):
    Q, D = 20, 8
    x, lab = synth.make_inputs(Q * world, D, seed=5, imgs_per_class=2)
    for kw in (dict(synth.USAGE_MINING), dict(ap_region=0, ap_method=3, an_region=1, an_method=4, identsn=-0.4, diffsn=-0.3)):
        t0, d0 = onp.step_world(x, lab, Q, world, 0.9, **kw)
        # None checks only that no weights take the unweighted path; w = 1 runs the weighted path against it
        for w in (None, np.ones(Q * world, np.float32)):
            t1, d1 = onp.step_world(x, lab, Q, world, 0.9, anchor_weight=w, **kw)
            np.testing.assert_array_equal(t1.view(np.uint32), t0.view(np.uint32))
            np.testing.assert_array_equal(d1.view(np.uint32), d0.view(np.uint32))
        cfg = oracle.make_config(Q, 8, world=world, **kw)
        tc0, dc0 = oracle.step_world(x, lab, cfg, 0.9)
        for w in (None, np.ones(Q * world, np.float32)):
            tc1, dc1 = oracle.step_world(x, lab, cfg, 0.9, anchor_weight=w)
            np.testing.assert_array_equal(tc1.view(np.uint32), tc0.view(np.uint32))
            np.testing.assert_array_equal(dc1.view(np.uint32), dc0.view(np.uint32))


def test_linearity_in_the_weights():
    """loss(w) = sum_i w_i row_loss_i / Q, and the gradient for w is sum_i w_i times the gradient for the one-hot e_i."""
    Q, D = 6, 4
    x, lab = synth.make_inputs(Q, D, seed=11, imgs_per_class=2, noise=0.8)
    kw = dict(synth.USAGE_MINING)
    w = np.array([1.0, 0.0, 0.25, 0.7, 0.5, 0.125], np.float32)
    _, st = onp.forward(x, lab, Q, **kw)
    row_loss = -st["logv"].astype(np.float64)
    t, dx = onp.step_world(x, lab, Q, 1, anchor_weight=w.astype(np.float64), **kw)
    assert t[0, 0] == pytest.approx(float((w * row_loss).sum() / Q), rel=1e-6)
    acc = np.zeros((Q, D))
    for i in range(Q):
        e = np.zeros(Q)
        e[i] = 1.0
        acc += w[i] * onp.step_world(x, lab, Q, 1, anchor_weight=e, **kw)[1].astype(np.float64)
    np.testing.assert_allclose(dx, acc, rtol=1e-6, atol=1e-8)


@pytest.mark.parametrize("mining", ["usage", "rand"])
def test_finite_differences_of_the_weighted_loss(mining):
    """The weighted oracle's gradient is half the gradient of its loss (the reference's 1/2 at world 1), rows with w = 0 included.  S is
    computed in fp64 here and the selects are held fixed by a margin away from every threshold."""
    Q, D = 8, 5
    x, lab = synth.make_inputs(Q, D, seed=23, imgs_per_class=2, noise=0.6)
    x = x.astype(np.float64)
    kw = dict(synth.USAGE_MINING) if mining == "usage" else dict(ap_method=2, an_method=2)
    w = np.array([1.0, 0.0, 0.5, 0.25, 1.0, 0.0, 0.75, 0.125])
    _, dx = onp.step_world(x, lab, Q, 1, anchor_weight=w, **kw)
    _, st = onp.forward(x, lab, Q, **kw)
    sel = st["sel"]
    same = lab[:, None] == lab[None, :]
    np.fill_diagonal(same, False)

    def loss(xx):                                          # the weighted loss with the forward's selects
        S = xx @ xx.T
        loss = 0.0
        for i in range(Q):
            m = S[i][np.arange(Q) != i].max()
            e = np.exp(S[i] - m) * sel[i]
            A, T = e[same[i]].sum(), e.sum()
            loss -= w[i] * (np.log(A / T) if A > 0 and T > 0 else 0.0)
        return loss / Q

    h = 1e-6
    fd = np.zeros_like(x)
    for i in range(Q):
        for d in range(D):
            xp, xm = x.copy(), x.copy()
            xp[i, d] += h
            xm[i, d] -= h
            fd[i, d] = (loss(xp) - loss(xm)) / (2 * h)
    np.testing.assert_allclose(2.0 * dx, fd, rtol=2e-4, atol=2e-6)


def test_masked_row_with_an_infinite_log_adds_nothing():
    """w = 0 removes a row's term even when its log value is -inf (A / T underflowed): the loss stays finite."""
    logv = np.array([-0.5, -np.inf, -1.25], np.float32)
    assert onp.weighted_loss(logv, np.array([1.0, 0.0, 0.5], np.float32), 3) == np.float32(np.float32(-0.5 - 0.625) / np.float32(-3))


def test_weighted_record_model():
    rng = np.random.default_rng(3)
    rec = rng.standard_normal((10, 8)).astype(np.float32)
    rec[:, 5] = -np.abs(rec[:, 5])
    w = np.array([1, 0, 0.5, 2 ** -10, 0.3, 1, 0, 0.75, 1e-30, 0.999], np.float32)
    out = forward_ref.weighted_records(rec, w)
    keep = [1, 2, 3, 4, 7]
    np.testing.assert_array_equal(out[:, keep], rec[:, keep])
    np.testing.assert_array_equal(out[w == 1], rec[w == 1])
    assert np.all(np.isposinf(out[w == 0, 0])) and np.all(out[w == 0, 5:7] == 0)
    assert out[2, 0] == rec[2, 0] + 1 and out[3, 0] == rec[3, 0] + 10
    np.testing.assert_array_equal(out[:, 5], (rec[:, 5] * w).astype(np.float32))


# ---- torch API plumbing, with a stand-in context ----
class FakeContext:
    def __init__(self, cfg, nccl_id):
        self.cfg, self.calls, self.io = cfg, [], (None, None)

    def set_anchor_io(self, weight, row_loss):
        self.calls.append(("io", weight is not None, row_loss is not None))
        self.io = (weight, row_loss)

    def forward(self, feat, label):
        w, rl = self.io
        self.calls.append(("fwd", w is not None, rl is not None))
        if rl is not None:
            rl.copy_(torch.arange(1, feat.shape[0] + 1, dtype=torch.float32))     # row losses 1, 2, ..., Q
        wv = torch.ones(feat.shape[0]) if w is None else w
        return [float((wv * torch.arange(1, feat.shape[0] + 1)).sum()) / feat.shape[0], 0.5, 0.75, 1.0, 3.0]

    def backward(self, loss_weight, diff):
        self.calls.append(("bwd", loss_weight))
        diff.fill_(loss_weight)


def _module(**kw):
    made = []
    m = torch_api.NPairLoss(_context_factory=lambda c, n: made.append(FakeContext(c, n)) or made[-1], **kw)
    return m, made


def test_torch_api_validates_anchor_weight():
    m, made = _module()
    x, lab = torch.randn(4, 3), torch.tensor([0, 0, 1, 1])
    for bad, exc in ((torch.ones(4, dtype=torch.float64), TypeError), (torch.ones(4, dtype=torch.int32), TypeError),
                     ([1.0, 1.0, 1.0, 1.0], TypeError), (torch.ones(3), ValueError), (torch.ones(4, 1), ValueError),
                     (torch.ones(2, 2), ValueError)):
        with pytest.raises(exc):
            m(x, lab, anchor_weight=bad)
    assert not made or not made[0].calls, "a refused weight reached the library"


def test_torch_api_third_output_on_request_only():
    m, made = _module()
    x, lab = torch.randn(4, 3), torch.tensor([0, 0, 1, 1])
    out = m(x, lab)
    assert len(out) == 2 and made[0].calls == [("fwd", False, False)]
    out = m(x, lab, row_losses=True)
    assert len(out) == 3 and out[2].tolist() == [1.0, 2.0, 3.0, 4.0] and not out[2].requires_grad
    assert made[0].calls[1:] == [("io", False, True), ("fwd", False, True), ("io", False, False)]
    w = torch.tensor([1.0, 0.0, 0.5, 0.25])
    loss, tops = m(x, lab, anchor_weight=w)
    assert loss.item() == pytest.approx((1 + 0 + 1.5 + 1.0) / 4)
    assert made[0].calls[4:] == [("io", True, False), ("fwd", True, False), ("io", False, False)]


def test_torch_api_weight_gradient_is_row_loss_over_z():
    for kw, z in ((dict(), 4), (dict(true_gradient=True), 4)):
        m, made = _module(**kw)
        x = torch.randn(4, 3, requires_grad=True)
        w = torch.tensor([1.0, 0.0, 0.5, 0.25], requires_grad=True)
        loss, _ = m(x, torch.tensor([0, 0, 1, 1]), anchor_weight=w)
        (3.0 * loss).backward()
        np.testing.assert_allclose(w.grad.numpy(), 3.0 * np.arange(1, 5) / z, rtol=1e-6)
        assert made[0].calls[0] == ("io", True, True)
        np.testing.assert_allclose(x.grad.numpy(), np.full((4, 3), 3.0 * (2.0 if kw else 1.0)), rtol=1e-6)
