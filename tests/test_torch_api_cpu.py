"""Autograd plumbing of npairloss_b200.torch_api with a stand-in context (no GPU): what reaches npair_forward/backward, how
the upstream gradient becomes the loss weight (.cu:435), what comes back.  The numerics are the GPU tests' business."""
import numpy as np
import torch

from npairloss_b200 import capi, torch_api


class FakeContext:
    def __init__(self, cfg, nccl_id):
        self.cfg, self.calls = cfg, []

    def forward(self, feat, label):
        self.calls.append(("fwd", tuple(feat.shape), tuple(label.shape), feat.is_contiguous(), label.dtype))
        return [float(feat.sum()) * 0 + 1.25, 0.5, 0.75, 1.0, 3.0]

    def backward(self, loss_weight, diff):
        self.calls.append(("bwd", loss_weight, tuple(diff.shape)))
        diff.fill_(2.0 * loss_weight)          # pretend dL/dx = 2 everywhere


def test_forward_backward_plumbing():
    made = []

    def factory(cfg, nid):
        made.append(FakeContext(cfg, nid)); return made[-1]

    m = torch_api.NPairLoss(_context_factory=factory, margin_diff=-0.05, an_method=capi.HARD if hasattr(capi, "HARD") else 0)
    x = torch.randn(6, 2, 2, requires_grad=True)                 # Q x C x H x W style bottom, D = 4 (.hpp:31 blob contract)
    lab = torch.tensor([0, 0, 1, 1, 2, 2])
    loss, tops = m(x, lab)
    assert loss.item() == 1.25 and tops.tolist() == [1.25, 0.5, 0.75, 1.0, 3.0] and not tops.requires_grad
    (3.0 * loss).backward()
    ctx = made[0]
    assert (ctx.cfg.Q, ctx.cfg.D) == (6, 4) and abs(ctx.cfg.margin_diff + 0.05) < 1e-7
    assert ctx.calls[0] == ("fwd", (6, 4), (6,), True, torch.float32)
    assert ctx.calls[1][0] == "bwd" and abs(ctx.calls[1][1] - 3.0) < 1e-7 and ctx.calls[1][2] == (6, 4)
    np.testing.assert_allclose(x.grad.numpy(), np.full((6, 2, 2), 6.0, np.float32))
    # same shape -> same context; new shape -> new context
    m(x.detach(), lab)
    assert len(made) == 1
    m(torch.randn(8, 4), torch.arange(8) // 2)
    assert len(made) == 2 and made[1].cfg.Q == 8


def test_rejects_other_dtypes():
    m = torch_api.NPairLoss(_context_factory=lambda c, n: FakeContext(c, n))
    try:
        m(torch.randn(4, 4, dtype=torch.float64), torch.zeros(4))
    except TypeError:
        return
    raise AssertionError("fp64 embeddings must be rejected")


def test_second_forward_invalidates_the_first_graph():
    """The library context holds ONE batch: backward of an older forward must fail loudly, not return the wrong batch's gradient."""
    m = torch_api.NPairLoss(_context_factory=lambda c, n: FakeContext(c, n))
    x1 = torch.randn(6, 4, requires_grad=True)
    x2 = torch.randn(6, 4, requires_grad=True)
    lab = torch.tensor([0, 0, 1, 1, 2, 2])
    l1, _ = m(x1, lab)
    l2, _ = m(x2, lab)
    l2.backward()                                              # the newest graph is fine
    try:
        l1.backward()
    except RuntimeError as e:
        assert "another forward" in str(e)
    else:
        raise AssertionError("stale backward must raise")


def test_labels_fp32_cannot_hold_are_refused():
    """The library compares labels in fp32: int64 ids that round onto each other, or float64 fractions, would merge classes."""
    made = []
    m = torch_api.NPairLoss(_context_factory=lambda c, n: made.append(FakeContext(c, n)) or made[-1])
    x = torch.randn(2, 4)
    for bad in (torch.tensor([2 ** 24, 2 ** 24 + 1], dtype=torch.int64), torch.tensor([0.1, 1.0], dtype=torch.float64)):
        try:
            m(x, bad)
        except ValueError as e:
            assert "fp32" in str(e)
        else:
            raise AssertionError(f"labels {bad.tolist()} ({bad.dtype}) must be refused")
    assert not made or not made[0].calls, "a refused batch reached the library"
    ok = torch.tensor([2 ** 24 - 1, -(2 ** 24) + 1], dtype=torch.int64)
    m(x, ok)
    m(x, torch.tensor([0.5, float("inf")], dtype=torch.float64))
    nan = torch.tensor([float("nan"), 3.0], dtype=torch.float32)
    assert torch_api._fp32_labels(nan) is nan or torch.equal(torch_api._fp32_labels(nan).view(torch.int32), nan.view(torch.int32))
    assert torch.equal(torch_api._fp32_labels(torch.tensor([float("nan"), 2.0], dtype=torch.float64)).isnan(), torch.tensor([True, False]))
    assert [c[0] for c in made[0].calls] == ["fwd", "fwd"] and made[0].calls[0][4] == torch.float32
    for bad in (torch.tensor([2 ** 24, 2 ** 24 + 1]), torch.tensor([0.1], dtype=torch.float64)):
        try:
            torch_api.clustering_scores(bad, torch.zeros(bad.numel(), dtype=torch.int64))
        except ValueError:
            continue
        raise AssertionError("clustering_scores must refuse labels fp32 cannot hold")


def test_true_gradient_doubles_the_reference_value():
    m = torch_api.NPairLoss(true_gradient=True, _context_factory=lambda c, n: FakeContext(c, n))
    x = torch.randn(4, 3, requires_grad=True)
    loss, _ = m(x, torch.tensor([0, 0, 1, 1]))
    loss.backward()
    np.testing.assert_allclose(x.grad.numpy(), np.full((4, 3), 4.0, np.float32))      # FakeContext: 2 * loss_weight, doubled
    try:
        torch_api.NPairLoss(world=2, true_gradient=True)
    except ValueError:
        return
    raise AssertionError("true_gradient with world > 1 must be rejected")
