"""The Caffe shim's optional third bottom of anchor weights (DESIGN 4.5): the prototxt (CPU) and the weighted tops and gradient through
the layer (GPU)."""
import numpy as np
import pytest

import grad_ref
from npairloss_b200 import caffe_layer, synth

THREE_BOTTOMS = caffe_layer.layer_prototxt(synth.USAGE_MINING, 5, anchor_weights=True)


def test_parse_three_bottoms():
    p = caffe_layer.parse_only(THREE_BOTTOMS)
    assert p["num_bottoms"] == 3 and p["num_tops"] == 5 and p["n_loss_weights"] == 5
    assert (p["ap_region"], p["ap_method"], p["an_region"], p["an_method"]) == (0, 3, 1, 0)
    assert caffe_layer.parse_only(caffe_layer.layer_prototxt(synth.USAGE_MINING, 5))["num_bottoms"] == 2


@pytest.mark.gpu
def test_third_bottom_gives_the_weighted_tops_and_gradient(oracle):
    """w = 1 in the third bottom is the two-bottom layer bit for bit; random weights give the weighted oracle's loss and gradient on
    the layer's S, and tops 1-4 of the unweighted layer."""
    import torch

    from npairloss_b200 import capi
    Q, D = 120, 256
    x, lab = synth.make_inputs(Q, D, seed=42, noise=2.5)
    w = grad_ref.make_weights(Q, np.random.default_rng(42))

    def run(prototxt, weights=None):
        layer = caffe_layer.Layer(prototxt, Q, D)
        try:
            layer.bottom_data(0)[:] = x.ravel()
            layer.bottom_data(1)[:] = lab
            if weights is not None:
                layer.bottom_data(2)[:] = weights
            tops, _ = layer.forward()
            layer.backward()
            return np.array(tops, np.float32), layer.bottom_diff().copy()
        finally:
            layer.close()

    t2, d2 = run(caffe_layer.layer_prototxt(synth.USAGE_MINING, 5))
    t1, d1 = run(THREE_BOTTOMS)                       # the harness fills the weight blob with 1
    np.testing.assert_array_equal(t1.view(np.uint32), t2.view(np.uint32))
    np.testing.assert_array_equal(d1.view(np.uint32), d2.view(np.uint32))
    tw, dw = run(THREE_BOTTOMS, w)
    np.testing.assert_array_equal(tw[1:], t2[1:])
    # S of the same forward, from a context of the same configuration (the similarity sweep is deterministic)
    ctx = capi.Context(capi.make_config(Q, D, **synth.USAGE_MINING))
    try:
        ctx.forward(torch.from_numpy(x).cuda(), torch.from_numpy(lab).cuda())
        S = ctx.debug_read(0, Q * Q).reshape(Q, Q)
    finally:
        ctx.close()
    cfg = oracle.make_config(Q, D, faithful_sorts=0, **synth.USAGE_MINING)
    tops_o, dx_o = oracle.step_world(x, lab, cfg, 1.0, S_inject_all=S, anchor_weight=w)
    np.testing.assert_allclose(tw[0], tops_o[0, 0], rtol=1e-5, atol=1e-6)
    assert np.linalg.norm(dw - dx_o) <= 1e-5 * np.linalg.norm(dx_o)
    assert np.linalg.norm(dw - d2) > 0
