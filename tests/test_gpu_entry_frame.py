"""A forward that its argument checks refuse leaves the context as the forward before it left it.

Every call of a layer context checks its arguments before it enters the context's frame (device, order across streams) and before
the forward resets the step it leaves for the backward.  So after a successful forward, a refused npair_forward and a refused
npair_forward_gathered return NPAIR_E_ARG, launch no kernel, and the backward that follows gives the gradient it gives without them,
bit for bit."""
import ctypes as C

import numpy as np
import pytest

from npairloss_b200 import capi, synth

pytestmark = pytest.mark.gpu

Q, D = 200, 72
E_ARG = next(c for c, n in capi.ERRORS.items() if n == "E_ARG")


@pytest.fixture(scope="module")
def cuda():
    import torch
    assert torch.cuda.is_available(), "GPU tests need an H100"
    assert torch.cuda.get_device_capability(0) == (9, 0)
    return torch


def _bits(a):
    return np.ascontiguousarray(np.asarray(a, np.float32)).view(np.uint32)


@pytest.mark.parametrize("backend", [capi.GEMM_TCGEN05, capi.GEMM_SIMT_CHECK], ids=["tc", "simt"])
def test_refused_forwards_keep_the_step(cuda, backend):
    torch = cuda
    x, lab = synth.make_inputs(Q, D, seed=31, imgs_per_class=4, noise=2.5)
    xt, lt = torch.from_numpy(x).cuda(), torch.from_numpy(lab).cuda()
    cfg = capi.make_config(Q, D, gemm_backend=backend, **synth.USAGE_MINING)

    def step(refuse):
        ctx = capi.Context(cfg)
        try:
            tops = ctx.forward(xt, lt)
            if refuse:
                stream = torch.cuda.current_stream().cuda_stream
                launches = capi.kernel_launches()
                with pytest.raises(capi.NpairError) as e:
                    ctx.forward_ptr(xt.data_ptr(), None, stream)          # null labels
                assert e.value.code == E_ARG, str(e.value)
                host_tops = (C.c_float * 5)()
                rc = capi.lib().npair_forward_gathered(ctx._h, xt.data_ptr(), None, host_tops, stream)
                assert rc == E_ARG, capi.lib().npair_last_error(ctx._h).decode()
                assert capi.kernel_launches() == launches, "a refused forward launched kernels"
            g = torch.full((Q, D), float("nan"), dtype=torch.float32, device="cuda")
            ctx.backward(0.8, g)
            torch.cuda.synchronize()
            return _bits(tops), _bits(g.cpu().numpy())
        finally:
            ctx.close()

    want_tops, want_grad = step(refuse=False)
    got_tops, got_grad = step(refuse=True)
    assert not np.isnan(want_grad.view(np.float32)).any()
    assert np.array_equal(got_tops, want_tops)
    assert np.array_equal(got_grad, want_grad), "the backward after the refused forwards"
