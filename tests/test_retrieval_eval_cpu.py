"""CPU-side checks of the retrieval evaluator (include/npair_b200.h, DESIGN 8): its symbols are exported, its workspace is linear in
the set sizes, it validates its arguments, and it fails loudly (no CPU fallback) when no device is present."""
import ctypes as C

import pytest

from npairloss_b200 import capi

EVAL_SYMBOLS = ["npair_eval_workspace_bytes", "npair_eval_create", "npair_eval_destroy", "npair_eval_last_error", "npair_eval_rank",
                "npair_eval_best_positive", "npair_eval_count"]


def _have_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def test_eval_symbols_declared_and_exported():
    L = capi.lib()
    for s in EVAL_SYMBOLS:
        assert s in capi.EXPORTS
        assert hasattr(L, s), s


@pytest.mark.parametrize("prec,segments", [(capi.PREC_FP32_BF16X3, 6), (capi.PREC_BF16, 1), (capi.PREC_FP32_FP16X2, 3)])
def test_eval_workspace_linear_in_set_sizes(prec, segments):
    D = 512
    ws = lambda q, g, d=D: capi.eval_workspace_bytes(q, g, d, prec)     # noqa: E731
    n = 60502                                                             # Stanford Online Products' test set
    operands = 2 * (n + n) * segments * D
    assert operands <= ws(n, n) <= operands + 20 * n + (1 << 20)         # + per-query statistics and the symmetric tile list
    assert ws(n, n) < 0.1 * 4 * n * n                                  # the fp32 similarity matrix would take 14.6 GB
    # one more query or gallery row costs its operand row (and a query its statistics), whatever the other set's size; the symmetric
    # tile list of min(max_queries, max_gallery) = 5000 rows gains at most a row and a column of 8-byte tiles
    row = 2 * segments * D
    for other in (1000, 100000):
        assert 0 <= ws(5000, other) - ws(4999, other) - (row + 20) <= 8 * 64
        assert 0 <= ws(other, 5000) - ws(other, 4999) - row <= 8 * 64
    # doubling both sets doubles the workspace (a product term would quadruple it)
    assert ws(2 * n, 2 * n) < 2.01 * ws(n, n)
    # and it is linear in D
    assert ws(n, 1000, 1024) - ws(n, 1000, 512) == 2 * (n + 1000) * segments * 512


@pytest.mark.parametrize("bad", [dict(max_q=0), dict(max_g=0), dict(D=0), dict(prec=3), dict(prec=-1), dict(max_q=-5),
                                 dict(max_g=1 << 30)])
def test_eval_invalid_arguments(bad):
    kw = dict(max_q=100, max_g=200, D=64, prec=capi.PREC_FP32_FP16X2)
    kw.update(bad)
    L = capi.lib()
    assert L.npair_eval_workspace_bytes(kw["max_q"], kw["max_g"], kw["D"], kw["prec"]) == 0
    h = C.c_void_p()
    assert L.npair_eval_create(kw["max_q"], kw["max_g"], kw["D"], kw["prec"], -1, C.byref(h)) == -1
    assert not h.value
    assert L.npair_eval_last_error(None)
    with pytest.raises(capi.NpairError) as e:
        capi.Evaluator(kw["max_q"], kw["max_g"], kw["D"], kw["prec"])
    assert e.value.code == -1


def test_eval_calls_without_evaluator():
    L = capi.lib()
    assert L.npair_eval_rank(None, None, None, 1, None, None, 1, -1, None, None) == -1
    assert L.npair_eval_best_positive(None, None, None, 1, None, None, 1, -1, 0, C.c_float(1.0), None, None) == -1
    assert L.npair_eval_count(None, None, 1, None, 1, -1, 0, C.c_float(1.0), None, None, None) == -1
    L.npair_eval_destroy(None)


@pytest.mark.skipif(_have_gpu(), reason="checks the no-GPU failure mode")
def test_eval_no_cpu_fallback():
    with pytest.raises(capi.NpairError) as e:
        capi.Evaluator(100, 200, 64)
    assert e.value.code == -2 and "no CPU fallback" in str(e.value)


def test_recall_at_k_rejects_cpu_tensors():
    torch = pytest.importorskip("torch")
    from npairloss_b200.torch_api import recall_at_k
    with pytest.raises(TypeError):
        recall_at_k(torch.zeros(8, 4), torch.zeros(8))
