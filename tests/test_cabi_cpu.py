"""CPU-side checks of the C-ABI library: it loads without a GPU, exports every symbol the header declares, validates
arguments, and fails loudly (no CPU fallback) when no device is present."""
import ctypes as C
import os
import re

import pytest

from npairloss_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _have_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def test_library_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, "include", "npair_b200.h")).read()
    declared = set(re.findall(r"\b(npair_[a-z0-9_]+)\s*\(", hdr))
    declared.discard("npair_ctx")
    L = capi.lib()
    for sym in sorted(declared):
        assert hasattr(L, sym), f"{sym} declared in include/npair_b200.h but not exported"
    assert set(capi.EXPORTS) <= declared


def test_version_and_defaults():
    L = capi.lib()
    assert b"npairloss_b200" in L.npair_version()
    cfg = capi.NpairConfig()
    L.npair_config_default(C.byref(cfg), 120, 1024)
    # caffe.proto:4-7,19-22 defaults
    assert (cfg.margin_ident, cfg.margin_diff, cfg.identsn, cfg.diffsn) == (0.0, 0.0, -1.0, -1.0)
    assert (cfg.ap_region, cfg.ap_method, cfg.an_region, cfg.an_method) == (capi.LOCAL, capi.RAND, capi.LOCAL, capi.RAND)
    assert cfg.world == 1 and cfg.rank == 0 and cfg.num_tops == 5
    assert L.npair_workspace_bytes(C.byref(cfg)) > 120 * 120 * 4


def test_argument_validation_without_gpu():
    for bad in (dict(Q=0), dict(num_tops=6), dict(world=2, rank=2), dict(ap_method=7), dict(sim_precision=9)):
        kw = dict(Q=8, D=4)
        kw.update(bad)
        Q, D = kw.pop("Q"), kw.pop("D")
        with pytest.raises(capi.NpairError) as e:
            capi.Context(capi.make_config(Q, D, **kw))
        assert e.value.code == -1


@pytest.mark.skipif(_have_gpu(), reason="checks the no-GPU failure mode")
def test_no_cpu_fallback():
    with pytest.raises(capi.NpairError) as e:
        capi.Context(capi.make_config(8, 4))
    assert e.value.code == -2 and "no CPU fallback" in str(e.value)


@pytest.mark.skipif(_have_gpu(), reason="checks the no-GPU failure mode")
def test_no_cpu_fallback_for_the_evaluator():
    """npair_eval_create fails like npair_create, and npair_eval_last_error(NULL) reads the message the shared device check wrote."""
    with pytest.raises(capi.NpairError) as e:
        capi.Evaluator(8, 8, 4)
    assert e.value.code == -2 and "no CPU fallback" in str(e.value)


def test_config_defaults_cover_the_abi2_extensions():
    """npair_config_default: proto defaults (caffe.proto:4-7,19-22) and every ABI-2 extension switched off."""
    import ctypes as C
    from npairloss_b200 import capi
    cfg = capi.NpairConfig()
    C.memset(C.byref(cfg), 0xFF, C.sizeof(cfg))
    capi.lib().npair_config_default(C.byref(cfg), 120, 1024)
    assert (cfg.Q, cfg.D, cfg.world, cfg.rank, cfg.num_tops) == (120, 1024, 1, 0, 5)
    assert (cfg.margin_ident, cfg.margin_diff, cfg.identsn, cfg.diffsn) == (0.0, 0.0, -1.0, -1.0)
    assert (cfg.ap_region, cfg.ap_method, cfg.an_region, cfg.an_method) == (1, 2, 1, 2)
    assert (cfg.global_scope, cfg.normalize_input, cfg.grad_chunk_cols, cfg.flags) == (0, 0, 0, 0)
    assert C.sizeof(cfg) == 21 * 4
    # argument validation of the extensions (no device needed: validation comes first)
    L = capi.lib()
    for field, bad in (("global_scope", 2), ("normalize_input", -1), ("grad_chunk_cols", 100)):
        c2 = capi.make_config(64, 32, **{field: bad})
        assert L.npair_workspace_bytes(C.byref(c2)) == 0, field
    assert L.npair_workspace_bytes(C.byref(capi.make_config(64, 32, normalize_input=1))) > L.npair_workspace_bytes(C.byref(capi.make_config(64, 32)))


def _workspace(Q, D, **kw):
    return capi.lib().npair_workspace_bytes(C.byref(capi.make_config(Q, D, **kw)))


def test_workspace_counts_the_materialised_gradient_weights():
    """NPAIR_FLAG_NO_FUSED_GRAD materialises the gradient weights H: ns pieces of Q x Np 2-byte values (fp16x2: ns = 2).
    At this shape both gradient paths split K the same way, so H is the whole difference."""
    Q, D = 4096, 512
    ns, Np = 2, Q
    assert _workspace(Q, D, flags=capi.FLAG_NO_FUSED_GRAD) - _workspace(Q, D) == 2 * ns * Q * Np


@pytest.mark.parametrize("side", ["ap", "an"])
def test_workspace_counts_the_global_select_candidates_on_every_backend(side):
    """A GLOBAL RELATIVE_* side with a general SN needs two candidate lists of cap 4-byte entries, whichever GEMM backend
    computes S.  With SN = -0.0 (the usage block's) its threshold is the list's maximum, no select runs and nothing is added."""
    Q, D = 1024, 256
    cap = min(Q * Q // 8 + 4096, 32 << 20)
    for backend in (capi.GEMM_TCGEN05, capi.GEMM_SIMT_CHECK):
        base = dict(gemm_backend=backend)
        rel = dict(base, **{f"{side}_region": capi.GLOBAL, f"{side}_method": capi.RELATIVE_HARD})
        closed_form = dict(rel, **{"identsn" if side == "ap" else "diffsn": -0.0})
        assert _workspace(Q, D, **rel) - _workspace(Q, D, **base) == 8 * cap, backend
        assert _workspace(Q, D, **closed_form) == _workspace(Q, D, **base), backend
