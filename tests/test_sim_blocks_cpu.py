"""Row-block similarity mode (NPAIR_SIM_BLOCK_ROWS) without a GPU: the configuration bits, the workspace it plans and the
configurations it refuses."""
import ctypes as C

import pytest

from npairloss_b200 import capi


def _workspace(Q, D, **kw):
    return capi.lib().npair_workspace_bytes(C.byref(capi.make_config(Q, D, **kw)))


def test_make_config_folds_the_height_into_flags():
    assert capi.make_config(64, 32).flags == 0
    assert capi.make_config(64, 32, sim_block_rows=128).flags == 1 << 16
    assert capi.make_config(64, 32, sim_block_rows=200).flags == 2 << 16          # rounded up to a multiple of 128
    assert capi.make_config(64, 32, sim_block_rows=2048).flags == 16 << 16
    f = capi.make_config(64, 32, flags=capi.FLAG_LSEL_WARP, sim_block_rows=384).flags
    assert f == capi.FLAG_LSEL_WARP | (3 << 16)
    assert (f >> capi.SIM_BLOCK_SHIFT) & capi.SIM_BLOCK_MAX_UNITS == 3
    with pytest.raises(ValueError):
        capi.make_config(64, 32, sim_block_rows=128 * 4096)


@pytest.mark.parametrize("world", [1, 2])
def test_workspace_keeps_one_block_of_s(world):
    """Only S shrinks: from Q x ldS to Qb x ldS fp32 values (ldS = N rounded up to 32)."""
    Q, D, Qb = 4096, 512, 1024
    N = Q * world
    ldS = (N + 31) // 32 * 32
    full = _workspace(Q, D, world=world)
    blk = _workspace(Q, D, world=world, sim_block_rows=Qb)
    assert full > 0 and blk > 0
    assert full - blk == 4 * (Q - Qb) * ldS


def test_height_at_least_q_is_the_materialised_path():
    Q, D = 1000, 256
    assert _workspace(Q, D, sim_block_rows=1024) == _workspace(Q, D)
    assert _workspace(Q, D, sim_block_rows=896) < _workspace(Q, D)


REFUSED = {
    "simt_backend": dict(gemm_backend=capi.GEMM_SIMT_CHECK),
    "no_fused_grad": dict(flags=capi.FLAG_NO_FUSED_GRAD),
    "reduce_scatter": dict(world=2, bwd_exchange=1),
    "global_scope_w1": dict(global_scope=1),
    "global_scope_w2": dict(world=2, global_scope=1),
    "global_rel_ap_general_sn": dict(ap_region=capi.GLOBAL, ap_method=capi.RELATIVE_HARD, identsn=-0.3),
    "global_rel_an_general_sn": dict(an_region=capi.GLOBAL, an_method=capi.RELATIVE_EASY, diffsn=1.0),
}


@pytest.mark.parametrize("name", sorted(REFUSED))
def test_refused_configurations_have_no_workspace(name):
    Q, D = 1024, 128
    kw = REFUSED[name]
    assert _workspace(Q, D, **kw) > 0, "the configuration itself is valid without row blocks"
    assert _workspace(Q, D, sim_block_rows=256, **kw) == 0


@pytest.mark.parametrize("kw", [
    dict(ap_region=capi.GLOBAL, ap_method=capi.RELATIVE_HARD, identsn=-0.0, an_region=capi.GLOBAL, an_method=capi.RELATIVE_HARD, diffsn=0.5),
    dict(ap_region=capi.LOCAL, ap_method=capi.RELATIVE_HARD, identsn=-0.3, an_region=capi.LOCAL, an_method=capi.RELATIVE_EASY, diffsn=-0.7),
    dict(ap_region=capi.GLOBAL, ap_method=capi.HARD, an_region=capi.GLOBAL, an_method=capi.EASY),
    dict(world=2, normalize_input=1, sim_precision=capi.PREC_BF16),
    dict(world=3, flags=capi.FLAG_NCCL_RECORDS | capi.FLAG_NCCL_FEATURES),
], ids=["global_closed_form", "local_general_sn", "global_plain", "w2_normalize_bf16", "w3_nccl"])
def test_accepted_configurations(kw):
    assert _workspace(1024, 128, sim_block_rows=256, **kw) > 0


def test_refused_at_create_with_an_argument_error():
    with pytest.raises(capi.NpairError) as e:
        capi.Context(capi.make_config(1024, 128, sim_block_rows=256, gemm_backend=capi.GEMM_SIMT_CHECK))
    assert e.value.code == -1 and "row-block" in str(e.value)
