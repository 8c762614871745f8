"""The exact-threshold reference of tests/select_ref.py against a full sort and against the C++ oracle, its pos() against the oracle's,
and its restated candidate-buffer size against the library's workspace size."""
import ctypes as C

import numpy as np
import pytest

import select_ref
from npairloss_b200 import capi, synth

SNS = [-0.3, -0.5, -0.97, -0.0, 0.0, 0.5, 1.0, 3.0, 7.0]


def _sorted_pick(vals, sn):
    p = select_ref.pos(sn, vals.size)
    return None if p is None else np.sort(vals, kind="stable")[p]


def _lists(S, lab, self_offset, i=None):
    same, diff = select_ref.side_masks(lab[self_offset:self_offset + S.shape[0]], lab, self_offset)
    if i is None:
        return S[same], S[diff]
    return S[i, same[i]], S[i, diff[i]]


@pytest.mark.parametrize("tied", [False, True])
@pytest.mark.parametrize("world,rank", [(1, 0), (2, 1)])
def test_reference_matches_full_sort_and_oracle(oracle, tied, world, rank):
    rng = np.random.default_rng(3 + tied + 2 * rank)
    Q, D = 24, 5
    N = Q * world
    if tied:       # a handful of distinct vectors and exact small values: long runs of equal entries, exact zeros
        base = rng.integers(-2, 3, size=(4, D)).astype(np.float32) / 4
        x = base[rng.integers(0, 4, N)]
    else:
        x = rng.standard_normal((N, D)).astype(np.float32)
    lab = rng.integers(0, 5, N).astype(np.float32)
    S = (x.astype(np.float64)[rank * Q:(rank + 1) * Q] @ x.astype(np.float64).T).astype(np.float32)
    off = rank * Q
    compared = 0
    for region in (synth.GLOBAL, synth.LOCAL):
        for identsn, diffsn in zip(SNS, SNS[::-1]):
            ref = select_ref.relative_thresholds(S, lab[off:off + Q], lab, off, region, identsn, diffsn)
            for i in range(Q):
                s_list, d_list = _lists(S, lab, off, None if region == synth.GLOBAL else i)
                for got, raw, lst, sn in ((ref["posi"][i], ref["posi_raw"][i], s_list, identsn), (ref["nega"][i], ref["nega_raw"][i], d_list, diffsn)):
                    want = _sorted_pick(lst, sn)
                    if want is None:
                        assert np.isnan(raw)
                        continue
                    assert raw == want
                    assert got == (want if want >= 0 else -select_ref.FLT_MAX)
            # the C++ oracle on the same S (where both sides are in range)
            if any(select_ref.pos(sn, n) is None for sn, n in ((identsn, _lists(S, lab, off)[0].size), (diffsn, _lists(S, lab, off)[1].size))):
                continue
            if region == synth.LOCAL and any(select_ref.pos(sn, l.size) is None for i in range(Q)
                                             for sn, l in zip((identsn, diffsn), _lists(S, lab, off, i))):
                continue
            cfg = oracle.make_config(Q, D, world=world, rank=rank, faithful_sorts=0, identsn=identsn, diffsn=diffsn, ap_region=region,
                                     ap_method=synth.RELATIVE_HARD, an_region=region, an_method=synth.RELATIVE_EASY)
            _, st = oracle.forward(x, lab, cfg, S_inject=S)
            np.testing.assert_array_equal(ref["posi"], st["posi_thr"])
            np.testing.assert_array_equal(ref["nega"], st["nega_thr"])
            compared += 1
    assert compared >= 8, compared


def test_pos_matches_oracle_around_2_pow_24():
    sizes = [1, 2, 3, 1000] + [(1 << e) + d for e in (24, 25, 26) for d in (-3, -2, -1, 0, 1, 2, 3)] + [67092480, 8192 * 8190]
    for size in sizes:
        for sn in (-0.3, -0.45, -0.5, -0.97, -1e-7, -0.0, 0.0, 0.9, 1.0, 3.0, 1000.0, 1e6, -1.0, -1.5):
            got = select_ref.pos(sn, size)
            want = oracle_pos(sn, size)
            assert (got if got is not None else -1) == want, (sn, size, got, want)
    assert select_ref.pos(-0.3, 8192 * 8190) == 46964736       # exact arithmetic gives 46 964 735


def oracle_pos(sn, size):
    from oracle import oracle_lib
    p = oracle_lib.pos(sn, size)
    return p if 0 <= p < size else -1


@pytest.mark.parametrize("Q,world", [(1024, 1), (512, 2), (8192, 1), (4608, 2), (100, 3), (16384, 1), (8192, 4)])
def test_gcand_cap_matches_the_library(Q, world):
    """A GLOBAL general-SN select allocates two candidate lists of gcand_cap 4-byte entries; SN = -0.0 (the list's maximum, a closed
    form) allocates none.  (16384, 1) and (8192, 4) reach the absolute cap of 32 Mi entries."""
    L = capi.lib()

    def ws(identsn, diffsn):
        cfg = capi.make_config(Q, 64, world=world, identsn=identsn, diffsn=diffsn, ap_region=capi.GLOBAL, ap_method=capi.RELATIVE_HARD,
                               an_region=capi.GLOBAL, an_method=capi.RELATIVE_EASY)
        n = L.npair_workspace_bytes(C.byref(cfg))
        assert n > 0
        return n

    closed = ws(-0.0, -0.0)
    assert ws(-0.3, -0.3) - closed == 8 * select_ref.gcand_cap(Q, Q * world)
    assert ws(-0.3, -0.0) - closed == 8 * select_ref.gcand_cap(Q, Q * world)      # one general-SN side allocates both lists
    assert ws(5.0, -0.0) - closed == 8 * select_ref.gcand_cap(Q, Q * world)


def test_bucket_of_rank_walks_value_order():
    """Buckets of negative floats come in descending raw digit: the bucket found for every rank holds the value at that rank."""
    rng = np.random.default_rng(8)
    vals = np.concatenate([rng.standard_normal(3000), [0.0, 0.5, 0.25, -0.5, 1.0]]).astype(np.float32) * np.float32(3.0)
    s = np.sort(vals)
    for bits in (10, 11):
        for p in range(0, s.size, 7):
            raw, pop = select_ref.bucket_of_rank(vals, p, bits)
            assert int(s[p:p + 1].view(np.uint32)[0] >> (32 - bits)) == raw
            assert pop == int(((vals.view(np.uint32) >> (32 - bits)) == raw).sum())
