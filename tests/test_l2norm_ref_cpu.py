"""Is l2norm_ref strong enough?  (no GPU)

An fp32 CPU emulation of l2norm_fwd_kernel / l2norm_bwd_kernel in their documented order (lane partial sums by fmaf, the 5-level
xor shuffle tree, sqrtf, IEEE division; the rescue pass on x 2^-e) meets the rules of l2norm_ref on adversarial rows and comes
within a stated factor of them, so the bounds are not vacuous; and the rules flag each planted fault of that emulation
(l2norm_ref.emulate_forward / emulate_backward, which test_gpu_l2norm_precision.py also holds the kernels to bit for bit)."""
import math

import numpy as np
import pytest

import l2norm_ref as ref

F32, F64 = np.float32, np.float64


# ---------------------------------------------------------------------------------------------------------------------------------
def _gauss(R, D, seed):
    return np.random.default_rng(seed).standard_normal((R, D)).astype(F32)


def _adversarial(D):
    """Every lane's first term is 1 and every later square just over half an ulp of 1: each fmaf rounds up by almost u."""
    x = np.full((1, D), F32(np.sqrt(2.0 ** -24 * (1 + 2.0 ** -10))), F32)
    first = np.arange(0, min(D, 128), 4) if D % 4 == 0 else np.arange(min(D, 32))
    x[0, first] = 1
    return x


def _range_rows(D, seed):
    """One Gaussian row at 2^k for k across the range the parent kernel got wrong, spikes, subnormals, zero rows."""
    g = _gauss(1, D, seed)[0]
    rows = [np.ldexp(g, k).astype(F32) for k in (0, -60, -62, -68, -72, -80, -120, 60, 62, 64, 100)]
    for e in (-149, -140, -126, -64, 0, 64, 127):
        s = np.zeros(D, F32); s[D // 2] = np.ldexp(F32(1.5) if e < 127 else F32(1.0), e); rows.append(s)
    rows.append(np.full(D, np.ldexp(F32(1.0), -149), F32))
    rows.append(np.full(D, np.ldexp(F32(1.75), 127), F32))
    rows.append(np.zeros(D, F32))
    rows.append(-np.zeros(D, F32))
    return np.stack(rows)


DS = [1, 3, 4, 5, 31, 32, 33, 127, 128, 129, 200, 512, 1024, 4095, 4096, 8192]


def test_reference_matches_python_loops():
    rng = np.random.default_rng(1)
    x = np.concatenate([_gauss(3, 37, 2), np.ldexp(_gauss(2, 37, 3), 120), np.ldexp(_gauss(2, 37, 4), -140)]).astype(F32)
    dy = rng.standard_normal(x.shape).astype(F32)
    y64, inv64 = ref.forward(x)
    for r in range(x.shape[0]):
        row = [float(v) for v in x[r]]
        n = math.sqrt(math.fsum(v * v for v in row))
        assert abs(inv64[r] - 1 / n) <= 4e-16 / n
        for d in range(x.shape[1]):
            assert abs(y64[r, d] - row[d] / n) <= 4e-16 * abs(row[d] / n)
    y, inv = ref.emulate_forward(x)
    dx64, B, _ = ref.backward(y, inv, dy)
    for r in range(x.shape[0]):
        yr, gr, iv = [float(v) for v in y[r]], [float(v) for v in dy[r]], float(inv[r])
        if not math.isfinite(iv):                                          # ||x|| < 2^-128: the +inf rule, tested below
            continue
        dot = math.fsum(a * b for a, b in zip(yr, gr))
        mag = math.fsum(abs(a * b) for a, b in zip(yr, gr))
        for d in range(x.shape[1]):
            want = (gr[d] - yr[d] * dot) * iv
            assert abs(dx64[r, d] - want) <= 1e-13 * abs(B[r, d])
            assert abs(B[r, d] - (abs(gr[d]) + abs(yr[d]) * mag) * iv) <= 1e-15 * B[r, d]


def test_nonfinite_and_zero_rows_in_the_reference():
    x = _gauss(4, 9, 5)
    x[1, 3] = np.nan
    x[2, 0] = -np.inf
    x[3] = 0
    y, inv = ref.forward(x)
    assert np.isnan(y[1:3]).all() and np.isnan(inv[1:3]).all()
    assert not y[3].any() and inv[3] == 0 and np.isfinite(y[0]).all()


@pytest.mark.parametrize("D", DS)
def test_emulation_meets_the_bounds(D):
    x = np.concatenate([_gauss(9, D, D), _range_rows(D, D + 1), _adversarial(D)])
    y, inv = ref.emulate_forward(x)
    v, m = ref.check_forward(x, y, inv)
    assert not v, v
    dy = _gauss(x.shape[0], D, D + 2)
    dy[3] = y[3] * 3                                                      # dy along y: dx cancels to the rounding level
    dx = ref.emulate_backward(y, inv, dy)
    vb, mb = ref.check_backward(y, inv, dy, dx)
    assert not vb, vb
    fin = np.isfinite(x).all(axis=1)
    vc, mc = ref.check_chain(x[fin], dy[fin], dx[fin])
    assert not vc, vc


@pytest.mark.parametrize("D", [1024, 4095, 8192])
def test_the_bounds_are_approached(D):
    """The adversarial rows reach more than half of tau_f and tau_b: the bounds are within a factor 2 of the worst case."""
    x = _adversarial(D)
    y, inv = ref.emulate_forward(x)
    _, m = ref.check_forward(x, y, inv)
    assert m["y"] >= 0.5 and m["inv"] >= 0.5, m
    yy = np.full((1, D), F32(2.0 ** -12), F32)
    gg = np.full((1, D), F32(2.0 ** -12 * (1 + 2.0 ** -10)), F32)
    first = np.arange(0, min(D, 128), 4) if D % 4 == 0 else np.arange(min(D, 32))
    yy[0, first] = gg[0, first] = 1
    inv1 = np.ones(1, F32)
    _, mb = ref.check_backward(yy, inv1, gg, ref.emulate_backward(yy, inv1, gg))
    assert mb >= 0.5, mb


def test_nonfinite_rows_leave_the_others_unchanged():
    x = _gauss(16, 200, 7)
    y0, i0 = ref.emulate_forward(x)
    x[5, 17] = np.nan
    x[9, 0] = np.inf
    x[12] = -np.inf
    y, inv = ref.emulate_forward(x)
    keep = np.ones(16, bool); keep[[5, 9, 12]] = False
    assert np.array_equal(y[keep].view(np.int32), y0[keep].view(np.int32))
    assert np.isnan(y[~keep]).all() and np.isnan(inv[~keep]).all()
    assert np.isnan(ref.emulate_backward(y, inv, _gauss(16, 200, 8))[~keep]).all()


def test_tiny_rows_give_inf_inv_and_no_nan_gradient():
    x = np.zeros((2, 64), F32)
    x[0, :3] = np.ldexp(F32(1.0), -140)
    x[1, 5] = np.ldexp(F32(1.0), -149)
    y, inv = ref.emulate_forward(x)
    assert (inv == np.inf).all()
    dy = np.zeros_like(x); dy[:, 1] = 1; dy[0, 0] = 1; dy[0, 1] = 1
    dx = ref.emulate_backward(y, inv, dy)
    assert not np.isnan(dx).any()
    assert not ref.check_backward(y, inv, dy, dx)[0]


FAULTS = {
    "drop_last_quad": ([200, 4095 - 3, 8192 + 64], "forward"),
    "skip_shuffle_level": ([33, 512, 8192], "forward"),
    "scalar_reads_d_plus_1": ([3, 33, 129, 4095], "forward"),
    "neighbour_norm": ([4, 129, 512], "forward"),
    "dot_missing_quad": ([128, 200, 4096], "backward"),
    "rescue_scales_ss_only": ([32, 129, 512], "forward"),
    "no_rescue": ([32, 129, 512], "forward"),           # the parent kernel: silent zero rows and subnormal loss at both ends
}


@pytest.mark.parametrize("fault", sorted(FAULTS))
def test_planted_faults_are_flagged(fault):
    Ds, which = FAULTS[fault]
    for D in Ds:
        x = np.concatenate([_gauss(8, D, D), _range_rows(D, D + 1)])
        if fault == "neighbour_norm":                    # rows 2r and 2r + 1 of one block of 8 differ in norm
            x = x[:8] * np.arange(1, 9, dtype=F32)[:, None]
        if which == "forward":
            y, inv = ref.emulate_forward(x, fault)
            v, _ = ref.check_forward(x, y, inv)
            if not v:
                dy = _gauss(x.shape[0], D, 3)
                v = ref.check_chain(x, dy, ref.emulate_backward(y, inv, dy))[0]
        else:
            y, inv = ref.emulate_forward(x)
            dy = _gauss(x.shape[0], D, 4)
            v, _ = ref.check_backward(y, inv, dy, ref.emulate_backward(y, inv, dy, fault))
        assert v, f"{fault} not flagged at D = {D}"


@pytest.mark.parametrize("D", [1, 3, 33, 128, 200])
def test_oracle_meets_the_rules_over_the_whole_range(oracle, D):
    """npo_l2normalize_forward / _backward: the same rules, the same non-finite and +inf conventions as the kernel."""
    x = np.concatenate([_gauss(9, D, D), _range_rows(D, D + 1), _adversarial(D)])
    x[2, 0] = np.nan
    x[4, -1] = -np.inf
    y, inv = oracle.l2normalize_forward(x)
    v, _ = ref.check_forward(x, y, inv)
    assert not v, v
    dy = _gauss(x.shape[0], D, D + 2)
    dx = oracle.l2normalize_backward(y, inv, dy)
    vb, _ = ref.check_backward(y, inv, dy, dx)
    assert not vb, vb


def test_fma_is_rounded_once():
    """The emulation's fmaf against the exactly rounded a b + c (Fractions), on operands whose sums land on fp32 midpoints."""
    from fractions import Fraction
    rng = np.random.default_rng(11)
    n = 4000
    a = np.ldexp(rng.uniform(1, 2, n), rng.integers(-20, 20, n)).astype(F32)
    b = np.ldexp(rng.uniform(1, 2, n), rng.integers(-20, 20, n)).astype(F32)
    c = np.ldexp(rng.uniform(-2, 2, n), rng.integers(-40, 40, n)).astype(F32)
    # a b = c' exactly plus a tiny tail: p + c within one fp32 half-ulp step of a midpoint
    c[: n // 2] = (-(a[: n // 2].astype(F64) * b[: n // 2]) + np.ldexp(1.5, rng.integers(-30, 0, n // 2))).astype(F32)
    got = ref._fma(a, b, c)
    for i in range(n):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        r = np.float32(float(exact))
        best = min((r, np.nextafter(r, F32(np.inf)), np.nextafter(r, F32(-np.inf))),
                   key=lambda v: (abs(Fraction(float(v)) - exact), int(np.array(v).view(np.uint32)) & 1))
        assert got[i] == best or (got[i] == 0 and best == 0), (i, got[i], best)
