"""CPU model of the value-bin map of local_select_block_kernel (npairloss_b200/csrc/select.cu, lsb_off): bin*4 is read from the mantissa of
fmaf(s, s4, c0) with s4 = 4*2048/(hi-lo), c0 = fmaf(-lo, s4, 2^23 + 4).  The kernel relies on three properties of that map, checked
here in float32 arithmetic for many value ranges: it is monotone in s, every s in [lo, hi] lands inside the 2304 bins the find walks
, and NaN (an excluded entry) lands in bin 4095.  Ranges for which the kernel's own guard (`map_ok`) rejects the
map are skipped the way the kernel skips them (it falls back to key digits)."""
import numpy as np

BINS, HIST = 2048, 2304


def fma32(a, b, c):
    # one rounding: the product of two float32 is exact in float64; the float64 sum is rounded once more to float32 (a double
    # rounding that can differ from a true fma by one ulp in rare ties -- irrelevant to monotonicity and range)
    return (a.astype(np.float64) * np.float64(b) + np.float64(c)).astype(np.float32)


def off_of(s, s4, c0):
    bits = fma32(s, s4, c0).view(np.uint32)
    return bits & np.uint32(0x3FFC)


def map_of(lo, hi):
    lo, hi = np.float32(lo), np.float32(hi)
    s4 = np.float32(np.float32(4.0 * BINS) / np.float32(hi - lo))
    c0 = fma32(np.array([-lo], np.float32), s4, np.float32(8388612.0))[0]
    o_lo = fma32(np.array([lo], np.float32), s4, c0).view(np.uint32)[0]
    o_hi = fma32(np.array([hi], np.float32), s4, c0).view(np.uint32)[0]
    ok = hi > lo and o_lo >= 0x4B000000 and o_hi >= o_lo and o_hi < 0x4B000000 + 4 * (HIST - 1)
    return s4, c0, bool(ok)


def test_value_bins_are_monotone_and_in_range():
    rng = np.random.default_rng(20171225)
    checked = 0
    for trial in range(400):
        kind = trial % 4
        if kind == 0:      # cosine similarities
            lo, hi = sorted(rng.uniform(-1, 1, 2))
        elif kind == 1:    # narrow range away from zero
            c = rng.uniform(-3, 3); w = 10.0 ** rng.uniform(-4, -1); lo, hi = c - w, c + w
        elif kind == 2:    # un-normalised features: large magnitudes
            lo, hi = sorted(rng.normal(0, 10.0 ** rng.uniform(0, 6), 2))
        else:              # straddling zero with tiny values
            lo, hi = -10.0 ** rng.uniform(-8, 0), 10.0 ** rng.uniform(-8, 0)
        lo, hi = np.float32(lo), np.float32(hi)
        if not hi > lo:
            continue
        s4, c0, ok = map_of(lo, hi)
        if not ok:
            continue
        s = np.sort(rng.uniform(lo, hi, 4096).astype(np.float32))
        s = np.clip(s, lo, hi)
        s[0], s[-1] = lo, hi
        off = off_of(s, s4, c0).astype(np.int64)
        assert np.all(np.diff(off) >= 0), (lo, hi)
        assert off.min() >= 0 and off.max() < 4 * HIST, (lo, hi, off.min(), off.max())
        checked += 1
    assert checked > 250            # the guard may reject extreme ranges, not the ordinary ones


def test_nan_goes_to_the_bin_nobody_reads():
    s4, c0, ok = map_of(-0.4, 0.7)
    assert ok
    nan = np.array([np.uint32(0x7FFFFFFF)], np.uint32).view(np.float32)
    assert int(off_of(nan, s4, c0)[0]) == 0x3FFC == 4 * 4095


def test_ranges_far_from_zero_are_rejected_not_mis_binned():
    # |lo| * s4 beyond 2^23: c0 loses its integer grid; the guard must say so (the kernel then refines by key digits)
    s4, c0, ok = map_of(1000.0, 1000.001)
    lo, hi = np.float32(1000.0), np.float32(1000.001)
    if ok:      # if the guard accepts it, the map must still be sound on this range
        s = np.sort(np.random.default_rng(1).uniform(lo, hi, 1024).astype(np.float32))
        off = off_of(np.clip(s, lo, hi), s4, c0).astype(np.int64)
        assert np.all(np.diff(off) >= 0) and off.min() >= 0 and off.max() < 4 * HIST
