"""k_match_topk decides "all four depths in front of the cameras" (REF_GPU, top-k and count) with depths_in_front
(line3dpp_b200/csrc/l3d_device.cuh): a sign test on each depth's numerator and denominator instead of the IEEE division
exact_depths performs.  These tests check, in numpy float32 (IEEE-rounded division, denormals kept), that the two decisions agree
on the domain the kernel feeds them: |dp| >= L3D_EPS_F (smaller ones are rejected by both) and |dp| <= 1 + 1e-6 (dot products of
unit vectors normalised with rsqrtf), and on the numerators and denominators of real view pairs of a golden fixture."""
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "ref_kernels_v1.npz")
EPS = np.float32(1e-12)            # L3D_EPS_F
f32 = np.float32


def by_division(num, dp):
    """exact_depths' decision for one depth: -1 when |dp| < eps, else num / dp, then > 0"""
    with np.errstate(all="ignore"):
        return ~(np.abs(dp) < EPS) & (num / dp > f32(0))


def by_sign(num, dp):
    """depths_in_front's decision for one depth"""
    return ~(np.abs(dp) < EPS) & (((num > 0) & (dp > 0)) | ((num < 0) & (dp < 0)))


def grid(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.repeat(a, b.size), np.tile(b, a.size)


def test_adversarial_pairs():
    tiny = f32(np.finfo(np.float32).smallest_subnormal)
    one_up, one_dn = np.nextafter(f32(1), f32(2)), np.nextafter(f32(1), f32(0))
    mags = [0.0, tiny, 2 * tiny, 3 * tiny, np.finfo(np.float32).tiny, 1e-30, 1e-12, 1.0, 3e38, np.finfo(np.float32).max, np.inf]
    nums = [s * m for m in mags for s in (1.0, -1.0)] + [np.nan]
    dmags = [0.0, tiny, 1e-13, np.nextafter(EPS, f32(0)), EPS, np.nextafter(EPS, f32(1)), 1e-6, 0.5, one_dn, 1.0, one_up,
             f32(1 + 1e-6)]
    dps = [s * m for m in dmags for s in (1.0, -1.0)] + [np.nan]
    num, dp = grid(nums, dps)
    np.testing.assert_array_equal(by_sign(num, dp), by_division(num, dp))
    # the bound on |dp| is what makes the sign test exact: the smallest denormal numerator over 2 rounds to +0
    num, dp = f32(tiny), f32(2.0)
    assert by_sign(num, dp) and not by_division(num, dp)


def test_random_bit_patterns():
    rng = np.random.default_rng(7)
    n = 1 << 20
    num = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32).view(np.float32)      # every exponent, denormals, inf, NaN
    mag = np.exp(rng.uniform(np.log(1e-12), np.log(1 + 1e-6), n)).astype(np.float32)
    mag = np.clip(mag, EPS, f32(1 + 1e-6))
    dp = np.where(rng.integers(0, 2, n) == 1, mag, -mag).astype(np.float32)
    np.testing.assert_array_equal(by_sign(num, dp), by_division(num, dp))
    small = rng.integers(1, 1 << 12, n, dtype=np.uint32).view(np.float32)                       # the smallest denormals
    small = np.where(rng.integers(0, 2, n) == 1, small, -small).astype(np.float32)
    np.testing.assert_array_equal(by_sign(small, dp), by_division(small, dp))


def _rays(R, segs):
    """the float ray cache of k_prep_segments (r1, r2, n), restated in numpy float32 (1 / sqrt in place of rsqrtf)"""
    def mul(x, y):
        return np.stack([(R[3 * i] * x + R[3 * i + 1] * y) + R[3 * i + 2] for i in range(3)], -1).astype(np.float32)

    def nrm(v):
        return (v * (f32(1) / np.sqrt((v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2]))[:, None]).astype(np.float32)

    r1, r2 = nrm(mul(segs[:, 0], segs[:, 1])), nrm(mul(segs[:, 2], segs[:, 3]))
    return r1, r2, nrm(np.cross(r1, r2).astype(np.float32))


def _dot(a, b):
    return ((a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]).astype(np.float32)


def test_golden_pairs():
    z = np.load(GOLD)
    segs = z["segs"].astype(np.float32)
    checked = 0
    for p in ("p01", "p24"):
        s, t = int(p[1]), int(p[2])
        Cs, Ct = z[f"{p}_Cs"].astype(np.float32), z[f"{p}_Ct"].astype(np.float32)
        s1, s2, sn = _rays(z[f"{p}_Rs"].astype(np.float32), segs[s])
        t1, t2, tn = _rays(z[f"{p}_Rt"].astype(np.float32), segs[t])
        num_t = (_dot(Ct, tn) - _dot(tn, Cs)).astype(np.float32)                # depth_num(t.n, Ct, Cs), per target
        num_s = (_dot(Cs, sn) - _dot(sn, Ct)).astype(np.float32)                # depth_num(s.n, Cs, Ct), per source row
        S, T = s1.shape[0], t1.shape[0]
        pairs = [(np.broadcast_to(num_t[None, :], (S, T)), _dot(tn[None, :, :], s1[:, None, :])),
                 (np.broadcast_to(num_t[None, :], (S, T)), _dot(tn[None, :, :], s2[:, None, :])),
                 (np.broadcast_to(num_s[:, None], (S, T)), _dot(sn[:, None, :], t1[None, :, :])),
                 (np.broadcast_to(num_s[:, None], (S, T)), _dot(sn[:, None, :], t2[None, :, :]))]
        for num, dp in pairs:
            assert np.all(np.abs(dp[np.isfinite(dp)]) <= 1 + 1e-6)
            np.testing.assert_array_equal(by_sign(num, dp), by_division(num, dp))
            checked += num.size
        front = np.logical_and.reduce([by_division(n, d) for n, d in pairs])
        assert 0 < front.sum() < front.size                                      # both outcomes occur
    assert checked == 2 * 4 * 160 * 160
