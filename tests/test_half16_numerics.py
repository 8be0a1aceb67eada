"""CPU check of the arithmetic behind MAGNET_SRC_HALF16 (DESIGN §3.7): an fp16 / bf16 feature map scaled by the
power-of-two s of the SPLIT16 rule (absmax * s in [2^14, 2^15)) is itself an fp16 number above a threshold, so the fp32
split of its upcast has a zero lo plane, the single plane is the split's hi plane, and the single hi*hi product equals
the three-product GEMM of tests/test_split16_numerics.py.  Restated in numpy, with torch's CPU bf16 / fp16 rounding."""
import numpy as np
import pytest
import torch

from tests.test_split16_numerics import split16


def half16(x):
    """The single plane of csrc/cost_mma.cu (split16_repack_kernel<T, 1>): fp16(x * s), s from the fp32 value of x."""
    xf = np.asarray(x, dtype=np.float32)
    _, _, s = split16(xf)
    return (xf * np.float32(s)).astype(np.float16), s


def _half_map(dt, scale, n=1 << 16, seed=0):
    x = torch.from_numpy(np.random.default_rng(seed).standard_normal(n).astype(np.float32) * np.float32(scale))
    return x.to(dt).float().numpy()


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("scale", [1e-3, 0.37, 1.0, 41.0, 1e3])
def test_scale_rule_and_exactness(dt, scale):
    x = _half_map(dt, scale)
    plane, s = half16(x)
    amax = np.abs(x).max()
    assert 2.0 ** 14 <= amax * s < 2.0 ** 15 and s == 2.0 ** round(np.log2(s))
    v = x.astype(np.float64) * s
    if dt == torch.float16:                                # absmax < 2^15: s >= 1, every element exact
        assert s >= 1.0 and np.array_equal(plane.astype(np.float64), v)
    else:                                                  # bf16: exact wherever |x| >= absmax 2^-31
        big = np.abs(x) >= amax * 2.0 ** -31
        assert np.array_equal(plane.astype(np.float64)[big], v[big])


def test_bf16_threshold_is_tight_and_elements_below_it_are_bounded():
    """bf16 elements at 2^-31 of absmax and just above: exact; far below: within the bound 2^-25 / s <= absmax 2^-39."""
    amax = np.float32(3.0)
    mant = np.float32(1.0 + 2.0 ** -7)                     # 8 significant bits: the bf16 worst case
    x = np.array([amax, mant * amax * np.float32(2.0 ** -31), mant * amax * np.float32(2.0 ** -36),
                  np.float32(amax * 2.0 ** -45), -mant * amax * np.float32(2.0 ** -33)], dtype=np.float32)
    x = torch.from_numpy(x).to(torch.bfloat16).float().numpy()
    plane, s = half16(x)
    rec = plane.astype(np.float64) / s
    err = np.abs(rec - x.astype(np.float64))
    assert err[0] == 0.0 and err[1] == 0.0                 # at the threshold: exact
    assert err[2] > 0.0                                    # below it the last bits run into fp16's subnormal step
    assert (err <= 2.0 ** -25 / s).all() and (err <= amax * 2.0 ** -39).all()


def test_fp16_near_65504():
    """absmax >= 2^15 gives s = 1/2: normal elements stay exact, subnormal ones may lose their last bit (within the
    bound)."""
    rng = np.random.default_rng(5)
    x = np.concatenate([np.float32([65504.0, -40000.0, 2.0 ** 15]), rng.standard_normal(4096).astype(np.float32),
                        (rng.standard_normal(256) * 2.0 ** -20).astype(np.float32)])
    x = torch.from_numpy(x).to(torch.float16).float().numpy()
    plane, s = half16(x)
    assert s == 0.5
    rec = plane.astype(np.float64) / s
    err = np.abs(rec - x.astype(np.float64))
    normal = np.abs(x) * s >= 2.0 ** -14
    assert (err[normal] == 0).all() and (err > 0).any()
    assert (err <= 2.0 ** -25 / s).all() and (err <= np.abs(x).max() * 2.0 ** -39).all()


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
def test_fp32_split_of_an_exact_map_has_zero_lo(dt):
    x = _half_map(dt, 7.0, seed=2)
    hi, lo, s = split16(x)
    plane, s1 = half16(x)
    assert s1 == s and not lo.astype(np.float32).any() and np.array_equal(hi, plane)


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
def test_single_product_equals_three_product_gemm(dt):
    """The window GEMM of the forward on HALF16 operands (hi*hi alone) against the SPLIT16 restatement of
    test_split16_numerics.py (lo*hi + hi*lo + hi*hi) on the upcast maps: equal, since both lo planes are zero."""
    rng = np.random.default_rng(3)
    a = torch.from_numpy(rng.standard_normal((512, 64)).astype(np.float32) * 3).to(dt).float().numpy()
    b = torch.from_numpy(rng.standard_normal((700, 64)).astype(np.float32) * 0.2).to(dt).float().numpy()
    ah, al, sa = split16(a)
    bh, bl, sb = split16(b)
    f = lambda t: t.astype(np.float64)
    three = (f(al) @ f(bh).T + f(ah) @ f(bl).T + f(ah) @ f(bh).T) / (sa * sb)
    pa, _ = half16(a)
    pb, _ = half16(b)
    one = (f(pa) @ f(pb).T) / (sa * sb)
    assert np.array_equal(one, three)
    assert np.abs(one - f(a) @ f(b).T).max() <= 1e-12 * (np.abs(f(a)) @ np.abs(f(b)).T).max()


def test_non_finite_half_elements_do_not_set_the_scale():
    x = torch.tensor([1.0, -3.0, float("inf"), float("nan"), 0.5], dtype=torch.float16).float().numpy()
    plane, s = half16(x)
    assert s == 2.0 ** 13
    assert np.isinf(plane[2]) and np.isnan(plane[3]) and float(plane[1]) == -3 * 2.0 ** 13
