"""CPU check of the device sampler's uniforms (include/valle_b200.h vb_sample_logits): for every one of the 2^23 values
m = h >> 41 of the hash, the fp32 arithmetic of the kernel, u = (m + 0.5) * 2^-23, must give exactly the real number
(2m + 1) / 2^24, strictly inside (0, 1), and a finite Gumbel value g = -log(-log(u)) within the bounds DESIGN states."""
import numpy as np


def test_every_uniform_is_exact_inside_the_unit_interval_and_its_gumbel_value_finite():
    m = np.arange(1 << 23, dtype=np.int64)
    u = (m.astype(np.float32) + np.float32(0.5)) * np.float32(2.0 ** -23)
    assert u.dtype == np.float32
    exact = (2 * m + 1).astype(np.float64) / float(1 << 24)             # the real value, exact in float64
    assert np.array_equal(u.astype(np.float64), exact)                  # no rounding: the 2^-24 grid, odd multiples
    assert float(u.min()) == 2.0 ** -24 and float(u.max()) == 1.0 - 2.0 ** -24
    assert bool((u > 0).all()) and bool((u < 1).all())
    g = -np.log(-np.log(u))
    assert bool(np.isfinite(g).all())
    assert -2.82 < float(g.min()) < -2.81 and 16.63 < float(g.max()) < 16.64


def test_a_24_bit_uniform_would_reach_one():
    """why the uniform has 23 bits: with 24, (2^24 - 1) + 0.5 needs a 25-bit significand and rounds up to 2^24"""
    top = (np.float32((1 << 24) - 1) + np.float32(0.5)) * np.float32(2.0 ** -24)
    assert top == np.float32(1.0)
