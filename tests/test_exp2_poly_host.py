"""CPU: the FMA-pipe exponential of the attention kernels (`f2_exp2_poly`, csrc/sm90_common.cuh) restated in numpy float32
with the coefficients READ FROM THE HEADER, against exp2 in float64: the error bound the header states (1.0e-4 relative,
far below one bf16 ulp = 3.9e-3, which is all a softmax probability keeps), the exponent assembly for negative and positive
integer parts, the round-to-nearest split at half-integers, and the clamp.  The kernels themselves are checked on the GPU
by tests/test_gemm_attn_gpu.py: the attention forward element by element with the default MUFU exponential, and
test_attention_forward_poly_exponential runs the same checks with DPIPE_ATTN_FWD_POLY = 2 and 4, with the error bound
widened by the relative error this file checks."""
import os
import re

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _coefficients():
    src = open(os.path.join(ROOT, 'diffusion-pipe_b200', 'csrc', 'sm90_common.cuh')).read()
    body = src[src.index('f32x2 f2_exp2_poly(f32x2 x)'):]
    body = body[:body.index('\n}\n')]
    packs = [float(a) for a, b in re.findall(r'f2_pack\(([-0-9.e]+)f, ([-0-9.e]+)f\)', body)]
    magic, c3, c2, c1, c0 = packs
    clamp, clamp1 = (float(v) for v in re.search(r'fmaxf\(x0, ([-0-9.e]+)f\), fmaxf\(x1, ([-0-9.e]+)f\)', body).groups())
    assert clamp == clamp1
    assert clamp == -125.0 and magic == 12582912.0 and c0 == 1.0, packs
    return np.float32(clamp), np.float32(magic), [np.float32(c) for c in (c3, c2, c1, c0)]


def _fma(a, b, c):
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)    # one rounding, like FFMA


def exp2_poly(x):
    clamp, magic, (c3, c2, c1, c0) = _coefficients()
    x = np.maximum(x.astype(np.float32), clamp)
    t = (x + magic).astype(np.float32)
    n = (t - magic).astype(np.float32)
    f = (x - n).astype(np.float32)
    p = _fma(f, np.full_like(f, c3), np.full_like(f, c2))
    p = _fma(p, f, np.full_like(f, c1))
    p = _fma(p, f, np.full_like(f, c0))
    bits = p.view(np.uint32) + (t.view(np.uint32) << np.uint32(23))       # wraps mod 2^32 exactly like the device code
    return bits.view(np.float32), n, f


def test_polynomial_exp2_meets_its_stated_error_bound_on_the_softmax_range():
    rng = np.random.default_rng(0)
    x = np.concatenate([np.linspace(-125.0, 0.0, 2_000_001), -np.abs(rng.standard_normal(500_000)) * 8.0,
                        np.linspace(0.0, 20.0, 200_001)]).astype(np.float32)
    y, n, f = exp2_poly(x)
    ref = np.exp2(x.astype(np.float64))
    rel = np.abs(y.astype(np.float64) - ref) / ref
    assert rel.max() <= 1.05e-4, rel.max()
    assert np.abs(f).max() <= 0.5 and np.array_equal(n, np.round(n))
    assert (y[x <= 0] <= 1.0 + 1.05e-4).all() and (y > 0).all() and np.isfinite(y).all()
    assert rel.max() < 2.0 ** -8 / 30                                       # > 30x below one bf16 ulp (relative 2^-8)


def test_integer_part_goes_into_the_exponent_field_exactly():
    ints = np.arange(-125, 64, dtype=np.float32)
    y, n, f = exp2_poly(ints)
    assert np.array_equal(n, ints) and not f.any()
    assert np.array_equal(y, np.exp2(ints.astype(np.float64)).astype(np.float32))      # 2^n exactly, negative n included
    half = np.array([-2.5, -1.5, -0.5, 0.5, 1.5], dtype=np.float32)                   # ties: either neighbour, |f| = 0.5
    y, n, f = exp2_poly(half)
    assert np.array_equal(np.abs(f), np.full_like(f, 0.5))
    assert np.allclose(y, np.exp2(half.astype(np.float64)), rtol=1.05e-4)


def test_arguments_below_the_clamp_give_a_tiny_positive_number_not_garbage():
    x = np.array([-126.0, -200.0, -1e4, -3e38, -np.inf], dtype=np.float32)
    y, _, _ = exp2_poly(x)
    assert np.array_equal(y, np.full_like(y, np.float32(2.0 ** -125)))                 # invisible next to a row maximum of 2^0
