"""Split-TF32 ("tf32x3") numerics and planning, without a GPU.

The fp32 pointwise convs of an fp32 plan with ``tf32x3`` = 1 run as three TF32 products per term:
a*b ~ a_lo*b_hi + a_hi*b_lo + a_hi*b_hi with a_hi = rna_tf32(a), a_lo = rna_tf32(a - a_hi) (round to nearest, ties away).
|a_lo| <= 2^-11 |a|, so the dropped a_lo*b_lo and the TF32 roundings of the two low parts leave |ab - sum3| <= 3*2^-22 |ab|,
and the kernel's result must lie in the fp32 interval of oracle/stage_ref.pointwise widened by 2^-20 per |term|.  Here a
numpy emulation shows that bound, that the widened interval admits the split and rejects a single TF32 product, and that the
planner's fp32 operand format fits shared memory."""
import ctypes

import numpy as np
import pytest

from oracle import stage_ref as sr

EPS_TF32X3 = sr.EPS + 2.0 ** -20


def rna_tf32(x):
    """fp32 -> TF32 (10 explicit significand bits), round to nearest with ties away from zero, as cvt.rna.tf32.f32."""
    u = np.asarray(x, np.float32).view(np.uint32).astype(np.uint64)
    u = ((u + 0x1000) & 0xFFFFE000).astype(np.uint32)
    return u.view(np.float32)


def split(x):
    x = np.asarray(x, np.float32)
    hi = rna_tf32(x)
    return hi, rna_tf32(x - hi)


def prod3(a, b):
    """The three products in fp64 (each exact: 11 x 11 significand bits)."""
    ah, al = (t.astype(np.float64) for t in split(a))
    bh, bl = (t.astype(np.float64) for t in split(b))
    return al * bh + ah * bl + ah * bh


def prod1(a, b):
    return rna_tf32(a).astype(np.float64) * rna_tf32(b).astype(np.float64)


def _wide(rng, n):
    """fp32 values over random signs, exponents (2^-30 .. 2^30) and significands."""
    return (rng.choice([-1.0, 1.0], n) * rng.uniform(1.0, 2.0, n) * 2.0 ** rng.integers(-30, 31, n)).astype(np.float32)


def test_rna_tf32_rounds_to_nearest_ties_away():
    one = np.float32(1.0)
    ulp = np.float32(2.0 ** -10)
    assert rna_tf32(one + ulp * np.float32(0.5)) == one + ulp           # tie: away from zero
    assert rna_tf32(-(one + ulp * np.float32(0.5))) == -(one + ulp)
    assert rna_tf32(one + ulp * np.float32(0.25)) == one
    x = _wide(np.random.default_rng(0), 100000)
    r = rna_tf32(x)
    assert np.all(r.view(np.uint32) & 0x1FFF == 0)
    assert np.all(np.abs(r.astype(np.float64) - x) <= 2.0 ** -11 * np.abs(x.astype(np.float64)))


def test_split_reconstructs_the_value():
    x = _wide(np.random.default_rng(1), 100000)
    hi, lo = split(x)
    xd = x.astype(np.float64)
    # |lo| <= 2^-11 |x|; lo loses at most its own TF32 rounding, 2^-11 |lo|
    assert np.all(np.abs(lo.astype(np.float64)) <= 2.0 ** -11 * np.abs(xd))
    assert np.all(np.abs(hi.astype(np.float64) + lo - xd) <= 2.0 ** -22 * np.abs(xd))
    # a value with at most 22 significant bits is split exactly
    y = rna_tf32(x).astype(np.float64) + rna_tf32(x * np.float32(2.0 ** -12)).astype(np.float64)
    y = y.astype(np.float32)
    yh, yl = split(y)
    assert np.array_equal(yh.astype(np.float64) + yl, y.astype(np.float64))


def test_three_products_meet_the_bound_and_one_does_not():
    rng = np.random.default_rng(2)
    a, b = _wide(rng, 200000), _wide(rng, 200000)
    exact = a.astype(np.float64) * b.astype(np.float64)
    err3 = np.abs(prod3(a, b) - exact) / np.abs(exact)
    err1 = np.abs(prod1(a, b) - exact) / np.abs(exact)
    assert err3.max() <= 3 * 2.0 ** -22 < 2.0 ** -20
    assert err1.max() > 2.0 ** -13 and (err1 > 2.0 ** -20).mean() > 0.9


def _layer(c_in, c_out, act, seed):
    """A pointwise layer on a live fp32 input (the depthwise intermediate it would read), BN calibrated as the kernel sweep
    calibrates it (test_kernel_sweep._bn: ~30 % zeros, ReLU6 clamping a tail)."""
    rng = np.random.default_rng(seed)
    x = np.maximum(rng.standard_normal((2, 6, 7, c_in)) + 0.5, 0.0).astype(np.float32)
    w = (rng.uniform(-1, 1, (c_out, c_in)) * np.sqrt(3.0 / c_in)).astype(np.float32)
    pre = x.astype(np.float64) @ w.T.astype(np.float64)
    m, s = pre.mean(axis=(0, 1, 2)), pre.std(axis=(0, 1, 2)) + 1e-6
    tgt_s = rng.uniform(0.8, 1.2, c_out) * (2.2 if act == sr.RELU6 else 1.0)
    scale = (tgt_s / s).astype(np.float32)
    bias = (0.5 * tgt_s - m * scale.astype(np.float64)).astype(np.float32)
    return x, w, scale, bias


def _emulate(x, w, scale, bias, act, prod):
    """The pointwise layer with every product formed by ``prod`` and summed exactly (fp64), then the affine, the act and one
    rounding to fp32."""
    acc = np.zeros(x.shape[:-1] + (w.shape[0],))
    for ci in range(x.shape[-1]):
        acc += prod(np.broadcast_to(x[..., ci:ci + 1], acc.shape), np.broadcast_to(w[:, ci], acc.shape))
    y = np.maximum(acc * scale.astype(np.float64) + bias, 0.0)
    if act == sr.RELU6:
        y = np.minimum(y, 6.0)
    return y.astype(np.float32)


@pytest.mark.parametrize('c_in,c_out,act', [(1024, 512, sr.RELU6), (64, 32, sr.RELU)])
def test_interval_admits_the_split_and_rejects_single_tf32(c_in, c_out, act):
    x, w, scale, bias = _layer(c_in, c_out, act, seed=c_in)
    iv = sr.pointwise(sr.exact(x), w, scale, bias, act, eps=EPS_TF32X3)
    got3 = _emulate(x, w, scale, bias, act, prod3)
    sr.check(got3, iv, 'float32', 'split tf32 %dx%d' % (c_in, c_out))
    assert (got3 == 0).mean() < 0.5
    # one TF32 product per term falls outside: the GPU check tells the two apart
    got1 = _emulate(x, w, scale, bias, act, prod1)
    with pytest.raises(AssertionError, match='outside the reference'):
        sr.check(got1, iv, 'float32', 'single tf32 %dx%d' % (c_in, c_out))
    # and the fp32 interval itself (sr.EPS, no allowance for the products) is what the widening adds to
    assert np.all(sr.pointwise(sr.exact(x), w, scale, bias, act).r <= iv.r)


# ---------------------------------------------------------------------------------------------------------------------
# the planner's fp32 operand format (host-only debug entry)
# ---------------------------------------------------------------------------------------------------------------------
SHAPES = [  # (h, w, n, c_in, c_out, upsample): MobileNet's pointwise convs at 224^2 (b1, b64) and the tails
    (112, 112, 1, 32, 64, 0), (56, 56, 64, 64, 128, 0), (14, 14, 64, 512, 512, 0), (7, 7, 64, 1024, 1024, 0),
    (7, 7, 1, 1024, 512, 1), (14, 14, 64, 512, 256, 1), (56, 56, 64, 128, 64, 1), (112, 112, 64, 64, 32, 1),
    (1, 1, 2, 72, 56, 1), (1, 2, 3, 24, 8, 1), (9, 11, 5, 40, 136, 0), (4, 4, 33, 264, 72, 1), (6, 6, 4, 16, 264, 0),
]


def _plan(built_lib, h, w, n, c_in, c_out, up, n_sms=132):
    from fastdepth_b200 import _lib
    lib = _lib.load()
    out = (ctypes.c_int * 16)()
    _lib.check(lib.fd_debug_pw_tf32x3_plan(h, w, n, c_in, c_out, up, n_sms, out, 16))
    keys = ('ok', 'ni', 'th', 'tw', 'bn', 'stages', 'm_tiles', 'n_splits', 'items', 'waves', 'kblocks', 'smem_bytes',
            'useful_permille', 'cost', 'stage_bytes')
    return dict(zip(keys, out))


@pytest.mark.parametrize('shape', SHAPES, ids=lambda s: 'x'.join(map(str, s)))
def test_tf32x3_plan_fits(built_lib, shape):
    h, w, n, c_in, c_out, up = shape
    q = _plan(built_lib, h, w, n, c_in, c_out, up)
    assert q['ok'] == 1
    assert q['bn'] in (64, 128)                              # bn 256 would exceed the register budget
    assert q['kblocks'] == (c_in + 31) // 32                 # 32 fp32 channels per 128-byte row
    assert q['stage_bytes'] == 128 * 128 + 2 * q['bn'] * 128
    assert q['stages'] >= 2
    assert q['smem_bytes'] <= 227 * 1024
    assert q['smem_bytes'] >= q['stages'] * q['stage_bytes'] + 2 * 16384
    assert q['ni'] * q['th'] * q['tw'] == 128
    assert q['n_splits'] == (c_out + q['bn'] - 1) // q['bn']
    assert q['items'] == q['m_tiles'] * q['n_splits']


def test_tf32x3_plan_ring_depths(built_lib):
    """16 KB of A + two bn x 128 B boxes per stage: bn 64 -> 6 stages, bn 128 -> 4, under the 227 KB budget."""
    from fastdepth_b200 import _lib
    depth = {}
    for shape in SHAPES:
        q = _plan(built_lib, *shape)
        depth.setdefault(q['bn'], set()).add(q['stages'])
    assert depth.get(64, {6}) == {6} and depth.get(128, {4}) == {4}, depth
    assert set(depth) == {64, 128}, depth
    out = (ctypes.c_int * 16)()
    lib = _lib.load()
    _lib.check(lib.fd_debug_pw_tf32x3_plan(7, 7, 1, 1024, 1024, 0, 132, out, 16))
    assert out[0] == 1
