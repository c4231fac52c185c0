"""Split TF32 ("tf32x3") on the dense decoder convs, without a GPU.

An fp32 plan with ``tf32x3`` = 1 runs every CONV, DECONV and UPCONV stage as three TF32 products per term
(tests/test_tf32x3_cpu.py derives the per-product bound 3*2^-22).  A dense stage sums far more terms than a pointwise
conv: 25 * 1024 for a 5x5 stage of 1024 channels, 25 * 1024 in the largest phase of a 9x9 DECONV.  The interval references
``dense_ref.conv`` / ``convt_ref.convt`` hold these stages to EPS_CONV_TF32X3 = 2 EPS_CONV + 2^-20 per |term|: 2^-20 for the
products, and twice the fp32 sum allowance because the tensor core's accumulator takes six times as many updates (three
k8 MMAs per 8 channels against one k16 MMA per 16) and on the H100 EPS_CONV alone did not cover the longest sums (DESIGN
section 3.7b).  Here a numpy emulation of the split at those full lengths lies inside that interval, and a single TF32
product per term falls outside.  Also the planner's split-TF32 plans of every dense
decoder stage, and the module routing of CPU tensors."""
import ctypes

import numpy as np
import pytest
import torch

import convt_ref as cr
import dense_ref as dr
from fastdepth_b200 import _lib
from oracle import stage_ref as sr
from test_tf32x3_cpu import rna_tf32, split

EPS_CONV_TF32X3 = 2 * dr.EPS_CONV + 2.0 ** -20
STAGES = ((1024, 512), (512, 256), (256, 128), (128, 64), (64, 32))
KINDS = [(dr.CONV, 5), (dr.CONV, 3), (cr.DECONV, 3), (cr.DECONV, 5), (cr.DECONV, 7), (cr.DECONV, 9), (cr.UPCONV, 5)]
KIDS = ['nnconv5', 'nnconv3', 'deconv3', 'deconv5', 'deconv7', 'deconv9', 'upconv5']


# ---------------------------------------------------------------------------------------------------------------------
# numerics at full length
# ---------------------------------------------------------------------------------------------------------------------
def _emulate_conv(x, w, scale, bias, act, three):
    """Stride-1 'same' conv of NHWC fp32 ``x`` with [c_out][c_in][k][k] fp32 ``w``: every product formed from TF32 parts
    (``three``: a_lo b_hi + a_hi b_lo + a_hi b_hi, else a_hi b_hi), summed in fp64 (each product is exact in fp64; the
    sum's own error, below 2^-40 of the term magnitudes, is far inside the allowance), then the fp32 affine and act."""
    k = w.shape[-1]
    p = (k - 1) // 2
    xp = np.pad(x, ((0, 0), (p, p), (p, p), (0, 0)))
    xh, xl = (t.astype(np.float64) for t in split(xp))
    wh, wl = (t.astype(np.float64) for t in split(w))
    if not three:
        xh, wh = rna_tf32(xp).astype(np.float64), rna_tf32(w).astype(np.float64)
    n, h, wd, _ = x.shape
    acc = np.zeros((n, h, wd, w.shape[0]))
    for ky in range(k):
        for kx in range(k):
            sl = (slice(None), slice(ky, ky + h), slice(kx, kx + wd))
            bh, bl = wh[:, :, ky, kx].T, wl[:, :, ky, kx].T
            acc += xh[sl] @ bh
            if three:
                acc += xl[sl] @ bh + xh[sl] @ bl
    y = np.maximum(acc.astype(np.float32) * scale + bias, np.float32(0.0))
    if act == sr.RELU6:
        y = np.minimum(y, np.float32(6.0))
    return y.astype(np.float32)


def _calibrated(x, w, k, act, rng):
    """BN scale / bias that put about a third of the outputs below zero and, for ReLU6, clamp a tail (as the GPU sweeps
    calibrate their stages)."""
    pre = dr.conv(sr.exact(x), w, np.ones(w.shape[0]), np.zeros(w.shape[0]), k, None).c
    m, s = pre.mean(axis=(0, 1, 2)), pre.std(axis=(0, 1, 2)) + 1e-6
    tgt = rng.uniform(0.8, 1.2, w.shape[0]) * (2.2 if act == sr.RELU6 else 1.0)
    scale = (tgt / s).astype(np.float32)
    return scale, (0.5 * tgt - m * scale.astype(np.float64)).astype(np.float32)


def _check_admits_three_rejects_one(x, w_conv, iv, scale, bias, act, what):
    got3 = _emulate_conv(x, w_conv, scale, bias, act, True)
    sr.check(got3, iv, 'float32', 'split tf32 ' + what)
    assert (got3 == 0).mean() < 0.5
    got1 = _emulate_conv(x, w_conv, scale, bias, act, False)
    with pytest.raises(AssertionError, match='outside the reference'):
        sr.check(got1, iv, 'float32', 'single tf32 ' + what)


def test_conv5_stage_of_1024_channels():
    """A 5x5 1024 -> 512 CONV stage: 25 600 terms per output."""
    rng = np.random.default_rng(5)
    x = np.maximum(rng.standard_normal((2, 5, 6, 1024)) + 0.5, 0.0).astype(np.float32)
    w = (rng.uniform(-1, 1, (512, 1024, 5, 5)) * np.sqrt(3.0 / 25600)).astype(np.float32)
    scale, bias = _calibrated(x, w, 5, sr.RELU, rng)
    iv = dr.conv(sr.exact(x), w, scale, bias, 5, sr.RELU, eps=EPS_CONV_TF32X3)
    _check_admits_three_rejects_one(x, w, iv, scale, bias, sr.RELU, 'conv5 1024x512')
    assert np.all(dr.conv(sr.exact(x), w, scale, bias, 5, sr.RELU).r <= iv.r)


def test_deconv9_phase_of_1024_channels():
    """A 9x9 DECONV stage of 1024 input channels: phase (0, 0) sums 5 x 5 taps x 1024 channels.  The split is emulated
    on the equivalent stride-1 conv of the zero-inserted input, whose inserted zeros add exactly nothing."""
    rng = np.random.default_rng(9)
    ci, co, k = 1024, 64, 9
    x = np.maximum(rng.standard_normal((1, 3, 4, ci)) + 0.5, 0.0).astype(np.float32)
    w = (rng.uniform(-1, 1, (ci, co, k, k)) * np.sqrt(3.0 / (ci * k * k / 4.0))).astype(np.float32)
    assert max(len(cr.phase_taps(cr.DECONV, k, r)) for r in (0, 1)) ** 2 * ci == 25 * 1024
    wc = cr.conv_weights(cr.DECONV, w, ci, co, k).astype(np.float32)       # exact: a permutation of fp32 values
    up = np.zeros((1, 6, 8, ci), np.float32)
    up[:, ::2, ::2] = x
    scale, bias = _calibrated(up, wc, k, sr.RELU6, rng)
    iv = cr.convt(sr.exact(x), w, scale, bias, cr.DECONV, k, sr.RELU6, eps=EPS_CONV_TF32X3)
    _check_admits_three_rejects_one(up, wc, iv, scale, bias, sr.RELU6, 'deconv9 1024x64')
    assert (_emulate_conv(up, wc, scale, bias, sr.RELU6, True) == 6).any()


# ---------------------------------------------------------------------------------------------------------------------
# the planner (host-only debug entry)
# ---------------------------------------------------------------------------------------------------------------------
KEYS = ('ok', 'ni', 'th', 'tw', 'bn', 'stages', 'm_tiles', 'n_splits', 'items', 'waves', 'kblocks', 'smem_bytes',
        'useful_permille', 'cost', 'stage_bytes', 'groups')


def tf32x3_plan(kind, k, h, w, n, ci, co, up=0, sms=132):
    out = (ctypes.c_int * 44)()
    _lib.check(_lib.load().fd_debug_conv_tf32x3_plan(kind, k, h, w, n, ci, co, up, sms, out, 44))
    q = dict(zip(KEYS, out[:16]))
    q['ph'] = [tuple(out[16 + 5 * p:21 + 5 * p]) for p in range(4)]
    q['group_ph'] = [tuple(out[36 + 2 * g:38 + 2 * g]) for g in range(4)]
    return q


def _check_plan(q, kind, k, h, w, n, ci, co):
    assert q['ok'] == 1, (kind, k, h, w, n, ci, co, q)
    assert q['bn'] in (64, 128)
    assert q['kblocks'] == -(-ci // 32)                      # 32 fp32 channels per 128-byte row
    assert q['stage_bytes'] == 128 * 128 + 2 * q['bn'] * 128
    assert q['stages'] == {64: 6, 128: 4}[q['bn']]           # the ring depth under the 227 KB budget
    assert q['stages'] * q['stage_bytes'] + 2 * 16384 <= q['smem_bytes'] <= 227 * 1024
    assert q['ni'] * q['th'] * q['tw'] == 128
    assert q['m_tiles'] == -(-n // q['ni']) * -(-h // q['th']) * -(-w // q['tw'])
    assert q['n_splits'] == -(-co // q['bn'])
    phased = kind != dr.CONV
    assert q['groups'] in ((2, 4) if phased else (1,))
    assert q['items'] == q['m_tiles'] * q['n_splits'] * q['groups']
    taps = sum(ny * nx for _, ny, nx, _, _ in q['ph'])
    assert taps == k * k                                     # the phases partition the k x k taps (CONV: one square)
    if not phased:
        assert q['ph'][0] == (0, k, k, -(k // 2), -(k // 2))


@pytest.mark.parametrize('kind,k', KINDS, ids=KIDS)
@pytest.mark.parametrize('n', [1, 64])
def test_plan_every_decoder_stage(built_lib, kind, k, n):
    h = w = 7
    for ci, co in STAGES:
        up = 1 if kind == dr.CONV else 0
        q = tf32x3_plan(kind, k, h, w, n, ci, co, up)
        _check_plan(q, kind, k, h, w, n, ci, co)
        h, w = 2 * h, 2 * w


@pytest.mark.parametrize('kind,k', KINDS, ids=KIDS)
def test_plan_channel_tails_and_small_maps(built_lib, kind, k):
    for h, w, n, ci, co in ((1, 1, 4, 40, 8), (1, 2, 3, 72, 136), (2, 3, 5, 264, 40), (7, 5, 2, 8, 264), (4, 4, 33, 520, 24)):
        _check_plan(tf32x3_plan(kind, k, h, w, n, ci, co, 1 if kind == dr.CONV else 0), kind, k, h, w, n, ci, co)


def test_plan_offers_both_bn_and_rejects_other_stages(built_lib):
    bns = {tf32x3_plan(kind, k, h, h, n, ci, co)['bn'] for kind, k in KINDS for n in (1, 64)
           for h, (ci, co) in zip((7, 14, 28, 56, 112), STAGES)}
    assert bns == {64, 128}, bns
    assert tf32x3_plan(dr.CONV, 7, 7, 7, 1, 64, 64)['ok'] == 0        # a 7x7 CONV is not a kernel target
    assert tf32x3_plan(cr.DECONV, 4, 7, 7, 1, 64, 64)['ok'] == 0
    assert tf32x3_plan(dr.CONV, 5, 7, 7, 1, 4, 64)['ok'] == 0          # c_in < 8
    out = (ctypes.c_int * 44)()
    with pytest.raises(RuntimeError, match='kind must be'):
        _lib.check(_lib.load().fd_debug_conv_tf32x3_plan(1, 3, 7, 7, 1, 64, 64, 0, 132, out, 44))
    with pytest.raises(RuntimeError, match='int\\[44\\]'):
        _lib.check(_lib.load().fd_debug_conv_tf32x3_plan(3, 3, 7, 7, 1, 64, 64, 0, 132, out, 16))


def test_pointwise_plan_unchanged(built_lib):
    """The 1x1 CONV through the new entry is the plan the pointwise step has always had."""
    pw = (ctypes.c_int * 16)()
    for shape in ((7, 7, 64, 1024, 1024, 0), (14, 14, 64, 512, 256, 1), (1, 2, 3, 24, 8, 1)):
        h, w, n, ci, co, up = shape
        _lib.check(_lib.load().fd_debug_pw_tf32x3_plan(h, w, n, ci, co, up, 132, pw, 16))
        q = tf32x3_plan(dr.CONV, 1, h, w, n, ci, co, up)
        assert [q[k] for k in KEYS[:15]] == list(pw[:15])
        assert q['groups'] == 1 and q['ph'][0] == (0, 1, 1, 0, 0)


# ---------------------------------------------------------------------------------------------------------------------
# routing of CPU tensors
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('decoder', ['nnconv5', 'nnconv3', 'deconv3', 'upconv', 'nnconv5dw'])
def test_cpu_tensors_never_build_an_engine(decoder):
    import models
    m = models.MobileNet(decoder, (64, 64), pretrained=False).eval()
    prev = torch.get_float32_matmul_precision()
    try:
        for prec in ('highest', 'high', 'medium'):
            torch.set_float32_matmul_precision(prec)
            with torch.no_grad():
                assert m(torch.rand(1, 3, 64, 64)).shape == (1, 1, 64, 64)
            assert '_fd_engine' not in m.__dict__, (decoder, prec)
    finally:
        torch.set_float32_matmul_precision(prev)
