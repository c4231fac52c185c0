"""oracle/stage_ref.py: the per-stage fp64 interval reference the kernel sweep (tests/test_kernel_sweep.py) checks against.

Pinned against the MobileNet oracle (fp64, and stage by stage with the product's storage roundings), its rounding helpers against numpy /
torch casts, and its checker against values it must accept and kernel mistakes it must reject.  CPU only."""
import numpy as np
import pytest
import torch

from conftest import rel_err, storage_emulated_forward
from fastdepth_b200 import plan as fplan
from fastdepth_b200 import synthetic
from oracle import fastdepth_oracle as orc
from oracle import stage_ref as sr


def _module(kind, sd):
    import models
    if kind == 'concat':
        m = models.MobileNetSkipConcat((64, 96), pretrained=False)
    elif kind == 'nnconv5dw':
        m = models.MobileNet('nnconv5dw', (64, 96), pretrained=False)
    else:
        m = models.MobileNetSkipAdd((64, 96), pretrained=False, widths=kind)
    m.load_state_dict(sd)
    return m.eval()


NETS = {'stock': synthetic.STOCK_WIDTHS, 'pruned': synthetic.PRUNED_WIDTHS, 'concat': 'concat', 'nnconv5dw': 'nnconv5dw'}


def _sd(name):
    if name == 'concat':
        return synthetic.synthetic_state_dict(seed=3, skip='concat')
    sd = synthetic.synthetic_state_dict(NETS[name] if name != 'nnconv5dw' else synthetic.STOCK_WIDTHS, seed=3)
    return synthetic.to_mobilenet_keys(sd) if name == 'nnconv5dw' else sd


def _oracle_forward(name, sd, x, dtype):
    if name == 'concat':
        return orc.skipconcat_forward(sd, x, dtype)
    if name == 'nnconv5dw':
        return orc.nnconv_dw_forward(sd, x, dtype)
    return orc.skipadd_forward(sd, x, dtype)


@pytest.mark.parametrize('name', sorted(NETS))
def test_fp64_composition_matches_the_oracle(name):
    """describe() + stage_ref without rounding == the MobileNet oracle in fp64, up to the fp32 BN folding (~4e-6 rel)."""
    sd = _sd(name)
    descs, weights, _ = fplan.describe(_module(NETS[name], sd))
    x = synthetic.synthetic_input(2, 64, 96, seed=5)
    got = sr.forward(descs, weights, x.double().numpy(), dtype=None)
    want = _oracle_forward(name, sd, x, torch.float64)
    assert np.all(got.r == 0)
    assert rel_err(torch.from_numpy(got.c), want) < 2e-5


@pytest.mark.parametrize('name', ['stock', 'pruned'])
@pytest.mark.parametrize('dtype', [torch.float16, torch.bfloat16])
def test_each_stage_contains_the_storage_emulated_oracle(name, dtype):
    """Stage by stage, fed the storage-emulated forward's OWN rounded input (conftest.storage_emulated_forward: fp32
    arithmetic in PyTorch's order, the product's rounding points), every stage_ref interval admits that forward's rounded
    output.  A rounding point stage_ref got wrong (the depthwise result or the upsampled value before the skip add left
    unrounded) puts 4-29 % of some stage's elements outside.  The floor on the determined fraction is lower than the
    sweep's 0.5: the fp16 intervals after the stock net's 1024-channel sums are about 40 % determined."""
    sd = synthetic.synthetic_state_dict(NETS[name], seed=3)
    sdq = {k: (v.to(dtype).float() if v.is_floating_point() else v) for k, v in sd.items()}
    descs, weights, names = fplan.describe(_module(NETS[name], sdq))
    x = synthetic.synthetic_input(2, 64, 96, seed=5)
    emu = {}
    final = storage_emulated_forward(sd, x, dtype, stages=emu)

    def nhwc(t):
        return sr.exact(t.permute(0, 2, 3, 1).double().numpy())
    xq = x.to(dtype).double().numpy()
    for i, (d, wt, nm) in enumerate(zip(descs, weights, names)):
        if d['kind'] == sr.STEM:
            ref = sr.stem(xq, wt[3], wt[4], wt[5], d['stride'], d['act'])
        elif d['kind'] == sr.DWPW:
            skip = nhwc(emu[names[d['skip_src']]]) if d['skip_src'] >= 0 else None
            ref = sr.dwpw(nhwc(emu[names[i - 1]]), wt, d, dtype, skip)['out']
        else:
            hd = sr.head(nhwc(emu[names[i - 1]]), wt[3], wt[4], wt[5], d['act'])
            ref = sr.Iv(hd.c[:, None], hd.r[:, None])
        got = final.numpy() if d['kind'] == sr.HEAD else emu[nm].permute(0, 2, 3, 1).numpy()
        assert sr.check(got, ref, dtype, nm) >= 0.35, nm


# ---------------------------------------------------------------------------------------------------------------------
# rounding helpers
# ---------------------------------------------------------------------------------------------------------------------
def test_fp16_rounding_matches_numpy():
    rng = np.random.default_rng(0)
    x = np.concatenate([rng.standard_normal(20000) * 10.0 ** rng.integers(-9, 5, 20000),
                        (np.arange(-3000, 3000) + 0.5) * 2.0 ** -10,               # exact ties at several binades
                        (np.arange(-3000, 3000) + 0.5) * 2.0 ** -24,               # ties between subnormals
                        [65504.0, 65519.99, 65520.0, -65520.0, 1e6, 0.0, -0.0, 2.0 ** -25, 3 * 2.0 ** -26]])
    want = x.astype(np.float16).astype(np.float64)
    got = sr.round_rne(x, torch.float16)
    assert np.array_equal(got, want, equal_nan=False)


def test_bf16_rounding_on_ties_and_near_ties():
    one = 1.0
    cases = [(one + 2.0 ** -8, one),                                   # tie between 1 and 1 + 2^-7: to even (1)
             (one + 3 * 2.0 ** -8, one + 2.0 ** -6),                   # tie between odd 1 + 2^-7 and even 1 + 2^-6
             (one + 2.0 ** -8 + 2.0 ** -30, one + 2.0 ** -7),          # just above a tie; fp64 -> fp32 -> bf16 would give 1
             (one + 2.0 ** -8 - 2.0 ** -40, one),
             (-(one + 2.0 ** -8 + 2.0 ** -30), -(one + 2.0 ** -7)),
             (6.0 + 2.0 ** -6, 6.0),                                   # tie at the ReLU6 clamp value
             (255.5 * 2.0 ** 100, 256.0 * 2.0 ** 100)]
    for x, want in cases:
        assert sr.round_rne(np.float64(x), torch.bfloat16) == want, x
    # single roundings agree with torch's fp32 -> bf16 cast
    rng = np.random.default_rng(1)
    f = (rng.standard_normal(50000) * 10.0 ** rng.integers(-20, 20, 50000)).astype(np.float32)
    want = torch.from_numpy(f).to(torch.bfloat16).double().numpy()
    assert np.array_equal(sr.round_rne(f.astype(np.float64), torch.bfloat16), want)


# ---------------------------------------------------------------------------------------------------------------------
# the checker
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('dtype', [torch.float16, torch.bfloat16])
def test_check_accepts_any_rounding_of_any_point_of_the_interval(dtype):
    rng = np.random.default_rng(2)
    c = rng.standard_normal((4, 5, 6, 16)) * 3
    r = np.abs(rng.standard_normal(c.shape)) * np.abs(c) * 2.0 ** -9 * (rng.random(c.shape) < 0.3)
    iv = sr.Iv(c, r)
    for _ in range(5):
        pt = c + r * rng.uniform(-1, 1, c.shape)
        sr.check(sr.round_rne(pt, dtype), iv, dtype)
    sr.check(sr.round_rne(iv.lo, dtype), iv, dtype)
    sr.check(sr.round_rne(iv.hi, dtype), iv, dtype)


def _f32(a):
    return np.asarray(a, np.float32)


def _stage(dtype, seed=3):
    """A realistic 3x3 s1 DWPW stage (c_in 40, c_out 24, ReLU6) on an exact 16-bit input, its interval reference and
    what a correct kernel computes: fp32 arithmetic in another summation order, rounded once per half-stage."""
    rng = np.random.default_rng(seed)
    rnd = (lambda a: sr.round_rne(a, dtype))
    n, h, w, ci, co = 2, 9, 11, 40, 24
    x = rnd(np.abs(rng.standard_normal((n, h, w, ci))))
    taps = rnd(rng.standard_normal((ci, 9)) / 3)
    pw = rnd(rng.uniform(-1, 1, (co, ci)) / np.sqrt(ci))
    d0 = sr.depthwise(sr.exact(x), taps, np.ones(ci), np.zeros(ci), 3, 1, sr.RELU, eps=0).c
    s1 = _f32(0.8 / d0.std(axis=(0, 1, 2))); b1 = _f32(0.5 - d0.mean(axis=(0, 1, 2)) * s1)
    d = rnd(np.clip(d0 * s1 + b1, 0, 6))
    p0 = d @ pw.T
    s2 = _f32(1.5 / p0.std(axis=(0, 1, 2))); b2 = _f32(1.0 - p0.mean(axis=(0, 1, 2)) * s2)
    wt = (taps, s1, b1, pw, s2, b2)
    desc = dict(kind=sr.DWPW, c_in=ci, c_out=co, ksize=3, stride=1, act=sr.RELU6, upsample=0, skip_src=-1)
    ref = sr.dwpw(sr.exact(x), wt, desc, dtype)
    # the "kernel": fp32, taps summed row by row from the bottom, pointwise by float32 BLAS
    xp = np.pad(_f32(x), ((0, 0), (1, 1), (1, 1), (0, 0)))
    acc = np.zeros((n, h, w, ci), np.float32)
    for ky in (2, 1, 0):
        for kx in range(3):
            acc = acc + xp[:, ky:ky + h, kx:kx + w, :] * _f32(taps[:, ky * 3 + kx])
    dk = rnd(np.clip(acc * s1 + b1, 0, 6).astype(np.float64))
    pk = np.clip(_f32(dk) @ _f32(pw.T) * s2 + b2, 0, 6).astype(np.float64)
    return ref, dk, pk


@pytest.mark.parametrize('dtype', [torch.float16, torch.bfloat16])
def test_check_on_a_realistic_stage(dtype):
    """A correct fp32 kernel passes with more than half of the elements determined; the mutations a kernel bug
    produces are all caught."""
    ref, dk, pk = _stage(dtype)
    good = sr.round_rne(pk, dtype)
    assert sr.check(dk, ref['dw'], dtype) >= 0.5
    assert sr.check(good, ref['pw'], dtype) >= 0.5
    assert (good == 0).mean() < 0.5 and (good == 6).any()
    p, emin, _ = sr._FMT[sr._dtname(dtype)]
    _, e = np.frexp(pk)
    q = np.ldexp(1.0, np.maximum(e, emin) - p)
    rtz = np.trunc(pk / q) * q                                   # round toward zero
    up = good.copy()
    up[..., 13] += np.ldexp(1.0, np.frexp(up[..., 13])[1] - p)  # +1 ulp on one output channel
    swap = good.copy()
    swap[..., [6, 7]] = swap[..., [7, 6]]                        # the two channels of one pair
    shift = good.copy()
    shift[1, 4, 1:] = good[1, 4, :-1]                            # one image row shifted by one pixel
    nan = good.copy()
    nan[0, 3, 5, 17] = np.nan
    for what, bad in (('rtz', rtz), ('+1ulp', up), ('swap', swap), ('shift', shift), ('nan', nan)):
        with pytest.raises(AssertionError):
            sr.check(bad, ref['pw'], dtype, what)


def test_check_fp32():
    iv = sr.Iv(np.array([1.0, -2.0, 3.0]), np.array([0.0, 1e-6, 0.0]))
    assert sr.check(np.array([1.0, -2.0 + 9e-7, 3.0], np.float32), iv, torch.float32) == 1.0
    with pytest.raises(AssertionError):
        sr.check(np.array([1.0, -2.0, 3.0 + 1e-5], np.float32), iv, torch.float32)
