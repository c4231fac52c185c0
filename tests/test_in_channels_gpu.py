"""MobileNet with 1 to 7 input channels (depth only, RGB-D) on the engine.

* every in_channels golden end to end through the module on path 0 and path 1 (fp16 1e-2, bf16 1e-1, fp32 1e-3; fp32 is
  nnconv5dw always and upconv under ``'high'``).  Storage-emulated conditioning of the goldens, measured on the CPU
  (tests/in_channels_ref.conditioning): fp16 2.0e-3 .. 2.2e-3 at 2x64x96 and 5.3e-3 at 1x224x224, bf16 1.5e-2 .. 2.1e-2
  and 4.5e-2;
* the stem, conv1 and conv2 buffers against the fp64 interval reference from the GPU's own input, on every image, for
  every c_in from 1 to 7, in every dtype, on maps of 32x32 (one front tile), 64x96 and 96x160 (odd tile counts);
* for every c_in the front route takes (1..4): ``front`` 1 and 0 give identical stage buffers and depth maps;
* a c_in = 4 plan serves smaller batches and resolutions with the bits of a fresh plan, and ``fd_forward_host`` copies
  c_in planes;
* module routing: c_in = 4 takes the engine and sees weight updates, c_in = 8 stays on stock PyTorch, a wrong channel
  count raises;
* every new kernel instance ran (the last test).
"""
import os

import numpy as np
import pytest
import torch

import in_channels_ref as icr
import plan_check as pc
import test_kernel_sweep as ks
from conftest import GOLDEN, rel_err
from fastdepth_b200 import plan as fplan
from oracle import stage_ref as sr

pytestmark = pytest.mark.gpu

F16, BF16, F32 = torch.float16, torch.bfloat16, torch.float32
R, R6 = sr.RELU, sr.RELU6
TOL = {F32: 1e-3, F16: 1e-2, BF16: 1e-1}
SEEN = set()             # (kernel name, dtype) of every step the tests below ran
FRONT_WIDTHS = (32, 64, 128, 128, 256, 32)           # the stock front: 32 -> 64 -> 128, eligible for the front route
SHAPES = [(3, 32, 32), (2, 64, 96), (1, 96, 160)]


def _record(p, dtype):
    for s in p.steps():
        SEEN.add((s['kernel'], str(dtype)))


# ------------------------------------------------------------------------------------------------ goldens + routing
def _module(name, dtype, path):
    from fastdepth_b200.engine import SkipAddEngine
    decoder, c, n, h, w = icr.GOLDENS[name]
    m = icr.model(decoder, c, (h, w)).cuda().to(dtype)
    eng = SkipAddEngine(m)
    eng.set_option('path', path)
    m.__dict__['_fd_engine'] = eng
    return m, eng


@pytest.mark.parametrize('name', list(icr.GOLDENS))
@pytest.mark.parametrize('dtype', [F32, F16, BF16])
@pytest.mark.parametrize('path', [0, 1])
def test_golden_through_the_module(name, dtype, path):
    fx = np.load(os.path.join(GOLDEN, name + '.npz'))
    decoder, c, n, h, w = icr.GOLDENS[name]
    m, eng = _module(name, dtype, path)
    x = icr.golden_input(name).cuda().to(dtype)
    prec = torch.get_float32_matmul_precision()
    torch.set_float32_matmul_precision('high' if decoder == 'upconv' else prec)
    try:
        with torch.no_grad():
            y = m(x)
        torch.cuda.synchronize()
    finally:
        torch.set_float32_matmul_precision(prec)
    assert m.__dict__['_fd_engine'] is eng and eng.plans                  # it ran on the engine
    p = next(iter(eng.plans.values()))
    _record(p, dtype)
    kernels = [s['kernel'] for s in p.steps()]
    if path == 1 and dtype != F32:
        assert kernels[0] == 'stem_tc+front<k3s1,k3s2,8x8>[n32,n64,n128,relu6,cin%d]' % c, kernels
    elif c != 3:
        assert kernels[0] == 'stem_kernel<cin%d>' % c, kernels
    assert rel_err(y.float().cpu(), torch.from_numpy(fx['output'])) <= TOL[dtype]


@pytest.mark.parametrize('dtype', [F16, BF16])
def test_module_routes_rgbd_and_sees_weight_updates(dtype):
    decoder, c, n, h, w = icr.GOLDENS['nnconv5dw_cin4_2x64x96']
    m = icr.model(decoder, c, (h, w)).cuda().to(dtype)
    x = icr.golden_input('nnconv5dw_cin4_2x64x96').cuda().to(dtype)
    with torch.no_grad():
        y = m(x)
        assert '_fd_engine' in m.__dict__
        m.mobilenet[0][0].weight.mul_(0.5)                     # the stem itself
        y2 = m(x)
        want = icr.torch_forward({k: v.float().cpu() for k, v in m.state_dict().items()}, x.float().cpu(), decoder,
                                 storage=dtype)
    torch.cuda.synchronize()
    assert not torch.equal(y, y2)
    assert rel_err(y2.float().cpu(), want) <= TOL[dtype]
    with pytest.raises(RuntimeError, match='expected input.*to have 4 channels, but got 3 channels'):
        with torch.no_grad():
            m(x[:, :3].contiguous())
    with pytest.raises(RuntimeError, match='expected input.*to have 4 channels, but got 3 channels'):
        m.__dict__['_fd_engine'](x[:, :3].contiguous())


def test_eight_channels_stay_on_pytorch():
    import models
    m = models.MobileNet('nnconv5dw', (64, 96), in_channels=8, pretrained=False).eval().cuda().half()
    x = torch.rand(2, 8, 64, 96, device='cuda').half()
    with torch.no_grad():
        y = m(x)
    assert '_fd_engine' not in m.__dict__ and y.shape == (2, 1, 64, 96)


# ------------------------------------------------------------------------------------------------ stage checks
def _descs(c_in, act=R6):
    acts = (R6, act, act, R6, R6, R, R, R)
    d = ks.enc_dec(FRONT_WIDTHS, acts)
    d[0]['c_in'] = c_in
    return d


def _weights(descs, dtype, x, seed):
    """Seeded weights representable in the plan dtype, BN calibrated stage by stage on the reference's point forward of
    the probe x (test_kernel_sweep.make_weights with a stem of any c_in)."""
    rng = np.random.default_rng(seed)
    q = None if dtype == F32 else dtype
    weights, outs, cur = [], [], None
    for d in descs:
        if d['kind'] == sr.STEM:
            w = ks._repr(rng.standard_normal((d['c_out'], d['c_in'], 3, 3)) * 0.7 / np.sqrt(d['c_in']), dtype)
            pre = icr.stem(x, w, np.ones(d['c_out']), np.zeros(d['c_out']), d['stride'], None, eps=0).c
            s, b = ks._bn(pre, d['act'], rng)
            wt = (None, None, None, w.reshape(d['c_out'], -1), s, b)
            y = sr.quantize(icr.stem(x, w, s, b, d['stride'], d['act'], eps=0), q)
        elif d['kind'] == sr.DWPW:
            k, ci, co = d['ksize'], d['c_in'], d['c_out']
            taps = ks._repr(rng.standard_normal((ci, k * k)) * (1.0 / k), dtype)
            dpre = sr.depthwise(cur, taps, np.ones(ci), np.zeros(ci), k, d['stride'], None, eps=0).c
            s1, b1 = ks._bn(dpre, d['act'], rng)
            dq = sr.quantize(sr.depthwise(cur, taps, s1, b1, k, d['stride'], d['act'], eps=0), q)
            pw = ks._repr(rng.uniform(-1, 1, (co, ci)) * np.sqrt(3.0 / ci), dtype)
            s2, b2 = ks._bn(dq.c @ pw.T.astype(np.float64), d['act'], rng)
            wt = (taps, s1, b1, pw, s2, b2)
            src = d['skip_src']
            y = sr.quantize(sr.dwpw(cur, wt, d, q, outs[src] if src >= 0 else None, eps=0)['out'], q)
        else:
            w = ks._repr(np.abs(rng.standard_normal(d['c_in'])) / np.sqrt(d['c_in']), dtype)
            pre = cur.c @ w.astype(np.float64)
            s = np.array([1.0 / (pre.std() + 1e-6)], np.float32)
            b = np.array([2.0 - pre.mean() * float(s[0])], np.float32)
            weights.append((None, None, None, w.reshape(1, -1), s, b))
            return weights
        weights.append(wt)
        outs.append(y)
        cur = sr.Iv(y.c)
    raise ValueError('no head')


def _case(c_in, dtype, n, h, w, act=R6, seed=0):
    descs = _descs(c_in, act)
    rng = np.random.default_rng(seed)
    x_host = ks._repr(rng.uniform(0.0, 1.0, (n, c_in, h, w)), dtype)
    probe = x_host.astype(np.float64)
    if h * w < 64 * 64:
        probe = np.concatenate([probe, ks._repr(rng.uniform(0.0, 1.0, (6, c_in, h, w)), dtype).astype(np.float64)])
    weights = _weights(descs, dtype, probe, seed + 1)
    p = fplan.Plan(descs, weights, ['s%d' % i for i in range(len(descs))], n, h, w, dtype, 0)
    x = torch.from_numpy(x_host).to(dtype).cuda()
    y = torch.empty((n, 1, h, w), dtype=dtype, device='cuda')
    return descs, weights, x_host, p, x, y


STAGE_CASES = []
for _c in range(1, 8):
    for _dt in (F16, BF16):
        for _a in (R6, R):
            STAGE_CASES.append((_c, _dt, 1, _a, SHAPES[(_c + (_a == R)) % 3]))
        STAGE_CASES.append((_c, _dt, 0, R6, SHAPES[_c % 3]))                    # SIMT stem_kernel, path 0
    STAGE_CASES.append((_c, F32, 1, R6, SHAPES[(_c + 1) % 3]))                  # fp32: stem_kernel on path 1 too


@pytest.mark.parametrize('c_in,dtype,path,act,shape', STAGE_CASES,
                         ids=['c%d-%s-path%d-%s-%dx%dx%d' % (c, str(d)[6:], pa, 'relu6' if a == R6 else 'relu', *s)
                              for c, d, pa, a, s in STAGE_CASES])
def test_front_stages_against_the_interval_reference(c_in, dtype, path, act, shape, monkeypatch):
    """The stem, conv1 and conv2 buffers from the GPU's own input, every image, every element (stage_ref.check)."""
    monkeypatch.setattr(sr, 'stem', icr.stem)                  # plan_check's stem reference, for any c_in
    n, h, w = shape
    case = 'cin%d_%s_path%d_%d' % (c_in, str(dtype)[6:], path, act)
    descs, weights, x_host, p, x, y = _case(c_in, dtype, n, h, w, act, seed=c_in * 7 + path)
    p.set_option('path', path)
    chk = pc.Checker(case, dtype)
    ran = pc.check_plan(p, descs, weights, dtype, x_host, x, y, range(n), chk, dict(path=path), 1,
                        torch.cuda.current_stream().cuda_stream, only={0, 1, 2}, rerun_all=False)
    for steps in ran:
        for s in steps:
            SEEN.add((s['kernel'], str(dtype)))
    kern = [s['kernel'] for s in ran[0]]
    front = path == 1 and dtype != F32 and c_in <= 4
    assert any(k.startswith('stem_tc+front<') for k in kern) == front, kern
    assert chk.zeros < 0.5 * chk.n
    p.close()


FRONT_CASES = [(c, d, s) for c in range(1, 5) for d in (F16, BF16) for s in (SHAPES[1], SHAPES[2])]


@pytest.mark.parametrize('c_in,dtype,shape', FRONT_CASES,
                         ids=['c%d-%s-%dx%dx%d' % (c, str(d)[6:], *s) for c, d, s in FRONT_CASES])
def test_front_equals_three_steps(c_in, dtype, shape):
    n, h, w = shape
    _, _, _, p, x, y = _case(c_in, dtype, n, h, w, R6 if c_in % 2 else R, seed=c_in)
    stream = torch.cuda.current_stream().cuda_stream
    res = {}
    for front in (1, 0):
        p.set_option('front', front)
        y.zero_()
        p.forward(x, y, stream)
        torch.cuda.synchronize()
        _record(p, dtype)
        kern = [s['kernel'] for s in p.steps()]
        assert any('stem_tc+front<' in k for k in kern) == bool(front), kern
        assert front or kern[0] == ('stem_tc<k3,s2,1x8x16>[n32]' if c_in == 3 else 'stem_tc<k3,s2,1x8x16,cin%d>[n32]' % c_in)
        res[front] = [p.stage_tensor(i).clone() for i in range(3)] + [y.clone()]
    for a, b in zip(res[1], res[0]):
        assert torch.equal(a, b)
    p.close()


# ------------------------------------------------------------------------------------------------ shapes, host copies
def test_rgbd_plan_serves_smaller_shapes_bit_for_bit():
    m = icr.model('nnconv5dw', 4).cuda().half()
    from fastdepth_b200 import synthetic
    stream = torch.cuda.current_stream().cuda_stream
    big = fplan.Plan.from_module(m, 4, 224, 224, F16, 0)
    for n, h, w in ((4, 224, 224), (2, 224, 224), (1, 96, 160), (3, 64, 96), (1, 32, 32)):
        x = synthetic.synthetic_input(n, h, w, seed=n + h, channels=4).cuda().half()
        y = torch.empty((n, 1, h, w), dtype=F16, device='cuda')
        big.forward(x, y, stream)
        fresh = fplan.Plan.from_module(m, n, h, w, F16, 0)
        y2 = torch.empty_like(y)
        fresh.forward(x, y2, stream)
        torch.cuda.synchronize()
        assert torch.equal(y, y2), (n, h, w)
        fresh.close()
    big.close()


def test_forward_host_copies_every_plane():
    from fastdepth_b200 import synthetic
    m = icr.model('nnconv5dw', 4).cuda().half()
    n, h, w = 2, 64, 96
    p = fplan.Plan.from_module(m, n, h, w, F16, 0)
    x = synthetic.synthetic_input(n, h, w, seed=3, channels=4).half()
    stream = torch.cuda.current_stream().cuda_stream
    y_dev = torch.empty((n, 1, h, w), dtype=F16, device='cuda')
    p.forward(x.cuda(), y_dev, stream)
    torch.cuda.synchronize()
    y_host = torch.empty((n, 1, h, w), dtype=F16).pin_memory()
    p.forward_host(x.pin_memory(), y_host, stream)
    assert torch.equal(y_host, y_dev.cpu())
    t = p.pipeline_submit(x.pin_memory(), y_host)
    p.pipeline_wait(t)
    assert torch.equal(y_host, y_dev.cpu())
    p.close()


def test_every_new_instance_ran():
    """Every stem_tc_kernel and SIMT stem_kernel c_in instance, and every front_tc_kernel (c_in, dtype, act) instance."""
    names = {(k, d) for k, d in SEEN}
    missing = []
    for c in range(1, 8):
        tag = '' if c == 3 else ',cin%d' % c
        for d in (F16, BF16):
            if ('stem_tc<k3,s2,1x8x16%s>[n32]' % tag, str(d)) not in names:
                missing.append(('stem_tc', c, str(d)))
            if c <= 4:
                for a in ('relu6', 'relu'):
                    if ('stem_tc+front<k3s1,k3s2,8x8>[n32,n64,n128,%s%s]' % (a, tag), str(d)) not in names:
                        missing.append(('front', c, str(d), a))
        for d in (F32, F16, BF16):
            if ('stem_kernel' if c == 3 else 'stem_kernel<cin%d>' % c, str(d)) not in names:
                missing.append(('stem_kernel', c, str(d)))
    if len(SEEN) < 40:
        pytest.skip('coverage is only meaningful after the whole file ran')
    assert not missing, missing
