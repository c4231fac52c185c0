"""Split TF32 ("tf32x3") on the dense decoders, on the GPU.

Under ``torch.set_float32_matmul_precision('high' | 'medium')`` an fp32 ``models.MobileNet('nnconv5' | 'nnconv3' |
'deconv<k>' | 'upconv')`` runs on the engine, every CONV, DECONV and UPCONV stage on conv_tc_tf32x3_kernel.  Checked here:
* the dense-decoder goldens through the module, within the fp32 bound of 1e-3;
* a stage sweep: every split-TF32 dense stage against the interval reference (tests/dense_ref.conv,
  tests/convt_ref.convt) from the GPU's own input tensor, with eps_conv = 2 EPS_CONV + 2^-20 (three TF32 products per
  term and six times as many accumulator updates, tests/test_tf32x3_dense_cpu.py);
* bitwise properties: a batch equals its images run alone, graph on equals graph off, the depth map does not depend on
  the tile, the bn or the phase grouping;
* switching the precision on one module, weight updates, and an explicit ``set_option('tf32x3', 0)``;
* the module's own plans at production size, every stage of every image.
"""
import os
import time

import numpy as np
import pytest
import torch

import convt_ref as cr
import dense_ref as dr
import plan_check as pc
from conftest import GOLDEN, rel_err
from fastdepth_b200 import plan as fplan
from fastdepth_b200 import synthetic
from fastdepth_b200.engine import SkipAddEngine
from oracle import stage_ref as sr
from test_convt_gpu import _rand_stage_list

pytestmark = pytest.mark.gpu

F32 = torch.float32
EPS_TF32X3 = sr.EPS + 2.0 ** -20
EPS_CONV_TF32X3 = 2 * dr.EPS_CONV + 2.0 ** -20
C, D, U = dr.CONV, cr.DECONV, cr.UPCONV
R, R6 = sr.RELU, sr.RELU6


@pytest.fixture
def precision():
    """Restores torch's fp32 matmul precision after the test."""
    prev = torch.get_float32_matmul_precision()
    yield torch.set_float32_matmul_precision
    torch.set_float32_matmul_precision(prev)


def _tag(d):
    if d['kind'] == C:
        return 'k%d' % d['ksize']
    return '%s%d' % ('deconv' if d['kind'] == D else 'upconv', d['ksize'])


def _tf32x3_prefix(d):
    return 'conv_tc_kernel<%s,tf32x3,' % _tag(d)


# ---------------------------------------------------------------------------------------------------------------------
# stage-by-stage check
# ---------------------------------------------------------------------------------------------------------------------
def check_stages(p, descs, weights, x_host, y, pick, chk, fold):
    """Every stage the plan materialised for the images ``pick``: STEM; DWPW as dw_kernel + the split-TF32 pointwise step
    (from the GPU's own intermediate, eps = EPS_TF32X3); CONV / DECONV / UPCONV from the GPU's own input tensor with
    eps_conv = EPS_CONV_TF32X3; the head from the last stage's buffer."""
    ns = len(descs)

    def buf(i):
        return sr.exact(pc.nhwc(p.stage_tensor(i), pick))

    for i in range(ns - 1):
        d, wt = descs[i], weights[i]
        last = i == ns - 2
        if d['kind'] == sr.STEM:
            chk(pc.nhwc(p.stage_tensor(0), pick), sr.stem(x_host[pick], *wt[3:], d['stride'], d['act']), 'stem')
        elif d['kind'] == sr.DWPW:
            mid = p.stage_tensor(i, which=1)
            chk(pc.nhwc(mid, pick), sr.depthwise(buf(i - 1), *wt[:3], d['ksize'], d['stride'], d['act']),
                'stage %d depthwise' % i)
            out = sr.pointwise(sr.exact(pc.nhwc(mid, pick)), *wt[3:], d['act'], eps=EPS_TF32X3)
            chk(pc.nhwc(p.stage_tensor(i), pick), sr.upsample(out) if d['upsample'] and not (last and fold) else out,
                'stage %d' % i)
        elif d['kind'] == C:
            r = dr.conv(buf(i - 1), wt[3], wt[4], wt[5], d['ksize'], d['act'], eps=EPS_CONV_TF32X3)
            chk(pc.nhwc(p.stage_tensor(i), pick), sr.upsample(r) if d['upsample'] and not (last and fold) else r,
                'stage %d' % i)
        else:
            r = cr.convt(buf(i - 1), wt[3], wt[4], wt[5], d['kind'], d['ksize'], d['act'], eps=EPS_CONV_TF32X3)
            chk(pc.nhwc(p.stage_tensor(i), pick), r, 'stage %d' % i)
    hd = sr.head(buf(ns - 2), *weights[-1][3:], descs[-1]['act'])
    chk(pc.nhwc(y[:, 0], pick), sr.upsample(hd) if fold else hd, 'head')


def assert_split_steps(steps, descs, fold):
    """Every dense stage runs one split-TF32 step (k*k*c_in*c_out dense MACs per conv-resolution pixel); a folded head
    runs head_kernel<up2x>."""
    dense = [i for i, d in enumerate(descs) if d['kind'] in pc.DENSE]
    for i in dense:
        mine = [s['kernel'] for s in steps if s['stage'] == i]
        assert len(mine) == 1 and mine[0].startswith(_tf32x3_prefix(descs[i])), (i, mine)
    for s in steps:
        d = descs[s['stage']]
        if d['kind'] in pc.DENSE:
            assert s['dw_macs'] == 0 and s['dense_macs'] == s['macs'] > 0
    assert steps[-1]['kernel'] == ('head_kernel<up2x>' if fold else 'head_kernel')
    return len(dense)


def fold_of(p, descs):
    return bool(p.get_option('fold_head') and descs[-2]['upsample'] and descs[-2]['skip_src'] < 0)


# ---------------------------------------------------------------------------------------------------------------------
# stage sweep
# ---------------------------------------------------------------------------------------------------------------------
def _dec(kind, k, cos):
    return tuple((kind, co, k) for co in cos)


# (name, n, h, w, down, decoder stages, act, options, env); c_in tails mod 32 = 8 / 16 / 24 come from c_out of the stage
# before; maps of 1x1 / 1x2 (h, w = 32 / 64 after five halvings) and several images per tile
SWEEP = [
    ('k5_tails', 3, 64, 96, 4, _dec(C, 5, (40, 88, 264, 72, 8)), R, {}, {}),
    ('k3_tails_r6_unfolded', 3, 64, 96, 4, _dec(C, 3, (48, 120, 136, 24, 8)), R6, {'fold_head': 0}, {}),
    ('k5_1x1_r6', 4, 32, 32, 4, _dec(C, 5, (24, 72, 40, 16, 8)), R6, {}, {}),
    ('d3_tails', 3, 64, 96, 4, _dec(D, 3, (40, 88, 264, 72, 8)), R, {}, {}),
    ('d5_1x2_r6', 2, 32, 64, 4, _dec(D, 5, (24, 136, 40, 16, 8)), R6, {}, {}),
    ('d7_tails', 3, 64, 96, 4, _dec(D, 7, (56, 88, 200, 24, 8)), R, {}, {}),
    ('d9_1x2', 2, 32, 64, 4, _dec(D, 9, (24, 136, 40, 16, 8)), R, {}, {}),
    ('u5_1x1_r6', 4, 32, 32, 4, _dec(U, 5, (24, 72, 40, 16, 8)), R6, {}, {}),
    ('u5_tails', 3, 64, 96, 4, _dec(U, 5, (40, 88, 264, 72, 8)), R, {}, {}),
    ('mixed', 3, 64, 96, 4, ((C, 40, 5), (D, 88, 5), (C, 24, 3), (U, 72, 5), (D, 8, 7)), R, {}, {}),
    ('bn64_d5', 2, 32, 64, 4, _dec(D, 5, (136, 72, 16, 8, 8)), R, {}, {'FD_CONV_BN': '64'}),
    ('bn128_k5_r6', 2, 32, 64, 4, _dec(C, 5, (136, 72, 16, 8, 8)), R6, {}, {'FD_CONV_BN': '128'}),
    ('bn128_u5', 2, 32, 64, 4, _dec(U, 5, (264, 72, 16, 8, 8)), R, {}, {'FD_CONV_BN': '128'}),
    ('bn128_d9_r6', 2, 32, 64, 4, _dec(D, 9, (136, 72, 16, 8, 8)), R6, {}, {'FD_CONV_BN': '128'}),
    ('bn64_k3', 3, 64, 96, 4, _dec(C, 3, (136, 72, 16, 8, 8)), R, {}, {'FD_CONV_BN': '64'}),
    ('bn128_k3', 3, 64, 96, 4, _dec(C, 3, (136, 72, 16, 8, 8)), R, {}, {'FD_CONV_BN': '128'}),
    ('bn64_u5_r6', 2, 32, 64, 4, _dec(U, 5, (136, 72, 16, 8, 8)), R6, {}, {'FD_CONV_BN': '64'}),
    ('pairs_d7', 3, 64, 96, 4, _dec(D, 7, (64, 128, 64, 32, 8)), R, {}, {'FD_CONV_PHASE_GROUP': '2'}),
    ('singles_u5_r6', 3, 64, 96, 4, _dec(U, 5, (64, 128, 64, 32, 8)), R6, {}, {'FD_CONV_PHASE_GROUP': '1'}),
]
SEEN = set()             # (bn, act, kind) of the split-TF32 dense steps the sweep ran


def _with_env(env, fn):
    saved = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return fn()
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _sweep_plan(descs, wts, n, h, w, opts, env, x, tf32x3=1):
    def run():
        p = fplan.Plan(descs, wts, ['s%d' % i for i in range(len(descs))], n, h, w, F32, 0)
        p.set_option('tf32x3', tf32x3)
        for k, v in opts.items():
            p.set_option(k, v)
        y = torch.empty((n, 1, h, w), dtype=F32, device='cuda')
        p.forward(x, y, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        return p, y
    return _with_env(env, run)


@pytest.mark.parametrize('case', SWEEP, ids=[c[0] for c in SWEEP])
def test_stage_sweep(case, built_lib):
    name, n, h, w, down, decs, act, opts, env = case
    descs, wts = _rand_stage_list(sum(map(ord, name)), F32, down, decs, act)
    x = synthetic.synthetic_input(n, h, w, seed=3).cuda()
    p, y = _sweep_plan(descs, wts, n, h, w, dict(opts, graph=0), env, x)
    fold = fold_of(p, descs)
    steps = p.steps()
    assert assert_split_steps(steps, descs, fold) == 5
    for s in steps:
        d = descs[s['stage']]
        if d['kind'] not in pc.DENSE:
            continue
        kn = s['kernel']
        if 'FD_CONV_BN' in env:
            assert ',bn%s,' % env['FD_CONV_BN'] in kn, kn
        if 'FD_CONV_PHASE_GROUP' in env and d['kind'] != C:
            assert (',4ph2>' in kn) == (env['FD_CONV_PHASE_GROUP'] == '2'), kn
        if d['kind'] == C:
            assert (',up>' in kn) == (not (fold and s['stage'] == len(descs) - 2)), kn
        SEEN.add((int(kn.split(',bn')[1].split(',')[0]), 'relu6' if act == R6 else 'relu', 'conv' if d['kind'] == C else 'phased'))
    chk = pc.Checker(name, F32)
    check_stages(p, descs, wts, x.cpu().numpy(), y, list(range(n)), chk, fold)
    chk.flush()
    p.close()


def test_sweep_coverage():
    """Both bn (64, 128) and both activations ran a CONV and a phased stage in the sweep above."""
    want = {(bn, a, k) for bn in (64, 128) for a in ('relu', 'relu6') for k in ('conv', 'phased')}
    assert want <= SEEN, sorted(want - SEEN)


# ---------------------------------------------------------------------------------------------------------------------
# bitwise properties
# ---------------------------------------------------------------------------------------------------------------------
BIT_DECS = ((D, 40, 5), (U, 264, 5), (C, 72, 5), (D, 24, 9), (C, 8, 3))


def _bit_plan(x, env=None, opts=None):
    descs, wts = _rand_stage_list(7, F32, 4, BIT_DECS, R)
    return _sweep_plan(descs, wts, x.shape[0], 64, 96, opts or {}, env or {}, x)


def test_batch_equals_images_alone(built_lib):
    x = synthetic.synthetic_input(3, 64, 96, seed=5).cuda()
    _, y = _bit_plan(x)
    for i in range(3):
        _, yi = _bit_plan(x[i:i + 1].contiguous())
        assert torch.equal(y[i:i + 1], yi), i


def test_graph_on_equals_graph_off(built_lib):
    x = synthetic.synthetic_input(3, 64, 96, seed=5).cuda()
    _, y0 = _bit_plan(x, opts={'graph': 0})
    p, y1 = _bit_plan(x, opts={'graph': 1})
    y2 = torch.empty_like(y1)
    p.forward(x, y2, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert torch.equal(y0, y1) and torch.equal(y1, y2)


def test_result_does_not_depend_on_tile_bn_or_grouping(built_lib):
    x = synthetic.synthetic_input(3, 64, 96, seed=5).cuda()
    p, ref = _bit_plan(x)
    names = [s['kernel'] for s in p.steps()]
    for env in ({'FD_CONV_PHASE_GROUP': '1'}, {'FD_CONV_PHASE_GROUP': '2'}, {'FD_CONV_TILE': '0'}, {'FD_CONV_TILE': '2'},
                {'FD_CONV_TILE': '4', 'FD_CONV_PHASE_GROUP': '2'}, {'FD_CONV_BN': '64'}, {'FD_CONV_BN': '128'},
                {'FD_CONV_TILE': '3', 'FD_CONV_BN': '128', 'FD_CONV_PHASE_GROUP': '1'}):
        q, y = _bit_plan(x, env=env)
        assert torch.equal(ref, y), (env, [s['kernel'] for s in q.steps()])
    assert any('tf32x3' in k for k in names)


def test_split_weights_are_counted(built_lib):
    """The split weights ([2][c_out][k*k][c_in] fp32) are device memory the built steps hold."""
    x = synthetic.synthetic_input(1, 64, 96, seed=5).cuda()
    descs, wts = _rand_stage_list(7, F32, 4, BIT_DECS, R)
    p0, _ = _sweep_plan(descs, wts, 1, 64, 96, {}, {}, x, tf32x3=0)
    p1, _ = _sweep_plan(descs, wts, 1, 64, 96, {}, {}, x, tf32x3=1)
    split = sum(2 * d['ksize'] ** 2 * d['c_in'] * d['c_out'] * 4 for d in descs if d['kind'] in pc.DENSE)
    pw = sum(2 * d['c_in'] * d['c_out'] * 4 for d in descs if d['kind'] == sr.DWPW)
    assert p1.workspace_bytes() - p0.workspace_bytes() == split + pw


# ---------------------------------------------------------------------------------------------------------------------
# the module under torch.set_float32_matmul_precision
# ---------------------------------------------------------------------------------------------------------------------
GOLDENS = ['nnconv5_stock_2x64x96', 'nnconv5_stock_1x224x224', 'deconv3_stock_2x64x96', 'deconv5_stock_2x64x96',
           'deconv7_stock_2x64x96', 'deconv9_stock_2x64x96', 'deconv5_stock_1x224x224', 'upconv5_stock_2x64x96',
           'upconv5_stock_1x224x224']


def _golden_model(name):
    import models
    fx = np.load(os.path.join(GOLDEN, name + '.npz'))
    n, h, w = (int(v) for v in fx['shape'])
    if name.startswith('nnconv5'):
        dec = 'nnconv5'
        sd = synthetic.synthetic_nnconv_state_dict(5, seed=int(fx['wseed']))
    else:
        dec = str(fx['decoder'])
        sd = synthetic.synthetic_convt_state_dict(dec, seed=int(fx['wseed']))
    m = models.MobileNet(dec, (h, w), pretrained=False)
    m.load_state_dict(sd)
    x = synthetic.synthetic_input(n, h, w, seed=int(fx['xseed']))
    return m.eval().cuda(), x.cuda(), torch.from_numpy(fx['output'])


def _forward(m, x):
    with torch.no_grad():
        y = m(x)
    torch.cuda.synchronize()
    return y


def _engine_steps(m):
    eng = m.__dict__['_fd_engine']
    return next(iter(eng.plans.values())).steps()


@pytest.mark.parametrize('name', GOLDENS)
def test_golden_under_high(name, built_lib, precision):
    m, x, want = _golden_model(name)
    precision('high')
    y = _forward(m, x)
    err = rel_err(y.cpu(), want)
    print('%s under high: rel err %.2e' % (name, err))
    assert err <= 1e-3
    descs, _, _ = fplan.describe(m)
    steps = _engine_steps(m)
    assert sum('tf32x3' in s['kernel'] and s['kernel'].startswith(_tf32x3_prefix(descs[s['stage']]))
               for s in steps if descs[s['stage']]['kind'] in pc.DENSE) == 5
    assert m.__dict__['_fd_engine'].options == {}


def test_switching_and_weight_updates(built_lib, precision):
    """'highest' -> 'high' -> 'medium' -> 'highest' on one module: stock PyTorch, the engine, the same bits, stock PyTorch
    again; a weight update under 'high' is picked up; an explicit set_option('tf32x3', 0) gives convt_kernel steps."""
    m, x, want = _golden_model('deconv5_stock_2x64x96')
    precision('highest')
    y_stock = _forward(m, x)
    assert '_fd_engine' not in m.__dict__
    precision('high')
    y_tf = _forward(m, x)
    eng = m.__dict__['_fd_engine']
    assert rel_err(y_tf.cpu(), want) <= 1e-3 and not torch.equal(y_tf, y_stock)
    assert sum(s['kernel'].startswith('conv_tc_kernel<deconv5,tf32x3,') for s in _engine_steps(m)) == 5
    precision('medium')
    assert torch.equal(_forward(m, x), y_tf)
    assert m.__dict__['_fd_engine'] is eng and len(eng.plans) == 1
    calls = []
    plan_for = eng.plan_for
    eng.plan_for = lambda t: calls.append(1) or plan_for(t)
    precision('highest')
    y_back = _forward(m, x)                          # stock PyTorch again: the engine is not called
    assert not calls and not torch.equal(y_back, y_tf) and rel_err(y_back.cpu(), y_stock.cpu()) <= 1e-2
    del eng.plan_for
    # a weight update under 'high': the engine sees it and matches a fresh engine on the updated module
    precision('high')
    with torch.no_grad():
        m.decoder.convt3[0].weight.mul_(0.5)
    y_new = _forward(m, x)
    assert not torch.equal(y_new, y_tf)
    eng1 = SkipAddEngine(m)
    eng1.set_option('tf32x3', 1)
    m.__dict__['_fd_engine'] = eng1
    assert torch.equal(_forward(m, x), y_new)
    eng1.set_option('tf32x3', 0)                     # explicit: wins over 'high'
    _forward(m, x)
    kernels = [s['kernel'] for s in _engine_steps(m)]
    assert not any('tf32x3' in k for k in kernels)
    assert sum(k == 'convt_kernel<deconv5>' for k in kernels) == 5


def _production(decoder, n, sd, precision):
    import models
    t0 = time.perf_counter()
    h = w = 224
    m = models.MobileNet(decoder, (h, w), pretrained=False)
    m.load_state_dict(sd)
    m = m.eval().cuda()
    x = synthetic.synthetic_input(n, h, w, seed=0).cuda()
    precision('high')
    y = _forward(m, x)
    p = m.__dict__['_fd_engine'].plan_for(x)
    descs, weights, _ = fplan.describe(m)
    fold = fold_of(p, descs)
    assert assert_split_steps(p.steps(), descs, fold) == 5
    x_host = x.cpu().numpy()
    chk = pc.Checker('production %s b%d' % (decoder, n), F32)
    for k in range(0, n, pc.CHUNK):
        check_stages(p, descs, weights, x_host, y, list(range(k, min(n, k + pc.CHUNK))), chk, fold)
    chk.flush()
    print('\nproduction %s fp32 tf32x3 b%d 224x224: %d tensors checked in %.1f s' %
          (decoder, n, len(chk.results), time.perf_counter() - t0))


def test_production_nnconv5_b64(built_lib, precision):
    _production('nnconv5', 64, synthetic.synthetic_nnconv_state_dict(5, seed=1), precision)


def test_production_deconv5_b16(built_lib, precision):
    _production('deconv5', 16, synthetic.synthetic_convt_state_dict('deconv5', seed=1), precision)
