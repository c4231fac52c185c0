"""Split-TF32 pointwise steps ("tf32x3") on the GPU: the default is unchanged, the modules follow
``torch.set_float32_matmul_precision``, and every split-TF32 step is checked stage by stage against the fp32 interval
reference (oracle/stage_ref.py) from the GPU's own depthwise intermediate, with the product allowance of three TF32
products: eps = sr.EPS + 2^-20 (tests/test_tf32x3_cpu.py derives it and shows that one TF32 product falls outside)."""
import os
import time

import numpy as np
import pytest
import torch

import plan_check as pc
import test_kernel_sweep as ks
from conftest import GOLDEN, rel_err
from fastdepth_b200 import plan as fplan
from fastdepth_b200 import synthetic
from fastdepth_b200.engine import SkipAddEngine
from oracle import stage_ref as sr

pytestmark = pytest.mark.gpu

F32 = torch.float32
EPS_TF32X3 = sr.EPS + 2.0 ** -20
R, R6 = sr.RELU, sr.RELU6
TF32X3 = 'conv_tc_kernel<pw,tf32x3,'


@pytest.fixture
def precision():
    """Restores torch's fp32 matmul precision after the test."""
    prev = torch.get_float32_matmul_precision()
    yield torch.set_float32_matmul_precision
    torch.set_float32_matmul_precision(prev)


# ---------------------------------------------------------------------------------------------------------------------
# stage-by-stage check of a plan whose fp32 DWPW stages run a dw_kernel step and a split-TF32 step
# ---------------------------------------------------------------------------------------------------------------------
def check_stages(p, descs, weights, x_host, pick, chk, fold, saved=None, only_adds=False):
    """Check every stage the plan materialised for the images ``pick`` (fp32: |got - centre| <= radius + ulp / 2).  DWPW
    stages: the depthwise half from the stage's input, the split-TF32 pointwise half from the GPU's own intermediate
    (``which=1``) with eps = EPS_TF32X3.  ``saved``: the skip sources as they were before an in-place add;
    ``only_adds``: check only the stages that add a skip (and the head)."""
    ns = len(descs)

    def buf(i):
        return sr.exact(pc.nhwc(p.stage_tensor(i), pick))

    def stage_input(i):
        d = descs[i - 1]
        t = buf(i - 1)
        if d['skip_src'] >= 0 and d['skip_mode']:
            t = sr.concat(t, buf(d['skip_src']))
        return t

    for i in range(ns - 1):
        d = descs[i]
        adds = d['skip_src'] >= 0 and not d['skip_mode']
        if only_adds and not adds:
            continue
        if d['kind'] == sr.STEM:
            chk(pc.nhwc(p.stage_tensor(0), pick), sr.stem(x_host[pick], *weights[0][3:], d['stride'], d['act']), 'stem')
            continue
        wt = weights[i]
        mid = p.stage_tensor(i, which=1)
        if not only_adds:
            chk(pc.nhwc(mid, pick), sr.depthwise(stage_input(i), *wt[:3], d['ksize'], d['stride'], d['act']),
                'stage %d depthwise' % i)
        out = sr.pointwise(sr.exact(pc.nhwc(mid, pick)), *wt[3:], d['act'], eps=EPS_TF32X3)
        if d['upsample'] and not (fold and i == ns - 2):
            out = sr.upsample(out)
            if adds:
                skip = sr.exact(pc.nhwc(saved[d['skip_src']], pick)) if saved else buf(d['skip_src'])
                out = sr.add(out, skip)
        chk(pc.nhwc(p.stage_tensor(i), pick), out, 'stage %d' % i)
    return ns


def check_head(p, descs, weights, y, pick, chk, fold):
    ns = len(descs)
    hin = sr.exact(pc.nhwc(p.stage_tensor(ns - 2), pick))
    if descs[-2]['skip_src'] >= 0 and descs[-2]['skip_mode']:
        hin = sr.concat(hin, sr.exact(pc.nhwc(p.stage_tensor(descs[-2]['skip_src']), pick)))
    hd = sr.head(hin, *weights[-1][3:], descs[-1]['act'])
    chk(pc.nhwc(y[:, 0], pick), sr.upsample(hd) if fold else hd, 'head')


def assert_split_steps(steps, descs):
    """Every DWPW stage runs dw_kernel + the split-TF32 step; nothing else changed kernels."""
    for i, d in enumerate(descs):
        mine = [s['kernel'] for s in steps if s['stage'] == i]
        if d['kind'] == sr.DWPW:
            assert len(mine) == 2 and mine[0].startswith('dw_kernel<') and mine[1].startswith(TF32X3), (i, mine)
        elif d['kind'] == sr.STEM:
            assert mine == ['stem_kernel'], mine
    for s in steps:
        if s['kernel'].startswith(TF32X3):
            assert s['dw_macs'] == 0 and s['dense_macs'] == s['macs'] > 0


def run_checked(p, descs, weights, x_host, x, y, pick, case, inplace=1):
    """Pass 1 (inplace_skip 0): every stage; pass 2 (inplace_skip 1, with skip adds): the adding stages against pass 1's
    sources, and the two passes' depth maps bitwise equal.  Returns the steps of pass 1 and the depth map."""
    stream = torch.cuda.current_stream().cuda_stream
    fold = p.get_option('fold_head') and descs[-2]['upsample'] and descs[-2]['skip_src'] < 0
    chk = pc.Checker(case, F32)
    p.set_option('inplace_skip', 0)
    p.forward(x, y, stream)
    torch.cuda.synchronize()
    steps = p.steps()
    assert_split_steps(steps, descs)
    check_stages(p, descs, weights, x_host, pick, chk, fold)
    check_head(p, descs, weights, y, pick, chk, fold)
    y0 = y.clone()
    srcs = {d['skip_src'] for d in descs if d['skip_src'] >= 0 and not d['skip_mode']}
    if srcs and inplace:
        saved = {s: p.stage_tensor(s).clone() for s in srcs}
        p.set_option('inplace_skip', 1)
        p.forward(x, y, stream)
        torch.cuda.synchronize()
        assert any('+skip(red)' in s['kernel'] for s in p.steps())
        check_stages(p, descs, weights, x_host, pick, chk, fold, saved=saved, only_adds=True)
        assert torch.equal(y, y0), case                          # inplace_skip 0 and 1 give the same bits
    chk.flush()
    assert chk.zeros < 0.5 * chk.n, (case, chk.zeros / chk.n)
    if any(d['act'] == R6 for d in descs[:-1]):
        assert chk.sixes > 0, case
    return steps, y0


def sweep_plan(descs, n, h, w, seed, opts=None):
    rng = np.random.default_rng(seed)
    x_host = rng.uniform(0.0, 1.0, (n, 3, h, w)).astype(np.float32)
    probe = x_host[:2].astype(np.float64)
    if h * w < 64 * 64:
        probe = np.concatenate([probe, rng.uniform(0.0, 1.0, (6, 3, h, w))])
    weights = ks.make_weights(descs, F32, probe, seed + 1)
    p = fplan.Plan(descs, weights, ['s%d' % i for i in range(len(descs))], n, h, w, F32, 0)
    p.set_option('tf32x3', 1)
    for k, v in (opts or {}).items():
        p.set_option(k, v)
    x = torch.from_numpy(x_host).cuda()
    y = torch.empty((n, 1, h, w), dtype=F32, device='cuda')
    return p, weights, x_host, x, y


def tails_net():
    """c_in mod 32 = 8, 16, 24 and c_out tails 8, 40, 72, 136, 264; stride-2 blocks, two skip adds, ReLU and ReLU6."""
    b = ks.blk
    return ks.link([ks.stem(16, 2, R6), b(40, 3, 1, R6), b(72, 3, 2, R), b(136, 3, 1, R6), b(264, 3, 2, R6),
                    b(136, 5, 1, R, 1, 3), b(40, 5, 1, R6, 1, 1), b(8, 5, 1, R, 1), ks.head(R)])


CASES = {
    # name: (descs, n, h, w, options)
    'tails_3x64x96': (tails_net, 3, 64, 96, {}),
    'tails_unfolded_2x32x64': (tails_net, 2, 32, 64, {'fold_head': 0}),
    'enc_dec_2x64x64': (lambda: ks.enc_dec((16, 24, 48, 56, 80, 24)), 2, 64, 64, {}),
    'deep_1x1_bottom_5x32x32': (lambda: ks.deep(3), 5, 32, 32, {}),             # tiles span images
    'deep_1x2_bottom_3x32x64': (lambda: ks.deep(5), 3, 32, 64, {}),
    'concat_2x64x64': (ks.concat_net, 2, 64, 64, {}),                           # a concat slice
}


@pytest.mark.parametrize('case', list(CASES))
def test_stage_sweep(case, built_lib):
    fn, n, h, w, opts = CASES[case]
    descs = fn()
    p, weights, x_host, x, y = sweep_plan(descs, n, h, w, seed=len(case), opts=opts)
    steps, _ = run_checked(p, descs, weights, x_host, x, y, list(range(n)), case)
    fold = opts.get('fold_head', 1)
    kern = ' '.join(s['kernel'] for s in steps)
    assert ('head_kernel<up2x>' in kern) == bool(fold), kern
    assert 'relu6]' in kern or 'relu6,' in kern
    p.close()


@pytest.mark.parametrize('bn', ['64', '128'])
def test_stage_sweep_pinned_bn(bn, built_lib, monkeypatch):
    """Every bn the planner offers (64, 128), pinned, on the tails network; and the depth map does not depend on it."""
    monkeypatch.setenv('FD_CONV_BN', bn)
    descs = tails_net()
    p, weights, x_host, x, y = sweep_plan(descs, 3, 64, 96, seed=11)
    steps, y_bn = run_checked(p, descs, weights, x_host, x, y, [0, 1, 2], 'bn' + bn)
    assert all(',bn%s,' % bn in s['kernel'] for s in steps if s['kernel'].startswith(TF32X3))
    monkeypatch.delenv('FD_CONV_BN')
    p.set_option('tf32x3', 0)
    p.set_option('tf32x3', 1)                      # rebuilt with the planner's own choice
    y2 = torch.empty_like(y)
    p.forward(x, y2, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert torch.equal(y2, y_bn)
    p.close()


def test_bitwise_properties(built_lib, monkeypatch):
    """A batch equals its images run alone; graph on equals graph off; the output does not depend on the tile."""
    descs = tails_net()
    n, h, w = 3, 64, 96
    p, weights, x_host, x, y = sweep_plan(descs, n, h, w, seed=5)
    stream = torch.cuda.current_stream().cuda_stream
    p.forward(x, y, stream)
    torch.cuda.synchronize()
    ref = y.clone()
    p.set_option('graph', 0)
    p.forward(x, y, stream)
    torch.cuda.synchronize()
    assert torch.equal(y, ref)
    p.set_option('graph', 1)
    for t in ('0', '1', '3'):                      # 1x8x16, 2x8x8, 8x4x4 tiles
        monkeypatch.setenv('FD_CONV_TILE', t)
        p.set_option('tf32x3', 0)
        p.set_option('tf32x3', 1)
        p.forward(x, y, stream)
        torch.cuda.synchronize()
        assert torch.equal(y, ref), t
    monkeypatch.delenv('FD_CONV_TILE')
    p1 = fplan.Plan(descs, weights, ['s%d' % i for i in range(len(descs))], 1, h, w, F32, 0)
    p1.set_option('tf32x3', 1)
    y1 = torch.empty((1, 1, h, w), dtype=F32, device='cuda')
    for i in range(n):
        p1.forward(x[i:i + 1].contiguous(), y1, stream)
        torch.cuda.synchronize()
        assert torch.equal(y1, ref[i:i + 1]), i
    p.close()
    p1.close()


# ---------------------------------------------------------------------------------------------------------------------
# the modules under torch.set_float32_matmul_precision
# ---------------------------------------------------------------------------------------------------------------------
def _golden_model(name):
    import models
    fx = np.load(os.path.join(GOLDEN, name + '.npz'))
    n, h, w = (int(v) for v in fx['shape'])
    if name.startswith('skipadd'):
        widths = (tuple(int(v) for v in fx['widths_enc']), tuple(int(v) for v in fx['widths_dec']))
        m = models.MobileNetSkipAdd((h, w), pretrained=False, widths=widths)
        m.load_state_dict(synthetic.synthetic_state_dict(widths, seed=int(fx['wseed']), recipe='hot'))
    elif name.startswith('skipconcat'):
        m = models.MobileNetSkipConcat((h, w), pretrained=False)
        m.load_state_dict(synthetic.synthetic_state_dict(seed=int(fx['wseed']), skip='concat'))
    else:
        m = models.MobileNet('nnconv5dw', (h, w), pretrained=False)
        m.load_state_dict(synthetic.to_mobilenet_keys(synthetic.synthetic_state_dict(seed=int(fx['wseed']))))
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


GOLDENS = ['skipadd_stock_2x64x96', 'skipadd_pruned_2x64x96', 'skipconcat_stock_2x64x96', 'nnconv5dw_stock_2x64x96',
           'skipadd_stock_1x224x224']


@pytest.mark.parametrize('name', GOLDENS)
def test_golden_under_high(name, built_lib, precision):
    m, x, want = _golden_model(name)
    precision('high')
    y = _forward(m, x)
    assert rel_err(y.float().cpu(), want) <= 1e-3
    steps = _engine_steps(m)
    descs, _, _ = fplan.describe(m)
    assert_split_steps(steps, descs)
    assert m.__dict__['_fd_engine'].options == {}


def test_default_unchanged(built_lib, precision):
    """'highest': the fp32 plan's step names are today's and its output is bitwise the explicit tf32x3=0 plan's;
    a 16-bit plan ignores tf32x3."""
    m, x, _ = _golden_model('skipadd_stock_2x64x96')
    precision('highest')
    y = _forward(m, x)
    names = [s['kernel'] for s in _engine_steps(m)]
    assert not any('tf32x3' in k for k in names)
    assert names[0] == 'stem_kernel' and names[-1] == 'head_kernel<up2x>'
    assert set(names[1:-1]) == {'dw_kernel<3>', 'dw_kernel<5>', 'pw_kernel'}
    eng = m.__dict__['_fd_engine']
    assert eng.options == {}
    eng.set_option('tf32x3', 0)
    y0 = _forward(m, x)
    assert torch.equal(y, y0)
    assert [s['kernel'] for s in _engine_steps(m)] == names
    mh = m.half()
    mh.__dict__.pop('_fd_engine', None)
    outs = []
    for v in (0, 1):
        eng = SkipAddEngine(mh)
        eng.set_option('tf32x3', v)
        mh.__dict__['_fd_engine'] = eng
        outs.append((_forward(mh, x.half()), [s['kernel'] for s in _engine_steps(mh)]))
    assert torch.equal(outs[0][0], outs[1][0]) and outs[0][1] == outs[1][1]


def test_switching_and_weight_updates(built_lib, precision):
    """Switching the precision between two calls switches the kernels without a new engine; a weight update under
    'high' is picked up; an explicit set_option wins over the precision."""
    m, x, want = _golden_model('skipadd_stock_2x64x96')
    precision('highest')
    y_hi = _forward(m, x)
    eng = m.__dict__['_fd_engine']
    assert not any('tf32x3' in s['kernel'] for s in _engine_steps(m))
    precision('high')
    y_tf = _forward(m, x)
    assert m.__dict__['_fd_engine'] is eng
    assert any('tf32x3' in s['kernel'] for s in _engine_steps(m))
    assert rel_err(y_tf.cpu(), want) <= 1e-3 and not torch.equal(y_tf, y_hi)
    precision('medium')
    assert torch.equal(_forward(m, x), y_tf)
    precision('highest')
    assert torch.equal(_forward(m, x), y_hi)
    # weight update under 'high': scale one decoder BN in place; the engine must see it and match the reference module
    precision('high')
    with torch.no_grad():
        m.decode_conv3[1][1].weight.mul_(1.5)
    y_new = _forward(m, x)
    assert not torch.equal(y_new, y_tf)
    eng0 = SkipAddEngine(m)
    eng0.set_option('tf32x3', 1)
    m.__dict__['_fd_engine'] = eng0
    assert torch.equal(_forward(m, x), y_new)
    eng0.set_option('tf32x3', 0)                     # explicit: wins over 'high'
    _forward(m, x)
    assert not any('tf32x3' in s['kernel'] for s in _engine_steps(m))


def test_production_size_every_image(built_lib, precision):
    """Stock widths, b64 at 224^2, fp32 under 'high': the plan the module builds, every stage of every image against
    the interval (the split-TF32 steps with eps = EPS_TF32X3), in chunks of 8 images."""
    import models
    t0 = time.perf_counter()
    n, h, w = 64, 224, 224
    m = models.MobileNetSkipAdd((h, w), pretrained=False, widths=synthetic.STOCK_WIDTHS)
    m.load_state_dict(synthetic.synthetic_state_dict(synthetic.STOCK_WIDTHS, seed=1))
    m = m.eval().cuda()
    x = synthetic.synthetic_input(n, h, w, seed=0).cuda()
    precision('high')
    y = _forward(m, x)
    p = m.__dict__['_fd_engine'].plan_for(x)
    descs, weights, _ = fplan.describe(m)
    descs = [dict({'skip_mode': 0}, **d) for d in descs]
    x_host = x.cpu().numpy()
    fold = descs[-2]['upsample'] and descs[-2]['skip_src'] < 0
    stream = torch.cuda.current_stream().cuda_stream
    chk = pc.Checker('production fp32 tf32x3', F32)
    p.set_option('inplace_skip', 0)
    p.forward(x, y, stream)
    torch.cuda.synchronize()
    assert_split_steps(p.steps(), descs)
    for k in range(0, n, pc.CHUNK):
        pick = list(range(k, min(n, k + pc.CHUNK)))
        check_stages(p, descs, weights, x_host, pick, chk, fold)
        check_head(p, descs, weights, y, pick, chk, fold)
    chk.flush()
    y0 = y.clone()
    p.set_option('inplace_skip', 1)                  # the module's own plan as it runs: adds in place, same bits
    p.forward(x, y, stream)
    torch.cuda.synchronize()
    assert torch.equal(y, y0)
    print('\nproduction fp32 tf32x3 b64 224x224: %d tensors checked in %.1f s' % (len(chk.results), time.perf_counter() - t0))
