"""GPU tests of the DECONV / UPCONV stages: conv_tc_kernel's four-phase path (path 1) and convt_kernel (path 0).

* goldens of the reference's MobileNet('upconv') / ('deconv<k>') end to end through Plan, all three dtypes, both paths.
  Storage-emulated conditioning, measured on the CPU (tests/convt_ref.torch_forward with storage= against the fp32
  golden): fp16 1.6e-3 .. 2.5e-3 at 2x64x96 and 4.3e-3 / 4.5e-3 (upconv5 / deconv5) at 1x224x224; bf16 1.6e-2 .. 2.1e-2 and
  3.3e-2 / 3.8e-2.  All are inside the NNConv5 end-to-end tolerances (fp16 1e-2, bf16 1e-1, fp32 1e-3), which hold for
  every golden here;
* module routing: fp16 / bf16 MobileNet('deconv5') / ('upconv') build the engine and see weight updates, fp32 does not;
* stage-list validation of the two kinds;
* a per-stage sweep against the fp64 interval reference (tests/convt_ref.py), computed from the GPU's own input tensors:
  deconv k = 3, 5, 7, 9 and upconv5, channel tails 8/24/40 mod 64, c_out 8..520, input maps 1x1, 1x2, 2x3, 7x7 and odd
  sizes, tiles that cross images, ReLU and ReLU6, DECONV next to CONV, every bn, both phase groupings, all dtypes on path 0;
* bitwise properties: a batch equals its images run alone, graph on == graph off, and the output does not depend on the
  tile, bn or phase grouping.
"""
import os

import numpy as np
import pytest
import torch

import convt_ref as cr
import dense_ref as dr
from conftest import GOLDEN, rel_err
from fastdepth_b200 import synthetic
from oracle import stage_ref as sr

pytestmark = pytest.mark.gpu

TOL = {torch.float32: 1e-3, torch.float16: 1e-2, torch.bfloat16: 1e-1}
SEEN = set()          # conv_tc_kernel instances the DECONV / UPCONV sweep ran: (dtype, bn, act)
GOLDENS = ['%s_stock_2x64x96' % d for d in ('upconv5', 'deconv3', 'deconv5', 'deconv7', 'deconv9')] + \
    ['upconv5_stock_1x224x224', 'deconv5_stock_1x224x224']


def _model(decoder, dtype, hw, wseed=1):
    import models
    m = models.MobileNet(decoder, hw, pretrained=False)
    m.load_state_dict(synthetic.synthetic_convt_state_dict(decoder, seed=wseed))
    return m.eval().cuda().to(dtype)


def _kernel_prefix(decoder, path, dtype):
    tag = 'upconv5' if decoder == 'upconv' else decoder
    return 'conv_tc_kernel<%s,' % tag if (path == 1 and dtype != torch.float32) else 'convt_kernel<%s>' % tag


# ------------------------------------------------------------------------------------------------ goldens + routing
@pytest.mark.parametrize('name', GOLDENS)
@pytest.mark.parametrize('dtype', [torch.float32, torch.float16, torch.bfloat16])
@pytest.mark.parametrize('path', [0, 1])
def test_golden_convt(name, dtype, path):
    from fastdepth_b200 import plan as _plan
    fx = np.load(os.path.join(GOLDEN, name + '.npz'))
    n, h, w = (int(v) for v in fx['shape'])
    dec = str(fx['decoder'])
    m = _model(dec, dtype, (h, w), int(fx['wseed']))
    x = synthetic.synthetic_input(n, h, w, seed=int(fx['xseed'])).cuda().to(dtype)
    p = _plan.Plan.from_module(m, n, h, w, dtype, 0)
    p.set_option('path', path)
    y = torch.empty((n, 1, h, w), dtype=dtype, device='cuda')
    p.forward(x, y, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    kernels = [s['kernel'] for s in p.steps()]
    assert sum(k.startswith(_kernel_prefix(dec, path, dtype)) for k in kernels) == 5, kernels
    assert kernels[-1] == 'head_kernel'                   # the map is already at full resolution: no folded head
    assert rel_err(y.float().cpu(), torch.from_numpy(fx['output'])) <= TOL[dtype]
    p.close()


@pytest.mark.parametrize('decoder', ['deconv5', 'upconv'])
@pytest.mark.parametrize('dtype', [torch.float16, torch.bfloat16])
def test_module_routes_16bit_convt_decoder(decoder, dtype):
    tag = 'upconv5' if decoder == 'upconv' else decoder
    fx = np.load(os.path.join(GOLDEN, '%s_stock_2x64x96.npz' % tag))
    n, h, w = (int(v) for v in fx['shape'])
    m = _model(decoder, dtype, (h, w))
    x = synthetic.synthetic_input(n, h, w, seed=int(fx['xseed'])).cuda().to(dtype)
    with torch.no_grad():
        y = m(x)
    torch.cuda.synchronize()
    assert '_fd_engine' in m.__dict__
    steps = next(iter(m.__dict__['_fd_engine'].plans.values())).steps()
    assert sum(s['kernel'].startswith(_kernel_prefix(decoder, 1, dtype)) for s in steps) == 5
    assert rel_err(y.float().cpu(), torch.from_numpy(fx['output'])) <= TOL[dtype]
    with torch.no_grad():                                  # a weight update through the module is picked up
        blk = m.decoder.upconv3[1] if decoder == 'upconv' else m.decoder.convt3[0]
        blk.weight.mul_(0.5)
        y2 = m(x)
        want = cr.torch_forward({k: v.float().cpu() for k, v in m.state_dict().items()}, x.float().cpu(), decoder,
                                storage=dtype)
    torch.cuda.synchronize()
    assert not torch.equal(y, y2)
    assert rel_err(y2.float().cpu(), want) <= TOL[dtype]


@pytest.mark.parametrize('decoder', ['deconv3', 'upconv'])
def test_fp32_convt_decoder_stays_on_pytorch(decoder):
    tag = 'upconv5' if decoder == 'upconv' else decoder
    fx = np.load(os.path.join(GOLDEN, '%s_stock_2x64x96.npz' % tag))
    n, h, w = (int(v) for v in fx['shape'])
    m = _model(decoder, torch.float32, (h, w))
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        with torch.no_grad():
            y = m(synthetic.synthetic_input(n, h, w, seed=int(fx['xseed'])).cuda())
    finally:
        torch.backends.cudnn.allow_tf32 = tf32
    assert '_fd_engine' not in m.__dict__
    assert rel_err(y.cpu(), torch.from_numpy(fx['output'])) <= 1e-3


# ------------------------------------------------------------------------------------------------ stage sweep
def _rand_stage_list(seed, dtype, down, decs, act_dec, c0=16):
    """STEM (stride 2, c0) -> `down` stride-2 DWPW blocks -> decoder stages (kind, c_out, k) -> HEAD.  A CONV stage
    upsamples x2, as do DECONV / UPCONV."""
    rng = np.random.Generator(np.random.PCG64(seed))

    def rep(a):
        return torch.from_numpy(np.asarray(a, np.float32)).to(dtype).float().numpy() if dtype != torch.float32 else \
            np.asarray(a, np.float32)

    def affine(c, lo=0.5, hi=1.5):
        return rng.uniform(lo, hi, c).astype(np.float32), rng.normal(0.2, 0.3, c).astype(np.float32)

    descs, wts = [], []
    descs.append(dict(kind=sr.STEM, c_in=3, c_out=c0, ksize=3, stride=2, act=sr.RELU6, upsample=0, skip_src=-1, skip_mode=0))
    s, b = affine(c0)
    wts.append((None, None, None, rep(rng.normal(0, np.sqrt(2 / 27), (c0, 27))), s, b))
    c = c0
    for _ in range(down):
        descs.append(dict(kind=sr.DWPW, c_in=c, c_out=c, ksize=3, stride=2, act=sr.RELU6, upsample=0, skip_src=-1, skip_mode=0))
        s1, b1 = affine(c)
        s2, b2 = affine(c)
        wts.append((rep(rng.normal(0, np.sqrt(2 / 9), (c, 9))), s1, b1, rep(rng.normal(0, np.sqrt(1 / c), (c, c))), s2, b2))
    for kind, co, k in decs:
        conv = kind == dr.CONV
        descs.append(dict(kind=kind, c_in=c, c_out=co, ksize=k, stride=1 if conv else 2, act=act_dec, upsample=1 if conv else 0,
                          skip_src=-1, skip_mode=0))
        s, b = affine(co, 0.3, 0.9)
        fan = c * k * k if conv else c * k * k / 4.0            # a phase sums about a quarter of the taps
        wts.append((None, None, None, rep(rng.uniform(-1, 1, (co, c * k * k)) * np.sqrt(3.0 / fan)), s, b))
        c = co
    descs.append(dict(kind=sr.HEAD, c_in=c, c_out=1, ksize=1, stride=1, act=sr.RELU, upsample=0, skip_src=-1, skip_mode=0))
    wts.append((None, None, None, rep(np.abs(rng.normal(0, 1 / np.sqrt(c), (1, c)))), np.ones(1, np.float32),
                np.full(1, 1.0, np.float32)))
    return descs, wts


D, U, C = cr.DECONV, cr.UPCONV, dr.CONV
F16, BF16, F32 = torch.float16, torch.bfloat16, torch.float32


def _dec(kind, k, cos):
    return tuple((kind, co, k) for co in cos)


# (name, dtype, path, n, h, w, down, decoder stages, act, env)
CASES = [
    ('d3_tails_2x3', F16, 1, 3, 64, 96, 4, _dec(D, 3, (40, 88, 264, 72, 8)), sr.RELU, {}),
    ('d5_tails_bf16', BF16, 1, 3, 64, 96, 4, _dec(D, 5, (40, 88, 264, 72, 8)), sr.RELU, {}),
    ('d7_1x2_relu6', F16, 1, 2, 32, 64, 4, _dec(D, 7, (24, 136, 40, 16, 8)), sr.RELU6, {}),
    ('d9_1x2_bf16_relu6', BF16, 1, 2, 32, 64, 4, _dec(D, 9, (24, 136, 40, 16, 8)), sr.RELU6, {}),
    ('u5_tails', F16, 1, 3, 64, 96, 4, _dec(U, 5, (40, 88, 264, 72, 8)), sr.RELU, {}),
    ('u5_1x1_bf16_relu6', BF16, 1, 4, 32, 32, 4, _dec(U, 5, (24, 72, 40, 16, 8)), sr.RELU6, {}),
    ('d5_7x7_c520', F16, 1, 2, 224, 224, 4, _dec(D, 5, (520, 32, 16, 8, 8)), sr.RELU, {}),
    ('d9_odd_7x5', BF16, 1, 5, 224, 160, 4, _dec(D, 9, (72, 24, 40, 8, 8)), sr.RELU, {}),
    ('d3_1x1_odd', F16, 1, 3, 32, 32, 4, _dec(D, 3, (200, 24, 8, 8, 8)), sr.RELU6, {}),
    ('mixed_conv_deconv', F16, 1, 3, 64, 96, 4, ((C, 40, 5), (D, 88, 5), (C, 24, 3), (U, 72, 5), (D, 8, 7)), sr.RELU, {}),
    ('pairs_f16', F16, 1, 3, 64, 96, 4, _dec(D, 5, (64, 128, 64, 32, 8)), sr.RELU, {'FD_CONV_PHASE_GROUP': '2'}),
    ('singles_bf16', BF16, 1, 3, 64, 96, 4, _dec(U, 5, (64, 128, 64, 32, 8)), sr.RELU6, {'FD_CONV_PHASE_GROUP': '1'}),
] + [
    ('bn%s_%s_%s' % (bn, 'f16' if dt == F16 else 'bf16', 'r6' if a == sr.RELU6 else 'r'), dt, 1, 2, 32, 64, 4,
     _dec(D if a == sr.RELU else U, 5 if a == sr.RELU6 else 7, (cos, 72, 16, 8, 8)), a, {'FD_CONV_BN': bn})
    for bn, cos in (('64', 64), ('128', 136), ('256', 264)) for dt in (F16, BF16) for a in (sr.RELU, sr.RELU6)
] + [
    ('path0_f32', F32, 0, 2, 64, 96, 4, ((D, 40, 3), (D, 88, 5), (U, 24, 5), (D, 16, 7), (D, 8, 9)), sr.RELU, {}),
    ('path0_f16', F16, 0, 2, 32, 64, 4, ((D, 24, 9), (U, 72, 5), (D, 40, 7), (C, 16, 5), (D, 8, 3)), sr.RELU6, {}),
    ('path0_bf16', BF16, 0, 3, 64, 96, 4, ((U, 40, 5), (D, 88, 5), (D, 24, 3), (D, 16, 9), (U, 8, 5)), sr.RELU, {}),
]


def _run_plan(descs, wts, n, h, w, dtype, opts, env, x):
    from fastdepth_b200 import plan as _plan
    saved = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        p = _plan.Plan(descs, wts, ['s%d' % i for i in range(len(descs))], n, h, w, dtype, 0)
        for k, v in opts.items():
            p.set_option(k, v)
        y = torch.empty((n, 1, h, w), dtype=dtype, device='cuda')
        p.forward(x, y, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    return p, y


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_convt_stage_sweep(case):
    name, dtype, path, n, h, w, down, decs, act, env = case
    descs, wts = _rand_stage_list(sum(map(ord, name)), dtype, down, decs, act)
    x = synthetic.synthetic_input(n, h, w, seed=3).cuda().to(dtype)
    p, y = _run_plan(descs, wts, n, h, w, dtype, {'path': path, 'graph': 0}, env, x)
    for s in p.steps():
        d = descs[s['stage']]
        if d['kind'] not in (D, U):
            continue
        kn, tag = s['kernel'], '%s%d' % ('deconv' if d['kind'] == D else 'upconv', d['ksize'])
        if path == 1 and dtype != F32:
            assert kn.startswith('conv_tc_kernel<%s,' % tag), kn
            if 'FD_CONV_BN' in env:
                assert ',bn%s,' % env['FD_CONV_BN'] in kn, kn
            if 'FD_CONV_PHASE_GROUP' in env:
                assert (',4ph2>' in kn) == (env['FD_CONV_PHASE_GROUP'] == '2'), kn
            bn = int(kn.split(',bn')[1].split(',')[0])
            SEEN.add((str(dtype), bn, 'relu6' if act == sr.RELU6 else 'relu'))
        else:
            assert kn == 'convt_kernel<%s>' % tag, kn
        assert s['dw_macs'] == 0 and s['dense_macs'] == s['macs'] > 0
    hh, ww = h >> (down + 1), w >> (down + 1)
    for i, d in enumerate(descs):
        if d['kind'] == sr.HEAD:
            break
        if d['kind'] not in (D, U, C):
            continue
        inp = sr.exact(p.stage_tensor(i - 1))
        assert inp.c.shape[1:3] == (hh, ww), (i, inp.c.shape)
        got = p.stage_tensor(i)
        if d['kind'] == C:
            iv = sr.upsample(sr.quantize(dr.conv(inp, wts[i][3], wts[i][4], wts[i][5], d['ksize'], d['act']), dtype))
        else:
            iv = sr.quantize(cr.convt(inp, wts[i][3], wts[i][4], wts[i][5], d['kind'], d['ksize'], d['act']), dtype)
        assert tuple(got.shape) == (n, 2 * hh, 2 * ww, d['c_out'])
        det = sr.check(got, iv, dtype, '%s stage %d' % (name, i))
        if dtype != F32:
            assert det >= 0.5, (name, i, det)
        print('%s stage %d %s: determined %.3f' % (name, i, (d['kind'], d['ksize'], d['c_in'], d['c_out'], hh, ww), det))
        hh, ww = 2 * hh, 2 * ww
        with pytest.raises(RuntimeError):
            p.stage_tensor(i, which=1)                    # no depthwise intermediate
    p.close()


def test_convt_step_bookkeeping():
    """k*k*c_in*c_out MACs per input pixel, all dense; input once + 2h x 2w output once + weights once."""
    descs, wts = _rand_stage_list(1, F16, 4, _dec(D, 7, (40, 24, 16, 8, 8)), sr.RELU)
    p, _ = _run_plan(descs, wts, 2, 64, 96, F16, {}, {}, synthetic.synthetic_input(2, 64, 96, seed=3).cuda().half())
    hh, ww = 2, 3
    for s in p.steps():
        d = descs[s['stage']]
        if d['kind'] != D:
            continue
        px = 2 * hh * ww
        assert s['macs'] == px * 49 * d['c_in'] * d['c_out'] and s['dense_macs'] == s['macs']
        assert s['alg_bytes'] == (px * d['c_in'] + 4 * px * d['c_out']) * 2 + 49 * d['c_in'] * d['c_out'] * 2 + 8 * d['c_out']
        hh, ww = 2 * hh, 2 * ww
    p.close()


def test_convt_tc_coverage():
    """Every conv_tc_kernel instance (dtype x bn x activation) ran a DECONV / UPCONV stage in the sweep above."""
    want = {(str(dt), bn, a) for dt in (F16, BF16) for bn in (64, 128, 256) for a in ('relu', 'relu6')}
    assert want <= SEEN, sorted(want - SEEN)


# ------------------------------------------------------------------------------------------------ validation
def test_convt_stage_validation():
    from fastdepth_b200 import plan as _plan
    descs, wts = _rand_stage_list(2, F16, 4, _dec(D, 5, (40, 24, 16, 8, 8)), sr.RELU)

    def bad(i, msg, **kw):
        ds = [dict(d) for d in descs]
        ds[i].update(kw)
        with pytest.raises(RuntimeError, match=msg):
            _plan.Plan(ds, wts, ['s%d' % j for j in range(len(ds))], 1, 64, 96, F16, 0)

    bad(5, 'a DECONV stage has stride 2', stride=1)
    bad(5, 'a DECONV stage has upsample 0', upsample=1)
    bad(5, 'a DECONV stage takes no skip', skip_src=2)
    bad(5, r'deconv stage needs k in \{3,5,7,9\}', ksize=4)
    bad(5, r'deconv stage needs k in \{3,5,7,9\}', ksize=11)
    bad(6, 'an UPCONV stage has stride 2', kind=U, stride=1)
    bad(6, 'upconv stage needs k 5', kind=U, ksize=3)
    bad(0, r'STEM, \(DWPW\|CONV\|DECONV\|UPCONV\)\.\.\., HEAD', kind=D)
    bad(5, r'STEM, \(DWPW\|CONV\|DECONV\|UPCONV\)', kind=6)
    p, _ = _run_plan(descs, wts, 1, 64, 96, F16, {}, {}, synthetic.synthetic_input(1, 64, 96, seed=3).cuda().half())
    with pytest.raises(RuntimeError, match='fused block kernels only'):
        p.trace_stage(5, torch.empty(1, 1, 64, 96, dtype=F16, device='cuda'), torch.cuda.current_stream().cuda_stream)
    p.close()


# ------------------------------------------------------------------------------------------------ bitwise properties
def _case_plan(env=None, n=3, opts=None, x=None):
    descs, wts = _rand_stage_list(7, F16, 4, ((D, 40, 5), (U, 264, 5), (D, 72, 9), (D, 24, 3), (D, 8, 7)), sr.RELU)
    if x is None:
        x = synthetic.synthetic_input(n, 64, 96, seed=5).cuda().half()
    return _run_plan(descs, wts, x.shape[0], 64, 96, F16, opts or {}, env or {}, x)


def test_convt_batch_equals_images_alone():
    x = synthetic.synthetic_input(3, 64, 96, seed=5).cuda().half()
    _, y = _case_plan(x=x)
    for i in range(3):
        _, yi = _case_plan(x=x[i:i + 1].contiguous())
        assert torch.equal(y[i:i + 1], yi), i


def test_convt_graph_on_equals_graph_off():
    x = synthetic.synthetic_input(3, 64, 96, seed=5).cuda().half()
    _, y0 = _case_plan(x=x, opts={'graph': 0})
    p, y1 = _case_plan(x=x, opts={'graph': 1})
    y2 = torch.empty_like(y1)
    p.forward(x, y2, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert torch.equal(y0, y1) and torch.equal(y1, y2)


def test_convt_result_does_not_depend_on_tile_bn_or_grouping():
    x = synthetic.synthetic_input(3, 64, 96, seed=5).cuda().half()
    _, ref = _case_plan(x=x)
    for env in ({'FD_CONV_PHASE_GROUP': '1'}, {'FD_CONV_PHASE_GROUP': '2'}, {'FD_CONV_TILE': '0'}, {'FD_CONV_TILE': '2'},
                {'FD_CONV_TILE': '4', 'FD_CONV_PHASE_GROUP': '2'}, {'FD_CONV_BN': '64'}, {'FD_CONV_BN': '256'},
                {'FD_CONV_TILE': '3', 'FD_CONV_BN': '128', 'FD_CONV_PHASE_GROUP': '1'}):
        p, y = _case_plan(x=x, env=env)
        assert torch.equal(ref, y), (env, [s['kernel'] for s in p.steps()])
