"""GPU tests of the dense conv stage (FD_STAGE_CONV): conv_tc_kernel (path 1) and conv_kernel (path 0).

* goldens of the reference's MobileNet('nnconv5') end to end, through models.MobileNet and through Plan;
* module routing: fp16 / bf16 MobileNet('nnconv5') builds the engine and sees weight updates, fp32 does not route;
* a per-stage sweep against the fp64 interval reference (tests/dense_ref.py), computed from the GPU's own input tensors:
  k = 3 and 5, channel tails 8/24/40 mod 64, c_out 8..520, maps 1x2 .. 28x28 and odd sizes, ReLU and ReLU6, upsample on
  and off, fold_head 0/1, tiles that cross images, fp16 and bf16 on path 1, all three dtypes on path 0;
* bitwise properties: a batch equals its images run alone, graph on == graph off, the tile / bn choice does not change
  a single bit.
"""
import os

import numpy as np
import pytest
import torch

import dense_ref as dr
from conftest import GOLDEN, rel_err
from fastdepth_b200 import synthetic
from oracle import stage_ref as sr

pytestmark = pytest.mark.gpu

TOL = {torch.float32: 1e-3, torch.float16: 1e-2, torch.bfloat16: 1e-1}
SEEN = set()          # conv_tc_kernel instances the sweep ran: (dtype, bn, act)


# ------------------------------------------------------------------------------------------------ goldens + routing
def _dense_model(dtype, hw, wseed=1):
    import models
    m = models.MobileNet('nnconv5', hw, pretrained=False)
    m.load_state_dict(synthetic.synthetic_nnconv_state_dict(5, seed=wseed))
    return m.eval().cuda().to(dtype)


@pytest.mark.parametrize('name', ['nnconv5_stock_2x64x96', 'nnconv5_stock_1x224x224'])
@pytest.mark.parametrize('dtype', [torch.float32, torch.float16, torch.bfloat16])
@pytest.mark.parametrize('path', [0, 1])
def test_golden_nnconv5_dense(name, dtype, path):
    from fastdepth_b200 import plan as _plan
    fx = np.load(os.path.join(GOLDEN, name + '.npz'))
    n, h, w = (int(v) for v in fx['shape'])
    m = _dense_model(dtype, (h, w), int(fx['wseed']))
    x = synthetic.synthetic_input(n, h, w, seed=int(fx['xseed'])).cuda().to(dtype)
    p = _plan.Plan.from_module(m, n, h, w, dtype, 0)
    p.set_option('path', path)
    y = torch.empty((n, 1, h, w), dtype=dtype, device='cuda')
    p.forward(x, y, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    kernels = [s['kernel'] for s in p.steps()]
    want_kernel = 'conv_tc_kernel<k5' if (path == 1 and dtype != torch.float32) else 'conv_kernel<k5>'
    assert sum(k.startswith(want_kernel) for k in kernels) == 5, kernels
    got, want = y.float().cpu(), torch.from_numpy(fx['output'])
    if n * h * w <= 2 * 64 * 96 or dtype == torch.float32:
        assert rel_err(got, want) <= TOL[dtype]
    else:
        # At 224 x 224 the product's own storage roundings, emulated on the CPU, already land 1.5e-2 (fp16) / 1.2e-1 (bf16)
        # from the fp32 reference on this recipe: no 16-bit implementation with these rounding points meets 1e-2.  The
        # kernels are held to the storage-emulated forward at the end-to-end tolerances instead, and to the reference
        # at the measured storage noise plus margin.
        sd = synthetic.synthetic_nnconv_state_dict(5, seed=int(fx['wseed']))
        emul = dr.torch_forward(sd, synthetic.synthetic_input(n, h, w, seed=int(fx['xseed'])), storage=dtype)
        assert rel_err(got, emul) <= {torch.float16: 1e-2, torch.bfloat16: 8e-2}[dtype]
        assert rel_err(got, want) <= {torch.float16: 2e-2, torch.bfloat16: 1.5e-1}[dtype]
    p.close()


@pytest.mark.parametrize('dtype', [torch.float16, torch.bfloat16])
def test_module_routes_16bit_dense_decoder(dtype):
    fx = np.load(os.path.join(GOLDEN, 'nnconv5_stock_2x64x96.npz'))
    n, h, w = (int(v) for v in fx['shape'])
    m = _dense_model(dtype, (h, w))
    x = synthetic.synthetic_input(n, h, w, seed=int(fx['xseed'])).cuda().to(dtype)
    with torch.no_grad():
        y = m(x)
    torch.cuda.synchronize()
    assert '_fd_engine' in m.__dict__
    steps = next(iter(m.__dict__['_fd_engine'].plans.values())).steps()
    assert sum(s['kernel'].startswith('conv_tc_kernel') for s in steps) == 5
    assert rel_err(y.float().cpu(), torch.from_numpy(fx['output'])) <= TOL[dtype]
    # a weight update through the module is picked up by the next forward
    with torch.no_grad():
        m.decoder.conv3[0].weight.mul_(0.5)
        y2 = m(x)
        want = dr.torch_forward({k: v.float().cpu() for k, v in m.state_dict().items()}, x.float().cpu(), storage=dtype)
    torch.cuda.synchronize()
    assert not torch.equal(y, y2)
    assert rel_err(y2.float().cpu(), want) <= (1e-2 if dtype == torch.float16 else 1e-1)


def test_fp32_dense_decoder_stays_on_pytorch():
    fx = np.load(os.path.join(GOLDEN, 'nnconv5_stock_2x64x96.npz'))
    n, h, w = (int(v) for v in fx['shape'])
    m = _dense_model(torch.float32, (h, w))
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False             # PyTorch's default lets cuDNN run fp32 convs on TF32 (~1e-2 here)
    try:
        with torch.no_grad():
            y = m(synthetic.synthetic_input(n, h, w, seed=int(fx['xseed'])).cuda())
    finally:
        torch.backends.cudnn.allow_tf32 = tf32
    assert '_fd_engine' not in m.__dict__
    assert rel_err(y.cpu(), torch.from_numpy(fx['output'])) <= 1e-3


# ------------------------------------------------------------------------------------------------ stage sweep
def _rand_stage_list(seed, dtype, h, w, down, convs, k, act_dec, c0=16):
    """STEM (stride 2, c0) -> `down` stride-2 DWPW blocks -> CONV stages ((c_out, upsample), ...) -> HEAD."""
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
    for co, up in convs:
        descs.append(dict(kind=dr.CONV, c_in=c, c_out=co, ksize=k, stride=1, act=act_dec, upsample=up, skip_src=-1, skip_mode=0))
        s, b = affine(co, 0.3, 0.9)
        wts.append((None, None, None, rep(rng.uniform(-1, 1, (co, c * k * k)) * np.sqrt(3.0 / (c * k * k))), s, b))
        c = co
    descs.append(dict(kind=sr.HEAD, c_in=c, c_out=1, ksize=1, stride=1, act=sr.RELU, upsample=0, skip_src=-1, skip_mode=0))
    wts.append((None, None, None, rep(np.abs(rng.normal(0, 1 / np.sqrt(c), (1, c)))), np.ones(1, np.float32),
                np.full(1, 1.0, np.float32)))
    return descs, wts


# (name, dtype, path, n, h, w, down, convs, k, act, fold, env)
CASES = [
    ('k5_tails_2x3', torch.float16, 1, 3, 64, 96, 4, ((40, 1), (88, 1), (264, 1), (72, 1), (8, 1)), 5, sr.RELU, 1, {}),
    ('k5_tails_bf16', torch.bfloat16, 1, 3, 64, 96, 4, ((40, 1), (88, 1), (264, 1), (72, 1), (8, 1)), 5, sr.RELU, 0, {}),
    ('k3_1x2_relu6', torch.float16, 1, 2, 32, 64, 4, ((24, 1), (136, 1), (40, 1), (16, 1), (8, 1)), 3, sr.RELU6, 1, {}),
    ('k3_1x2_bf16_relu6', torch.bfloat16, 1, 2, 32, 64, 4, ((24, 1), (136, 1), (40, 1), (16, 1), (8, 1)), 3, sr.RELU6, 0, {}),
    ('k5_7x7_noup', torch.float16, 1, 2, 224, 224, 4, ((64, 0), (520, 1), (32, 1), (16, 1), (8, 1), (8, 1)), 5, sr.RELU, 1, {}),
    ('k5_odd_rows', torch.float16, 1, 5, 224, 160, 4, ((72, 1), (24, 0), (40, 1), (8, 1), (8, 1), (8, 1)), 5, sr.RELU, 0, {}),
    ('bn64_f16', torch.float16, 1, 3, 64, 96, 4, ((64, 1), (128, 1), (64, 1), (32, 1), (8, 1)), 5, sr.RELU, 0, {'FD_CONV_BN': '64'}),
    ('bn64_f16_r6', torch.float16, 1, 2, 32, 64, 4, ((64, 1), (72, 1), (16, 1), (8, 1), (8, 1)), 3, sr.RELU6, 0, {'FD_CONV_BN': '64'}),
    ('bn64_bf16', torch.bfloat16, 1, 3, 64, 96, 4, ((64, 1), (128, 1), (64, 1), (32, 1), (8, 1)), 5, sr.RELU, 0, {'FD_CONV_BN': '64'}),
    ('bn64_bf16_r6', torch.bfloat16, 1, 2, 32, 64, 4, ((64, 1), (72, 1), (16, 1), (8, 1), (8, 1)), 3, sr.RELU6, 0, {'FD_CONV_BN': '64'}),
    ('bn128_f16', torch.float16, 1, 3, 64, 96, 4, ((136, 1), (128, 1), (64, 1), (32, 1), (8, 1)), 5, sr.RELU, 0, {'FD_CONV_BN': '128'}),
    ('bn128_f16_r6', torch.float16, 1, 2, 32, 64, 4, ((200, 1), (72, 1), (16, 1), (8, 1), (8, 1)), 3, sr.RELU6, 0, {'FD_CONV_BN': '128'}),
    ('bn128_bf16', torch.bfloat16, 1, 3, 64, 96, 4, ((136, 1), (128, 1), (64, 1), (32, 1), (8, 1)), 5, sr.RELU, 0, {'FD_CONV_BN': '128'}),
    ('bn128_bf16_r6', torch.bfloat16, 1, 2, 32, 64, 4, ((200, 1), (72, 1), (16, 1), (8, 1), (8, 1)), 3, sr.RELU6, 0, {'FD_CONV_BN': '128'}),
    ('bn256_f16', torch.float16, 1, 3, 64, 96, 4, ((264, 1), (512, 1), (64, 1), (32, 1), (8, 1)), 5, sr.RELU, 0, {'FD_CONV_BN': '256'}),
    ('bn256_f16_r6', torch.float16, 1, 2, 32, 64, 4, ((264, 1), (72, 1), (16, 1), (8, 1), (8, 1)), 3, sr.RELU6, 0, {'FD_CONV_BN': '256'}),
    ('bn256_bf16', torch.bfloat16, 1, 3, 64, 96, 4, ((264, 1), (512, 1), (64, 1), (32, 1), (8, 1)), 5, sr.RELU, 0, {'FD_CONV_BN': '256'}),
    ('bn256_bf16_r6', torch.bfloat16, 1, 2, 32, 64, 4, ((264, 1), (72, 1), (16, 1), (8, 1), (8, 1)), 3, sr.RELU6, 0, {'FD_CONV_BN': '256'}),
    ('tile_8x4x4', torch.float16, 1, 3, 64, 96, 3, ((40, 1), (24, 1), (8, 1), (8, 1)), 5, sr.RELU, 0, {'FD_CONV_TILE': '3'}),
    ('tile_32x2x2', torch.bfloat16, 1, 5, 64, 96, 3, ((40, 1), (24, 1), (8, 1), (8, 1)), 3, sr.RELU6, 0, {'FD_CONV_TILE': '4'}),
    ('path0_f32', torch.float32, 0, 2, 64, 96, 4, ((40, 1), (88, 1), (24, 1), (16, 1), (8, 1)), 5, sr.RELU, 1, {}),
    ('path0_f16', torch.float16, 0, 2, 32, 64, 4, ((24, 1), (72, 1), (40, 1), (16, 1), (8, 1)), 3, sr.RELU6, 0, {}),
    ('path0_bf16', torch.bfloat16, 0, 2, 64, 96, 4, ((40, 1), (88, 1), (24, 0), (16, 1), (8, 1), (8, 1)), 5, sr.RELU, 1, {}),
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
def test_conv_stage_sweep(case):
    name, dtype, path, n, h, w, down, convs, k, act, fold, env = case
    descs, wts = _rand_stage_list(sum(map(ord, name)), dtype, h, w, down, convs, k, act)
    x = synthetic.synthetic_input(n, h, w, seed=3).cuda().to(dtype)
    p, y = _run_plan(descs, wts, n, h, w, dtype, {'path': path, 'fold_head': fold, 'graph': 0}, env, x)
    steps = p.steps()
    conv_steps = [s for s in steps if descs[s['stage']]['kind'] == dr.CONV]
    assert len(conv_steps) == len(convs)
    for s in conv_steps:
        kn = s['kernel']
        if path == 1 and dtype != torch.float32:
            assert kn.startswith('conv_tc_kernel<k%d,' % k), kn
            if 'FD_CONV_BN' in env:
                assert ',bn%s,' % env['FD_CONV_BN'] in kn, kn
            bn = int(kn.split(',bn')[1].split(',')[0])
            SEEN.add((str(dtype), bn, 'relu6' if act == sr.RELU6 else 'relu'))
        else:
            assert kn == 'conv_kernel<k%d>' % k, kn
        assert s['dw_macs'] == 0 and s['dense_macs'] == s['macs'] > 0
    last_conv = len(descs) - 2
    for i, d in enumerate(descs):
        if d['kind'] != dr.CONV:
            continue
        inp = sr.exact(p.stage_tensor(i - 1))
        got = p.stage_tensor(i)
        iv = sr.quantize(dr.conv(inp, wts[i][3], wts[i][4], wts[i][5], k, d['act']), dtype)
        if d['upsample'] and not (fold and i == last_conv):
            iv = sr.upsample(iv)
        det = sr.check(got, iv, dtype, '%s stage %d' % (name, i))
        if dtype != torch.float32:
            assert det >= 0.5, (name, i, det)
        print('%s stage %d %s: determined %.3f' % (name, i, (d['c_in'], d['c_out'], tuple(got.shape)), det))
    with pytest.raises(RuntimeError):
        p.stage_tensor(len(descs) - 2, which=1)           # a CONV stage has no depthwise intermediate
    p.close()


def test_conv_tc_coverage():
    """Every conv_tc_kernel instance (dtype x bn x activation) ran in the sweep above."""
    want = {(str(dt), bn, a) for dt in (torch.float16, torch.bfloat16) for bn in (64, 128, 256) for a in ('relu', 'relu6')}
    assert want <= SEEN, sorted(want - SEEN)


# ------------------------------------------------------------------------------------------------ bitwise properties
def _case_plan(env=None, n=3, opts=None, x=None):
    descs, wts = _rand_stage_list(7, torch.float16, 64, 96, 4, ((40, 1), (264, 1), (72, 1), (24, 1), (8, 1)), 5, sr.RELU)
    if x is None:
        x = synthetic.synthetic_input(n, 64, 96, seed=5).cuda().half()
    return _run_plan(descs, wts, x.shape[0], 64, 96, torch.float16, opts or {}, env or {}, x)


def test_batch_equals_images_alone():
    x = synthetic.synthetic_input(3, 64, 96, seed=5).cuda().half()
    _, y = _case_plan(x=x)
    for i in range(3):
        _, yi = _case_plan(x=x[i:i + 1].contiguous())
        assert torch.equal(y[i:i + 1], yi), i


def test_graph_on_equals_graph_off():
    x = synthetic.synthetic_input(3, 64, 96, seed=5).cuda().half()
    _, y0 = _case_plan(x=x, opts={'graph': 0})
    p, y1 = _case_plan(x=x, opts={'graph': 1})
    y2 = torch.empty_like(y1)
    p.forward(x, y2, torch.cuda.current_stream().cuda_stream)      # replayed from the captured graph
    torch.cuda.synchronize()
    assert torch.equal(y0, y1) and torch.equal(y1, y2)


def test_result_does_not_depend_on_tile_choice():
    x = synthetic.synthetic_input(3, 64, 96, seed=5).cuda().half()
    _, ref = _case_plan(x=x)
    for env in ({'FD_CONV_TILE': '0'}, {'FD_CONV_TILE': '1'}, {'FD_CONV_TILE': '2'}, {'FD_CONV_TILE': '4'},
                {'FD_CONV_BN': '64'}, {'FD_CONV_BN': '256'}, {'FD_CONV_TILE': '3', 'FD_CONV_BN': '128'}):
        p, y = _case_plan(x=x, env=env)
        assert torch.equal(ref, y), (env, [s['kernel'] for s in p.steps()])
