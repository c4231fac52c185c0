"""Any resolution up to a plan's pixel capacity from one plan (fd_forward_shape), on the GPU.

A plan built for (N, H, W) runs any (n, h, w) with h, w multiples of 32 and n*h*w <= N*H*W through a step set of its own
(every stage's geometry, planner choices, grids, tensor maps and the chain-kernel decision for that shape) over the front of
the plan's activation buffers and its weights.  Checked here:
* for every model family the engine runs, on plans of capacity 16 @ 480x640, the depth maps of seven shapes from 64 @ 224x224
  down to 1 @ 32x32 (in a shuffled order) equal, bit for bit, those of a plan built for that shape, and nothing is written
  past n*h*w of y;
* conv7..conv11 run as the chain kernel in the 224x224 set and as separate blocks in the 480x640 set, as dedicated plans
  of those shapes decide;
* the workspace grows only by step state, a repeated shape reuses its set, at most 8 sets are held, and new weights or a
  changed option rebuild every set and still give a fresh plan's bits;
* graphs are keyed by shape as well as by (x, y): one x / y storage used alternately at four shapes of the same pixel
  count gives each shape's own result;
* an oversized request, h or w not a multiple of 32 and n = 0 fail with FD_ERR_INVALID and leave the plan usable;
* the engine keeps one plan per (device, dtype): 224x224 b64, 480x640 b16, 224x224 b64 leave one plan of 16 @ 480x640,
  and ``evaluate()`` over batches of mixed resolution gives the sums of dedicated plans, bit for bit.
"""
import ctypes
import random

import pytest
import torch

from fastdepth_b200 import _lib
from fastdepth_b200 import plan as fplan
from fastdepth_b200 import synthetic
from fastdepth_b200.engine import SkipAddEngine
from fastdepth_b200.evaluate import evaluate

pytestmark = pytest.mark.gpu

F16, BF16, F32 = torch.float16, torch.bfloat16, torch.float32
CAP = (16, 480, 640)
SHAPES = [(64, 224, 224), (8, 480, 640), (16, 480, 640), (5, 256, 320), (3, 64, 96), (1, 32, 32), (2, 32, 64)]
STEP_STATE_MAX = 16 << 20          # packed affines / depthwise taps of one step set: far below one activation buffer
GUARD = -7.0                       # the head ends in ReLU: no depth value is negative
FD_ERR_INVALID = -1

# name -> (net, dtype, tf32x3)
CONFIGS = {
    'skipadd_f16': ('stock', F16, 0),
    'skipadd_bf16': ('stock', BF16, 0),
    'skipadd_f32_highest': ('stock', F32, 0),
    'skipadd_f32_tf32x3': ('stock', F32, 1),
    'pruned_f16': ('pruned', F16, 0),
    'skipconcat_f16': ('concat', F16, 0),
    'nnconv5dw_f16': ('nnconv5dw', F16, 0),
    'nnconv5_f16': ('nnconv5', F16, 0),
    'nnconv5_f32_tf32x3': ('nnconv5', F32, 1),
    'deconv5_f16': ('deconv5', F16, 0),
    'upconv_f16': ('upconv', F16, 0),
}


def _module(net, dtype, hw=(224, 224)):
    import models
    if net in ('stock', 'pruned'):
        widths = synthetic.STOCK_WIDTHS if net == 'stock' else synthetic.PRUNED_WIDTHS
        m = models.MobileNetSkipAdd(hw, pretrained=False, widths=widths)
        m.load_state_dict(synthetic.synthetic_state_dict(widths, seed=1))
    elif net == 'concat':
        m = models.MobileNetSkipConcat(hw, pretrained=False)
        m.load_state_dict(synthetic.synthetic_state_dict(seed=1, skip='concat'))
    elif net == 'nnconv5dw':
        m = models.MobileNet('nnconv5dw', hw, pretrained=False)
        m.load_state_dict(synthetic.to_mobilenet_keys(synthetic.synthetic_state_dict(seed=1)))
    elif net == 'nnconv5':
        m = models.MobileNet('nnconv5', hw, pretrained=False)
        m.load_state_dict(synthetic.synthetic_nnconv_state_dict(5, seed=1))
    else:
        m = models.MobileNet(net, hw, pretrained=False)
        m.load_state_dict(synthetic.synthetic_convt_state_dict(net, seed=1))
    return m.eval().cuda().to(dtype)


def _plan(descs, weights, names, shape, dtype, tf32x3, opts=None):
    n, h, w = shape
    p = fplan.Plan(descs, weights, names, n, h, w, dtype, 0)
    if dtype == F32:
        p.set_option('tf32x3', tf32x3)
    for k, v in (opts or {}).items():
        p.set_option(k, v)
    return p


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _input(shape, dtype, seed=0):
    """[n,3,h,w] synthetic images, followed in memory by one image of NaNs"""
    n, h, w = shape
    buf = torch.full(((n + 1) * 3 * h * w,), float('nan'), dtype=dtype, device='cuda')
    buf[:n * 3 * h * w] = synthetic.synthetic_input(n, h, w, seed=seed).reshape(-1).to(dtype)
    return buf[:n * 3 * h * w].view(n, 3, h, w)


def _bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


def _run(p, x, dtype):
    """forward of x on p into a y followed by a guard region of one image; checks the guard"""
    n, _, h, w = x.shape
    buf = torch.full(((n + 1) * h * w,), GUARD, dtype=dtype, device='cuda')
    y = buf[:n * h * w].view(n, 1, h, w)
    p.forward(x, y, _stream())
    torch.cuda.synchronize()
    assert bool((buf[n * h * w:] == GUARD).all()), '%s wrote past its last pixel' % (tuple(x.shape),)
    return y


def _dedicated(descs, weights, names, x, dtype, tf32x3, opts=None, keep=False):
    n, _, h, w = x.shape
    q = _plan(descs, weights, names, (n, h, w), dtype, tf32x3, opts)
    y = torch.empty((n, 1, h, w), dtype=dtype, device='cuda')
    q.forward(x.contiguous(), y, _stream())
    torch.cuda.synchronize()
    if keep:
        return y, q
    q.close()
    return y


@pytest.mark.parametrize('cfg', list(CONFIGS))
def test_every_shape_from_one_plan(cfg, built_lib):
    net, dtype, tf32x3 = CONFIGS[cfg]
    m = _module(net, dtype)
    descs, weights, names = fplan.describe(m)
    p = _plan(descs, weights, names, CAP, dtype, tf32x3)
    xs = {s: _input(s, dtype, seed=i) for i, s in enumerate(SHAPES)}
    p.forward(xs[CAP], torch.empty((CAP[0], 1) + CAP[1:], dtype=dtype, device='cuda'), _stream())
    torch.cuda.synchronize()
    ws = p.workspace_bytes()
    order = list(SHAPES)
    random.Random(cfg).shuffle(order)
    for s in order:
        y = _run(p, xs[s], dtype)
        assert not torch.isnan(y.float()).any(), (cfg, s)
        grown = p.workspace_bytes() - ws
        assert 0 <= grown <= STEP_STATE_MAX and (s != CAP or grown == 0), (s, grown)
        ws += grown
        assert torch.equal(_bits(y), _bits(_dedicated(descs, weights, names, xs[s], dtype, tf32x3))), (cfg, s)
    # the step functions still describe the plan's own (N, H, W)
    assert all(st['macs'] > 0 for st in p.steps())
    assert p.stage_tensor(0).shape[:3] == (CAP[0], CAP[1] // 2, CAP[2] // 2)
    p.close()


def test_chain_kernel_follows_the_set_geometry(built_lib):
    """conv7..conv11 on a 14x14 map (224x224) run as the chain kernel, on 15x20 (480x640) as separate blocks.  Dedicated
    plans name the kernels; on the capacity plan the chain shows by what it leaves alone: it keeps conv8's output in shared
    memory, so the front of conv8's stage buffer keeps a fill in the 224x224 set and is overwritten in the 480x640 set."""
    m = _module('stock', F16)
    descs, weights, names = fplan.describe(m)
    small, large = (64, 224, 224), (8, 480, 640)
    for shape, chained in ((small, True), (large, False)):
        _, q = _dedicated(descs, weights, names, _input(shape, F16), F16, 0, keep=True)
        kernels = [st['kernel'] for st in q.steps()]
        assert any('chain_tc' in k for k in kernels) == chained, (shape, kernels)
        q.close()
    p = _plan(descs, weights, names, CAP, F16, 0)
    c8 = names.index('conv8')
    flat = p.stage_tensor(c8).reshape(-1)
    for shape, chained in ((small, True), (large, False)):
        n, h, w = shape
        used = n * (h // 16) * (w // 16) * flat.numel() // (CAP[0] * (CAP[1] // 16) * (CAP[2] // 16))
        flat.fill_(GUARD)
        torch.cuda.synchronize()
        _run(p, _input(shape, F16), F16)
        kept = bool((flat[:used] == GUARD).all())
        assert kept == chained, (shape, kept)
    p.close()


@pytest.mark.parametrize('cfg', ['skipadd_f16', 'nnconv5_f32_tf32x3'])
def test_repeat_replays_and_rebuilds_on_change(cfg, built_lib):
    net, dtype, tf32x3 = CONFIGS[cfg]
    m = _module(net, dtype)
    descs, weights, names = fplan.describe(m)
    p = _plan(descs, weights, names, CAP, dtype, tf32x3)
    xc = _input(CAP, dtype)
    p.forward(xc, torch.empty((CAP[0], 1) + CAP[1:], dtype=dtype, device='cuda'), _stream())
    two = [(64, 224, 224), (5, 256, 320)]
    xs = {s: _input(s, dtype, seed=3) for s in two}
    ys = {s: torch.empty((s[0], 1) + s[1:], dtype=dtype, device='cuda') for s in two}
    ws0 = p.workspace_bytes()
    for s in two:
        p.forward(xs[s], ys[s], _stream())
    torch.cuda.synchronize()
    first = {s: ys[s].clone() for s in two}
    ws = p.workspace_bytes()
    assert ws > ws0
    for _ in range(3):
        for s in two:
            p.forward(xs[s], ys[s], _stream())
    torch.cuda.synchronize()
    assert p.workspace_bytes() == ws
    assert all(torch.equal(_bits(first[s]), _bits(ys[s])) for s in two)
    # at most 8 step sets: the plan's own (never evicted) and the 7 most recently used, of 12 new shapes (small maps, so
    # that every set makes the same kernel choices and holds about the same step state)
    many = [(n, 64, 96) for n in range(1, 7)] + [(n, 96, 64) for n in range(1, 7)]
    grown = {}
    for s in many:
        before = p.workspace_bytes()
        _run(p, _input(s, dtype), dtype)
        grown[s] = p.workspace_bytes() - before
    assert p.workspace_bytes() - ws0 <= 7 * max(grown.values()), grown
    # new weights: every step set is rebuilt from them
    w2 = [tuple(None if a is None else (a * 0.75 if i == 3 else a) for i, a in enumerate(wt)) for wt in weights]
    p.set_weights(w2)
    for s in two:
        p.forward(xs[s], ys[s], _stream())
        torch.cuda.synchronize()
        assert torch.equal(_bits(ys[s]), _bits(_dedicated(descs, w2, names, xs[s], dtype, tf32x3))), s
    # a changed option: the same
    p.set_option('fold_head', 0)
    for s in two:
        p.forward(xs[s], ys[s], _stream())
        torch.cuda.synchronize()
        assert torch.equal(_bits(ys[s]), _bits(_dedicated(descs, w2, names, xs[s], dtype, tf32x3, {'fold_head': 0}))), s
    p.close()


def test_graphs_are_keyed_by_shape(built_lib):
    """One x and one y storage, used alternately as four shapes of 200704 pixels.  Two of them share n, and two share
    (n, h*w): a graph keyed without h and w would replay the wrong geometry for one of them."""
    m = _module('stock', F16)
    descs, weights, names = fplan.describe(m)
    p = _plan(descs, weights, names, (4, 224, 224), F16, 0)
    assert p.get_option('graph') == 1
    shapes = [(4, 224, 224), (1, 448, 448), (2, 224, 448), (2, 448, 224)]
    px = 4 * 224 * 224
    xbuf = torch.empty(3 * px, dtype=F16, device='cuda')
    ybuf = torch.empty(px, dtype=F16, device='cuda')
    want = {}
    for i, (n, h, w) in enumerate(shapes):
        xs = synthetic.synthetic_input(n, h, w, seed=50 + i).cuda().half()
        want[(n, h, w)] = (xs, _dedicated(descs, weights, names, xs, F16, 0))
    for _ in range(3):
        for s in shapes:
            n, h, w = s
            x = xbuf.view(n, 3, h, w)
            y = ybuf.view(n, 1, h, w)
            x.copy_(want[s][0])
            p.forward(x, y, _stream())
            torch.cuda.synchronize()
            assert torch.equal(_bits(y), _bits(want[s][1])), s
    p.close()


def test_invalid_shapes(built_lib):
    m = _module('stock', F16, (64, 96))
    descs, weights, names = fplan.describe(m)
    p = fplan.Plan(descs, weights, names, 4, 64, 96, F16, 0)
    lib = _lib.load()
    x = _input((4, 64, 96), F16)
    y = torch.empty((4, 1, 64, 96), dtype=F16, device='cuda')

    def call(n, h, w):
        return lib.fd_forward_shape(p.handle, n, h, w, x.data_ptr(), y.data_ptr(), _stream())

    for n, h, w in ((5, 64, 96), (1, 160, 160), (3, 96, 96)):           # 4*64*96 = 24576 pixels
        assert call(n, h, w) == FD_ERR_INVALID, (n, h, w)
        msg = lib.fd_last_error().decode()
        assert '24576 pixels' in msg and '4 x 64 x 96' in msg, msg
    for n, h, w in ((1, 48, 64), (1, 64, 80), (0, 64, 96), (-1, 64, 96), (1, 0, 64)):
        assert call(n, h, w) == FD_ERR_INVALID, (n, h, w)
    with pytest.raises(RuntimeError, match='multiples of 32'):
        p.forward(torch.empty((1, 3, 40, 64), dtype=F16, device='cuda'), y, _stream())
    # the plan is still usable, at its own shape and another
    for s in ((4, 64, 96), (2, 96, 64)):
        xs = _input(s, F16, seed=1)
        assert torch.equal(_bits(_run(p, xs, F16)), _bits(_dedicated(descs, weights, names, xs, F16, 0))), s
    p.close()


def test_engine_keeps_one_plan_across_resolutions(built_lib):
    m = _module('stock', F16)
    descs, weights, names = fplan.describe(m)
    eng = SkipAddEngine(m)
    m.__dict__['_fd_engine'] = eng
    xs = {s: synthetic.synthetic_input(*s, seed=9).cuda().half() for s in ((64, 224, 224), (16, 480, 640))}
    live = [(64, 224, 224), (16, 480, 640), (16, 480, 640)]
    with torch.no_grad():
        for s, cap in zip([(64, 224, 224), (16, 480, 640), (64, 224, 224)], live):
            y = m(xs[s])
            torch.cuda.synchronize()
            assert len(eng.plans) == 1
            p = next(iter(eng.plans.values()))
            assert (p.n, p.h, p.w) == cap, s
            assert torch.equal(_bits(y), _bits(_dedicated(descs, weights, names, xs[s], F16, 0))), s


def test_evaluate_mixed_resolutions(built_lib):
    """batches of 224x224 and 480x640 (and a short one of each) through ``evaluate()``: one plan, and the 11 sums of
    dedicated plans per shape, bit for bit."""
    m = _module('stock', F16)
    descs, weights, names = fplan.describe(m)
    gen = torch.Generator().manual_seed(5)
    shapes = [(32, 224, 224), (8, 480, 640), (32, 224, 224), (5, 480, 640), (14, 224, 224), (8, 480, 640)]
    batches = [(synthetic.synthetic_input(*s, seed=100 + i), 0.5 + 9.5 * torch.rand(s[0], 1, s[1], s[2], generator=gen))
               for i, s in enumerate(shapes)]
    eng = SkipAddEngine(m)
    m.__dict__['_fd_engine'] = eng
    _, sums = evaluate(m, batches, 'cuda', return_sums=True)
    assert len(eng.plans) == 1
    p = next(iter(eng.plans.values()))
    assert (p.n, p.h, p.w) == (8, 480, 640)
    want = torch.zeros(fplan.N_METRICS, dtype=torch.float64, device='cuda')
    plans = {}
    for inp, tgt in batches:
        s = (inp.shape[0], inp.shape[2], inp.shape[3])
        if s not in plans:
            plans[s] = _plan(descs, weights, names, s, F16, 0)
        pred = torch.empty((s[0], 1, s[1], s[2]), dtype=F16, device='cuda')
        plans[s].forward(inp.cuda().half(), pred, _stream())
        fplan.metrics_accumulate(pred, tgt.cuda(), want)
    torch.cuda.synchronize()
    for q in plans.values():
        q.close()
    assert sums[-1].item() == sum(s[0] for s in shapes)
    assert torch.equal(sums, want), (sums, want)
