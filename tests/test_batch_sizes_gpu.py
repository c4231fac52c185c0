"""Any batch size up to a plan's capacity from one plan (fd_forward_batch), on the GPU.

A plan built for N images runs the first n <= N through a step set of its own (planner choices, grids, tensor maps for n)
over the plan's activation buffers and weights.  Checked here, on plans of capacity 64 at 224x224 for every model family the
engine runs:
* the depth maps of n in {1, 5, 14, 63, 64} (in a shuffled order) equal, bit for bit, those of a plan built for n and the
  first n rows of the capacity run on the same inputs;
* nothing is written past image n of y (a guard region right after it keeps its fill);
* the workspace grows only by step state, never by activation buffers or weights;
* a repeated size reuses its step set (the workspace does not move) and the plan holds at most 8 step sets; new weights
  or a changed option rebuild every step set and give the same bits as a fresh plan;
* n = 0 and n = N + 1 fail with a message naming the capacity;
* the engine keeps one plan per (device, H, W, dtype): b64, b14, b64 hold one plan of 64; a b80 call replaces it with one
  of 80; ``evaluate()`` over 654 images (ten batches of 64 and a tail of 14) gives the sums of dedicated plans, bit for bit.
"""
import random

import pytest
import torch

from fastdepth_b200 import plan as fplan
from fastdepth_b200 import synthetic
from fastdepth_b200.engine import SkipAddEngine
from fastdepth_b200.evaluate import evaluate

pytestmark = pytest.mark.gpu

F16, BF16, F32 = torch.float16, torch.bfloat16, torch.float32
CAP, H, W = 64, 224, 224
SIZES = [1, 5, 14, 63, 64]
STEP_STATE_MAX = 16 << 20          # packed affines / depthwise taps of one step set: far below one activation buffer
GUARD = -7.0                       # the head ends in ReLU: no depth value is negative

# name -> (net, dtype, tf32x3)
CONFIGS = {
    'skipadd_f16': ('stock', F16, 0),
    'skipadd_bf16': ('stock', BF16, 0),
    'skipadd_f32_highest': ('stock', F32, 0),
    'skipadd_f32_high': ('stock', F32, 1),
    'pruned_f16': ('pruned', F16, 0),
    'skipconcat_f16': ('concat', F16, 0),
    'nnconv5_f16': ('nnconv5', F16, 0),
    'nnconv5_f32_high': ('nnconv5', F32, 1),
    'deconv5_f16': ('deconv5', F16, 0),
    'deconv5_f32_high': ('deconv5', F32, 1),
    'upconv_f16': ('upconv', F16, 0),
    'upconv_f32_high': ('upconv', F32, 1),
}


def _module(net, dtype, hw=(H, W)):
    import models
    if net in ('stock', 'pruned'):
        widths = synthetic.STOCK_WIDTHS if net == 'stock' else synthetic.PRUNED_WIDTHS
        m = models.MobileNetSkipAdd(hw, pretrained=False, widths=widths)
        m.load_state_dict(synthetic.synthetic_state_dict(widths, seed=1))
    elif net == 'concat':
        m = models.MobileNetSkipConcat(hw, pretrained=False)
        m.load_state_dict(synthetic.synthetic_state_dict(seed=1, skip='concat'))
    elif net == 'nnconv5':
        m = models.MobileNet('nnconv5', hw, pretrained=False)
        m.load_state_dict(synthetic.synthetic_nnconv_state_dict(5, seed=1))
    else:
        m = models.MobileNet(net, hw, pretrained=False)
        m.load_state_dict(synthetic.synthetic_convt_state_dict(net, seed=1))
    return m.eval().cuda().to(dtype)


def _plan(descs, weights, names, n, dtype, tf32x3, opts=None):
    p = fplan.Plan(descs, weights, names, n, H, W, dtype, 0)
    if dtype == F32:
        p.set_option('tf32x3', tf32x3)
    for k, v in (opts or {}).items():
        p.set_option(k, v)
    return p


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _guarded(n, dtype):
    """y [n,1,H,W] at the front of a buffer whose next H*W elements are a guard region; both filled with GUARD."""
    buf = torch.full(((n + 1) * H * W,), GUARD, dtype=dtype, device='cuda')
    return buf[:n * H * W].view(n, 1, H, W), buf[n * H * W:]


def _input(x, n):
    """the first n images of x, followed in memory by an image of NaNs"""
    buf = torch.full(((n + 1) * 3 * H * W,), float('nan'), dtype=x.dtype, device='cuda')
    buf[:n * 3 * H * W] = x[:n].reshape(-1)
    return buf[:n * 3 * H * W].view(n, 3, H, W)


def _bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


def _run(p, x, n, dtype):
    y, guard = _guarded(n, dtype)
    p.forward(_input(x, n), y, _stream())
    torch.cuda.synchronize()
    assert bool((guard == GUARD).all()), 'batch %d wrote past its last image' % n
    return y


def _dedicated(descs, weights, names, x, n, dtype, tf32x3, opts=None):
    q = _plan(descs, weights, names, n, dtype, tf32x3, opts)
    y = torch.empty((n, 1, H, W), dtype=dtype, device='cuda')
    q.forward(x[:n].contiguous(), y, _stream())
    torch.cuda.synchronize()
    q.close()
    return y


@pytest.mark.parametrize('cfg', list(CONFIGS))
def test_every_batch_size_from_one_plan(cfg, built_lib):
    net, dtype, tf32x3 = CONFIGS[cfg]
    m = _module(net, dtype)
    descs, weights, names = fplan.describe(m)
    x = synthetic.synthetic_input(CAP, H, W, seed=0).cuda().to(dtype)
    p = _plan(descs, weights, names, CAP, dtype, tf32x3)
    y_cap = torch.empty((CAP, 1, H, W), dtype=dtype, device='cuda')
    p.forward(x, y_cap, _stream())
    torch.cuda.synchronize()
    assert not torch.isnan(y_cap.float()).any()
    ws = p.workspace_bytes()
    order = list(SIZES)
    random.Random(cfg).shuffle(order)
    for n in order:
        y = _run(p, x, n, dtype)
        grown = p.workspace_bytes() - ws
        assert 0 <= grown <= STEP_STATE_MAX and (n < CAP or grown == 0), (n, grown)
        ws += grown
        assert torch.equal(_bits(y), _bits(y_cap[:n])), (cfg, n)
        assert torch.equal(_bits(y), _bits(_dedicated(descs, weights, names, x, n, dtype, tf32x3))), (cfg, n)
    # the step functions still describe the plan's own batch
    assert all(s['macs'] > 0 for s in p.steps())
    p.close()


@pytest.mark.parametrize('cfg', ['skipadd_f16', 'nnconv5_f32_high'])
def test_repeat_replays_and_rebuilds_on_change(cfg, built_lib):
    net, dtype, tf32x3 = CONFIGS[cfg]
    m = _module(net, dtype)
    descs, weights, names = fplan.describe(m)
    x = synthetic.synthetic_input(CAP, H, W, seed=3).cuda().to(dtype)
    p = _plan(descs, weights, names, CAP, dtype, tf32x3)
    p.forward(x, torch.empty((CAP, 1, H, W), dtype=dtype, device='cuda'), _stream())
    xs = {n: _input(x, n) for n in (5, 14)}
    ys = {n: torch.empty((n, 1, H, W), dtype=dtype, device='cuda') for n in (5, 14)}
    ws0 = p.workspace_bytes()
    for n in (5, 14):
        p.forward(xs[n], ys[n], _stream())
    torch.cuda.synchronize()
    first = {n: ys[n].clone() for n in (5, 14)}
    ws = p.workspace_bytes()
    assert ws > ws0
    for _ in range(3):
        for n in (5, 14):
            p.forward(xs[n], ys[n], _stream())
    torch.cuda.synchronize()
    assert p.workspace_bytes() == ws
    assert all(torch.equal(_bits(first[n]), _bits(ys[n])) for n in (5, 14))
    # at most 8 step sets: the plan's own (never evicted) and the 7 most recently used
    grown = {}
    for n in range(1, 13):
        before = p.workspace_bytes()
        y, _ = _guarded(n, dtype)
        p.forward(_input(x, n), y, _stream())
        grown[n] = p.workspace_bytes() - before
    torch.cuda.synchronize()
    assert p.workspace_bytes() - ws0 <= 7 * max(grown[n] for n in range(1, 8)), grown
    # new weights: every step set is rebuilt from them
    w2 = [tuple(None if a is None else (a * 0.75 if i == 3 else a) for i, a in enumerate(wt)) for wt in weights]
    p.set_weights(w2)
    for n in (5, 14):
        p.forward(xs[n], ys[n], _stream())
        torch.cuda.synchronize()
        assert torch.equal(_bits(ys[n]), _bits(_dedicated(descs, w2, names, x, n, dtype, tf32x3))), n
    # a changed option: the same
    p.set_option('fold_head', 0)
    for n in (5, 14):
        p.forward(xs[n], ys[n], _stream())
        torch.cuda.synchronize()
        assert torch.equal(_bits(ys[n]), _bits(_dedicated(descs, w2, names, x, n, dtype, tf32x3, {'fold_head': 0}))), n
    p.close()


def test_out_of_range_batch(built_lib):
    m = _module('stock', F16, (64, 96))
    descs, weights, names = fplan.describe(m)
    p = fplan.Plan(descs, weights, names, 4, 64, 96, F16, 0)
    x = synthetic.synthetic_input(5, 64, 96, seed=0).cuda().half()
    y = torch.empty((5, 1, 64, 96), dtype=F16, device='cuda')
    for n in (0, 5):
        with pytest.raises(RuntimeError, match=r'batch size %d is outside \[1, 4\]' % n):
            p.forward(x[:n], y[:n], _stream(), n=n)
    with pytest.raises(RuntimeError, match='outside'):
        p.forward(x, y, _stream())
    p.forward(x[:3], y[:3], _stream())                    # the plan is still usable
    torch.cuda.synchronize()
    p.close()


def test_engine_keeps_one_plan(built_lib):
    m = _module('stock', F16)
    descs, weights, names = fplan.describe(m)
    eng = SkipAddEngine(m)
    m.__dict__['_fd_engine'] = eng
    x = synthetic.synthetic_input(80, H, W, seed=9).cuda().half()
    with torch.no_grad():
        for n in (64, 14, 64):
            y = m(x[:n])
            torch.cuda.synchronize()
            assert len(eng.plans) == 1 and next(iter(eng.plans.values())).n == 64
            assert torch.equal(_bits(y), _bits(_dedicated(descs, weights, names, x, n, F16, 0))), n
        y = m(x)
        torch.cuda.synchronize()
    assert len(eng.plans) == 1 and next(iter(eng.plans.values())).n == 80
    assert torch.equal(_bits(y), _bits(_dedicated(descs, weights, names, x, 80, F16, 0)))


def test_evaluate_tail_batch_on_full_plan(built_lib):
    """654 images (the NYU val set's count) at batch 64: the tail of 14 runs on the 64-image plan; the 11 sums equal those
    of a dedicated plan per batch size, bit for bit."""
    m = _module('stock', F16)
    descs, weights, names = fplan.describe(m)
    total, bs = 654, 64
    gen = torch.Generator().manual_seed(5)
    batches = []
    for lo in range(0, total, bs):
        n = min(bs, total - lo)
        batches.append((synthetic.synthetic_input(n, H, W, seed=100 + lo), 0.5 + 9.5 * torch.rand(n, 1, H, W, generator=gen)))
    eng = SkipAddEngine(m)
    m.__dict__['_fd_engine'] = eng
    _, sums = evaluate(m, batches, 'cuda', return_sums=True)
    assert len(eng.plans) == 1 and next(iter(eng.plans.values())).n == bs
    want = torch.zeros(fplan.N_METRICS, dtype=torch.float64, device='cuda')
    plans = {}
    for inp, tgt in batches:
        n = inp.shape[0]
        if n not in plans:
            plans[n] = _plan(descs, weights, names, n, F16, 0)
        pred = torch.empty((n, 1, H, W), dtype=F16, device='cuda')
        plans[n].forward(inp.cuda().half(), pred, _stream())
        fplan.metrics_accumulate(pred, tgt.cuda(), want)
    torch.cuda.synchronize()
    assert sums[-1].item() == total
    assert torch.equal(sums, want), (sums, want)
