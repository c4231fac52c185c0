"""The stem, conv1 and conv2 as one kernel (plan option ``front``) on the GPU.

* It computes what the three kernels it replaces compute, bit for bit: the conv0, conv1 and conv2 buffers and the depth
  map of ``front`` 1 equal those of ``front`` 0, in fp16 and bf16, at b64 224x224, b16 480x640, b8 96x128 and b1 32x32,
  for the stock SkipAdd network and the stock encoders of MobileNet('nnconv5') and ('nnconv5dw'), below the capacity
  through ``fd_forward_shape``, with the graph on and off and through three ``ForwardLanes``.
* Nothing past a request's pixels is written: the rest of each of the three buffers keeps its fill.
* The step passes the per-stage fp64 interval reference at ReLU and ReLU6 (tiles at every corner and edge of the map).
* Its name, the stage it is reported under and the launch count are as documented, and other widths keep three steps."""
import pytest
import torch

import test_kernel_sweep as ks
from fastdepth_b200 import plan as fplan
from fastdepth_b200 import synthetic

pytestmark = pytest.mark.gpu

F16, BF16 = torch.float16, torch.bfloat16
R, R6 = ks.R, ks.R6
FRONT = 'stem_tc+front<'


def _module(net, dtype, hw):
    import models
    if net in ('stock', 'pruned'):
        widths = synthetic.STOCK_WIDTHS if net == 'stock' else synthetic.PRUNED_WIDTHS
        m = models.MobileNetSkipAdd(hw, pretrained=False, widths=widths)
        m.load_state_dict(synthetic.synthetic_state_dict(widths, seed=1))
    elif net == 'concat':
        m = models.MobileNetSkipConcat(hw, pretrained=False)
        m.load_state_dict(synthetic.synthetic_state_dict(seed=1, skip='concat'))
    elif net == 'nnconv5':
        m = models.MobileNet(net, hw, pretrained=False)
        m.load_state_dict(synthetic.synthetic_nnconv_state_dict(5, seed=1))
    else:
        m = models.MobileNet(net, hw, pretrained=False)
        m.load_state_dict(synthetic.to_mobilenet_keys(synthetic.synthetic_state_dict(seed=1)))
    return m.eval().cuda().to(dtype)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _forward(p, x):
    y = torch.empty((x.shape[0], 1) + tuple(x.shape[2:]), dtype=x.dtype, device='cuda')
    p.forward(x, y, _stream())
    torch.cuda.synchronize()
    return y


def _front_steps(p):
    return [s for s in p.steps() if s['kernel'].startswith(FRONT)]


def _both(p, x, ns):
    """(depth, buffers of stages 0..2) with front 0 and with front 1"""
    out = []
    for f in (0, 1):
        p.set_option('front', f)
        assert bool(_front_steps(p)) == bool(f)
        y = _forward(p, x)
        out.append((y, [p.stage_tensor(i).clone() for i in range(min(3, ns - 1))]))
    return out


@pytest.mark.parametrize('dtype', [F16, BF16], ids=['f16', 'bf16'])
@pytest.mark.parametrize('shape', [(64, 224, 224), (16, 480, 640), (8, 96, 128), (1, 32, 32)],
                         ids=['b64_224', 'b16_480x640', 'b8_96x128', 'b1_32'])
def test_front_equals_three_steps_bitwise(shape, dtype, built_lib):
    n, h, w = shape
    m = _module('stock', dtype, (h, w))
    descs, weights, names = fplan.describe(m)
    ns = len(descs)
    x = synthetic.synthetic_input(n, h, w, seed=0).cuda().to(dtype)
    p = fplan.Plan(descs, weights, names, n, h, w, dtype, 0)
    (y0, b0), (y1, b1) = _both(p, x, ns)
    assert torch.equal(y1, y0)
    for i in range(3):
        assert torch.equal(b1[i], b0[i]), names[i]
    assert bool((b1[2] > 0).any())
    if n == 8:                                            # graph off
        p.set_option('graph', 0)
        assert torch.equal(_forward(p, x), y0)
    p.close()


@pytest.mark.parametrize('net', ['nnconv5', 'nnconv5dw'])
def test_front_in_the_mobilenet_decoders(net, built_lib):
    dtype, n, h, w = F16, 4, 96, 128
    m = _module(net, dtype, (h, w))
    descs, weights, names = fplan.describe(m)
    x = synthetic.synthetic_input(n, h, w, seed=2).cuda().to(dtype)
    p = fplan.Plan(descs, weights, names, n, h, w, dtype, 0)
    (y0, b0), (y1, b1) = _both(p, x, len(descs))
    assert torch.equal(y1, y0)
    for i in range(3):
        assert torch.equal(b1[i], b0[i]), names[i]
    p.close()


def test_front_below_capacity_and_guard_regions(built_lib):
    """fd_forward_shape on a 16 @ 96x128 plan: smaller n and other (h, w) equal dedicated three-step plans, and the
    three buffers keep their fill past the request's pixels."""
    dtype, N, H, W = F16, 16, 96, 128
    m = _module('stock', dtype, (H, W))
    descs, weights, names = fplan.describe(m)
    p = fplan.Plan(descs, weights, names, N, H, W, dtype, 0)
    assert _front_steps(p)
    for n, h, w in ((5, 96, 128), (16, 64, 64), (3, 32, 96), (1, 128, 96)):
        x = synthetic.synthetic_input(n, h, w, seed=n).cuda().to(dtype)
        q = fplan.Plan(descs, weights, names, n, h, w, dtype, 0)
        q.set_option('front', 0)
        want = _forward(q, x)
        want_b = [q.stage_tensor(i).clone() for i in range(3)]
        q.close()
        fill = []
        for i in range(3):
            t = p.stage_tensor(i)
            t.view(-1).fill_(-3.0)
            fill.append(t.numel())
        y = torch.empty((n, 1, h, w), dtype=dtype, device='cuda')
        p.forward(x, y, _stream())
        torch.cuda.synchronize()
        assert torch.equal(y, want), (n, h, w)
        for i in range(3):
            flat = p.stage_tensor(i).reshape(-1)
            k = want_b[i].numel()
            assert torch.equal(flat[:k], want_b[i].reshape(-1)), (n, h, w, names[i])
            assert bool((flat[k:] == -3.0).all()), (n, h, w, names[i])
    p.close()


def test_front_through_lanes(built_lib):
    from fastdepth_b200.engine import ForwardLanes
    dtype, n, h, w = F16, 8, 96, 128
    m = _module('stock', dtype, (h, w))
    xs = [synthetic.synthetic_input(n, h, w, seed=10 + i).cuda().to(dtype) for i in range(3)]
    want = []
    for x in xs:
        with torch.no_grad():
            want.append(m(x).clone())
    torch.cuda.synchronize()
    ref = []
    descs, weights, names = fplan.describe(m)
    p = fplan.Plan(descs, weights, names, n, h, w, dtype, 0)
    p.set_option('front', 0)
    for x in xs:
        ref.append(_forward(p, x))
    p.close()
    for a, b in zip(want, ref):
        assert torch.equal(a, b)
    lanes = ForwardLanes(m, lanes=3)
    plans = lanes.plans_for(xs[0])
    streams = lanes.streams_for(torch.device('cuda', 0))
    ys = [torch.empty((n, 1, h, w), dtype=dtype, device='cuda') for _ in range(3)]
    for i in range(3):
        assert any(s['kernel'].startswith(FRONT) for s in plans[i].steps())
        plans[i].forward(xs[i], ys[i], streams[i].cuda_stream)
    torch.cuda.synchronize()
    for i in range(3):
        assert torch.equal(ys[i], ref[i]), i


STOCK_ENC_DEC = (32, 64, 128, 128, 256, 32)


@pytest.mark.parametrize('act', [R6, R], ids=['relu6', 'relu'])
def test_front_against_the_interval_reference(act, built_lib, monkeypatch):
    acts = (R6, act, act, R6, R6, R, R, R)
    ks.run_case('front_' + ('relu6' if act == R6 else 'relu'), ks.link([dict(d) for d in ks.enc_dec(STOCK_ENC_DEC, acts=acts)]),
                F16 if act == R6 else BF16, 3, 64, 96, must=(FRONT,), seed=11, monkeypatch=monkeypatch)


def test_front_step_name_stage_and_launches(built_lib):
    dtype, n, h, w = F16, 64, 224, 224
    m = _module('stock', dtype, (h, w))
    descs, weights, names = fplan.describe(m)
    p = fplan.Plan(descs, weights, names, n, h, w, dtype, 0)
    assert p.get_option('front') == 1
    fs = _front_steps(p)
    assert len(fs) == 1 and 'stem_tc' in fs[0]['kernel'] and 'chain_tc' not in fs[0]['kernel'] and '+head' not in fs[0]['kernel']
    assert names[fs[0]['stage']] == 'conv2'
    assert not any(s['stage'] in (0, 1) for s in p.steps())
    assert p.launches_per_forward() == 16
    p.set_option('front', 0)
    assert p.launches_per_forward() == 18 and not _front_steps(p)
    with pytest.raises(Exception):
        p.set_option('front', 2)
    p.close()
    q_m = _module('pruned', dtype, (64, 96))
    d2, w2, n2 = fplan.describe(q_m)
    q = fplan.Plan(d2, w2, n2, 2, 64, 96, dtype, 0)
    assert not _front_steps(q) and any(s['kernel'].startswith('stem_tc<') for s in q.steps())
    q.close()
