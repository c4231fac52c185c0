"""The two-step route of a 16-bit DWPW stage (plan option ``unfuse``) on the GPU: dw_mid_kernel writes the depthwise half
to the stage's intermediate, conv_tc_kernel runs the pointwise half over it as a 1x1 conv.

* It computes what the fused block kernel computes, bit for bit: every stage buffer and the depth map of ``unfuse`` 1
  and 2 equal those of ``unfuse`` 0, for the stock and pruned SkipAdd, SkipConcat and nnconv5dw networks in fp16 and
  bf16, with and without the chain kernel, the in-place skip add and the folded head.
* The 1x1 steps are held to the per-stage fp64 interval reference by the kernel sweep's checker, over channel tails,
  pinned bn and tiles, both strides and kernel sizes, upsample, the reduce-add skip, both activations and 1x1 / 1x2 maps.
* At b64 224x224 the stock network's default plan takes the route for conv12, conv13 and decode_conv1 and nothing else;
  ``fd_forward_batch`` below the capacity equals dedicated plans."""
import itertools

import pytest
import torch

import test_kernel_sweep as ks
from fastdepth_b200 import plan as fplan
from fastdepth_b200 import synthetic

pytestmark = pytest.mark.gpu

F16, BF16 = torch.float16, torch.bfloat16
R, R6 = ks.R, ks.R6


def _module(net, dtype, hw):
    import models
    if net in ('stock', 'pruned'):
        widths = synthetic.STOCK_WIDTHS if net == 'stock' else synthetic.PRUNED_WIDTHS
        m = models.MobileNetSkipAdd(hw, pretrained=False, widths=widths)
        m.load_state_dict(synthetic.synthetic_state_dict(widths, seed=1))
    elif net == 'concat':
        m = models.MobileNetSkipConcat(hw, pretrained=False)
        m.load_state_dict(synthetic.synthetic_state_dict(seed=1, skip='concat'))
    else:
        m = models.MobileNet('nnconv5dw', hw, pretrained=False)
        m.load_state_dict(synthetic.to_mobilenet_keys(synthetic.synthetic_state_dict(seed=1)))
    return m.eval().cuda().to(dtype)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _forward(p, x):
    y = torch.empty((x.shape[0], 1) + tuple(x.shape[2:]), dtype=x.dtype, device='cuda')
    p.forward(x, y, _stream())
    torch.cuda.synchronize()
    return y


def _two_step_stages(p):
    return sorted({s['stage'] for s in p.steps() if s['kernel'].startswith('dw_mid_kernel')})


@pytest.mark.parametrize('dtype', [F16, BF16], ids=['f16', 'bf16'])
@pytest.mark.parametrize('net', ['stock', 'pruned', 'concat', 'nnconv5dw'])
def test_two_steps_equal_the_fused_kernel_bitwise(net, dtype, built_lib):
    n, h, w = 8, 96, 128                       # 3x4 bottom maps: 96 rows, planned as a 6 x 16 matrix image
    m = _module(net, dtype, (h, w))
    descs, weights, names = fplan.describe(m)
    ns = len(descs)
    x = synthetic.synthetic_input(n, h, w, seed=0).cuda().to(dtype)
    p = fplan.Plan(descs, weights, names, n, h, w, dtype, 0)
    taken = set()
    for chain, inplace, fold in itertools.product((0, 1), (0, 1), (0, 1)):
        for k, v in (('chain', chain), ('inplace_skip', inplace), ('fold_head', fold)):
            p.set_option(k, v)
        p.set_option('unfuse', 0)
        assert _two_step_stages(p) == []
        y0 = _forward(p, x)
        bufs0 = [p.stage_tensor(i).clone() for i in range(ns - 1)]
        n0 = p.launches_per_forward()
        for u in (1, 2):
            p.set_option('unfuse', u)
            two = _two_step_stages(p)
            assert p.launches_per_forward() == n0 + len(two)
            yu = _forward(p, x)
            assert torch.equal(yu, y0), (chain, inplace, fold, u)
            for i in range(ns - 1):
                assert torch.equal(p.stage_tensor(i), bufs0[i]), (chain, inplace, fold, u, names[i])
            for i in two:              # the intermediate is there to look at: the depthwise half of this stage, after its act
                mid = p.stage_tensor(i, which=1)
                assert mid.shape[-1] == descs[i]['c_in'] and bool((mid >= 0).all()) and bool((mid > 0).any()), names[i]
            if u == 2:
                assert len(two) >= 5 and set(two) >= taken, (two, taken)
                if inplace:
                    kern = ' '.join(s['kernel'] for s in p.steps())
                    assert (',+skip(red)]' in kern) == (net in ('stock', 'pruned')), kern
            else:
                taken = set(two)
                assert two, 'the 3x4 stages of 1024 channels are split 8 ways or more'
    p.close()


# stage sweep: the 1x1 steps against the fp64 interval reference (plan_check), forced with unfuse = 2
TWO = ('dw_mid_kernel<3>', 'dw_mid_kernel<5>', 'conv_tc_kernel<k1,')
SWEEP = {
    # c_in mod 64 in {8, 24, 40} (72, 24 / 88, 40 / 104), c_out tails 8, 40, 72, 136, 264; skips added by reduce-add
    'tails_f16': dict(descs=lambda: ks.enc_dec((24, 72, 88, 136, 264, 8)), dtype=F16, n=3, h=64, w=96,
                      must=TWO + (',+skip(red)]', ',up>', ',noup>')),
    'tails_bf16': dict(descs=lambda: ks.enc_dec((40, 104, 72, 264, 136, 40), acts=(R6, R, R6, R, R6, R6, R, R6)), dtype=BF16,
                       n=2, h=64, w=64, must=TWO + (',+skip(red)]', 'relu6')),
    'bn64': dict(descs=lambda: ks.enc_dec((24, 72, 88, 136, 264, 8)), dtype=F16, n=3, h=64, w=96, env={'FD_CONV_BN': '64'},
                 must=TWO + ('conv_tc_kernel<k1,bn64,',)),
    'bn128': dict(descs=lambda: ks.enc_dec((24, 72, 88, 136, 264, 8)), dtype=BF16, n=3, h=64, w=96, env={'FD_CONV_BN': '128'},
                  must=TWO + ('conv_tc_kernel<k1,bn128,',)),
    'bn256_tile1': dict(descs=lambda: ks.enc_dec((24, 72, 88, 136, 264, 8)), dtype=F16, n=4, h=64, w=64,
                        env={'FD_CONV_BN': '256', 'FD_CONV_TILE': '1'}, must=TWO + ('conv_tc_kernel<k1,bn256,', '[2x8x8,')),
    'tile3': dict(descs=lambda: ks.enc_dec((24, 72, 88, 136, 264, 8)), dtype=F16, n=5, h=64, w=64, env={'FD_CONV_TILE': '3'},
                  must=TWO + ('[8x4x4,',)),
    'bottom_1x1': dict(descs=lambda: ks.deep(3), dtype=F16, n=5, h=32, w=32, must=TWO),
    'bottom_1x2': dict(descs=lambda: ks.deep(5), dtype=BF16, n=16, h=32, w=64, must=TWO),
    'concat': dict(descs=ks.concat_net, dtype=F16, n=2, h=64, w=64, must=TWO),
}


@pytest.mark.parametrize('case', list(SWEEP))
def test_pointwise_steps_against_the_interval_reference(case, built_lib, monkeypatch):
    c = SWEEP[case]
    ks.run_case('unfuse_' + case, c['descs'](), c['dtype'], c['n'], c['h'], c['w'], must=c['must'],
                opts={'unfuse': 2, 'chain': 0}, env=c.get('env'), seed=7, monkeypatch=monkeypatch)


def test_a_batch_equals_its_images_alone_and_graph_off(built_lib):
    dtype, h, w = F16, 64, 96
    m = _module('stock', dtype, (h, w))
    descs, weights, names = fplan.describe(m)
    x = synthetic.synthetic_input(16, h, w, seed=3).cuda().to(dtype)
    p = fplan.Plan(descs, weights, names, 16, h, w, dtype, 0)
    p.set_option('unfuse', 2)
    y = _forward(p, x)
    p.set_option('graph', 0)
    assert torch.equal(_forward(p, x), y)
    one = fplan.Plan(descs, weights, names, 1, h, w, dtype, 0)
    one.set_option('unfuse', 2)
    for i in (0, 7, 15):
        assert torch.equal(_forward(one, x[i:i + 1].contiguous()), y[i:i + 1]), i
    one.close()
    p.close()


def test_stock_b64_takes_the_route_for_the_three_wide_7x7_stages(built_lib):
    dtype, n, h, w = F16, 64, 224, 224
    m = _module('stock', dtype, (h, w))
    descs, weights, names = fplan.describe(m)
    x = synthetic.synthetic_input(n, h, w, seed=0).cuda().to(dtype)
    p = fplan.Plan(descs, weights, names, n, h, w, dtype, 0)
    assert p.get_option('unfuse') == 1
    steps = p.steps()
    two = _two_step_stages(p)
    assert [names[i] for i in two] == ['conv12', 'conv13', 'decode_conv1'], [names[i] for i in two]
    for i in two:
        kinds = [s['kernel'].split('<')[0] for s in steps if s['stage'] == i]
        assert kinds == ['dw_mid_kernel', 'pw:conv_tc_kernel'], kinds
    assert not any(',cl' in s['kernel'] for s in steps)
    n1 = p.launches_per_forward()
    y1 = _forward(p, x)
    ws = p.workspace_bytes()
    # smaller batches on the same plan: per-n tensor maps over the same intermediate
    for k in (1, 14, 63):
        q = fplan.Plan(descs, weights, names, k, h, w, dtype, 0)
        want = _forward(q, x[:k].contiguous())
        q.close()
        yk = torch.empty((k, 1, h, w), dtype=dtype, device='cuda')
        p.forward(x[:k].contiguous(), yk, _stream(), n=k)
        torch.cuda.synchronize()
        assert torch.equal(yk, want), k
        assert torch.equal(yk, y1[:k]), k
    assert ws < p.workspace_bytes() < ws + (16 << 20)
    p.set_option('unfuse', 0)
    assert _two_step_stages(p) == [] and p.launches_per_forward() == n1 - 3
    assert torch.equal(_forward(p, x), y1)
    with pytest.raises(Exception):
        p.set_option('unfuse', 3)
    p.close()
