"""The plans the benchmarks time, checked stage by stage against the per-stage fp64 interval reference on EVERY image of
the batch (tests/plan_check.py, the kernel sweep's checker).

At the benchmarked shapes the planners choose block ring depths, output-channel splits, cluster and multiwave modes, conv
tiles, bn and n-splits with dozens of items per persistent CTA that the synthetic geometries of test_kernel_sweep.py,
test_conv_gpu.py and test_convt_gpu.py never build.  A fault confined to some work items (one n-split, the later items
of a persistent CTA, a ring slot reused only after many items) on an image outside a pick passes an end-to-end
comparison of picked images, and the decoder can dilute it below the end-to-end tolerance; here every 16-bit element of
every stage of every image is held to the strict rule.

Each configuration is built the way its benchmark builds it: the module class and widths, the synthetic recipe with
seed 1, ``.to(dtype)``, the benchmark's options and ``synthetic.synthetic_input``.  The plan is the module's own
``SkipAddEngine``'s, so the checked plan is the timed plan, and ``plan.describe`` gives the reference exactly the
weights the kernels hold (16-bit parameters, fp32 BN affines)."""
import time

import pytest
import torch

import dense_ref as dr
import plan_check as pc
from fastdepth_b200 import plan as fplan
from fastdepth_b200 import synthetic
from fastdepth_b200.engine import ForwardLanes, SkipAddEngine

pytestmark = pytest.mark.gpu

F16, BF16 = torch.float16, torch.bfloat16
OPTIONS = {'path': 1, 'fold_head': 1, 'graph': 1}        # bench.py's defaults (chain, inplace_skip, TMA epilogue: plan defaults)
SKIPADD = ('stem_tc', 'chain_tc<', '[5 layers', '+head', '+skip(red)')
# fp16 on the benchmark weights: every element lies inside its interval and every determined one is the round-to-nearest
# value, but fewer than half are determined in the deep and decoder stages.  Measured on an H100 80GB HBM3 (700 W):
# SkipAdd conv7..conv13 0.41-0.49, decode_conv1..4 0.33-0.44 (A, C, D, E); NNConv5 decoder.conv1..3 0.36-0.45.  The bench
# recipe calibrates BN on the pre-activations, so its scales are large where a channel's sum varies little against the
# sum of its |terms|; the interval's radius (2^-18 times that sum, times the scale) then spans a rounding midpoint of
# an fp16 output for about half of them.  bf16, with an 8x coarser ulp, stays at 0.69 and above on the same stages.
FP16_BENCH_FLOOR = 0.3

CONFIGS = {
    'A_stock_b64_224_f16': dict(net='stock', n=64, h=224, w=224, dtype=F16, must=SKIPADD, lanes=True),   # bench.py default
    'B_stock_b64_224_bf16': dict(net='stock', n=64, h=224, w=224, dtype=BF16, must=SKIPADD),   # its bf16 evaluation leg
    'C_pruned_b64_224_f16': dict(net='pruned', n=64, h=224, w=224, dtype=F16, must=('stem_tc', '+head', '+skip(red)')),
    'D_stock_b32_224_f16': dict(net='stock', n=32, h=224, w=224, dtype=F16, must=SKIPADD),
    'E_stock_b16_480x640_f16': dict(net='stock', n=16, h=480, w=640, dtype=F16,     # 15x20 maps: conv7..11 run one by one
                                    must=('stem_tc', '+head', '+skip(red)', 'block_tc<k3,s1,1x8x16>+tmast[n128x4')),
    'F_nnconv5_b64_224_f16': dict(net='nnconv5', n=64, h=224, w=224, dtype=F16, must=('conv_tc_kernel<k5',)),
    'F_nnconv5_b64_224_bf16': dict(net='nnconv5', n=64, h=224, w=224, dtype=BF16, must=('conv_tc_kernel<k5',)),
}


def _build(c):
    import models
    n, h, w, dtype = c['n'], c['h'], c['w'], c['dtype']
    if c['net'] == 'nnconv5':
        m = models.MobileNet('nnconv5', (h, w), pretrained=False)
        m.load_state_dict(synthetic.synthetic_nnconv_state_dict(5, seed=1))
    else:
        widths = synthetic.STOCK_WIDTHS if c['net'] == 'stock' else synthetic.PRUNED_WIDTHS
        m = models.MobileNetSkipAdd((h, w), pretrained=False, widths=widths)
        m.load_state_dict(synthetic.synthetic_state_dict(widths, seed=1))
    m = m.eval().cuda().to(dtype)
    eng = SkipAddEngine(m)
    for k, v in OPTIONS.items():
        eng.set_option(k, v)
    m.__dict__['_fd_engine'] = eng
    x = synthetic.synthetic_input(n, h, w, seed=0).cuda().to(dtype)
    return m, eng.plan_for(x), x


@pytest.mark.parametrize('cfg', list(CONFIGS))
def test_production_plan_every_image(cfg, built_lib):
    c = CONFIGS[cfg]
    n, h, w, dtype = c['n'], c['h'], c['w'], c['dtype']
    t0 = time.perf_counter()
    m, plan, x = _build(c)
    descs, weights, _ = fplan.describe(m)
    ns = len(descs)
    dense = c['net'] == 'nnconv5'
    # NNConv5: the five CONV stages and the head (its encoder is the stock encoder, checked in A-E)
    only = {i for i, d in enumerate(descs) if d['kind'] == dr.CONV} | {ns - 1} if dense else None
    y = torch.empty((n, 1, h, w), dtype=dtype, device='cuda')
    chk = pc.Checker(cfg, dtype, FP16_BENCH_FLOOR if dtype == F16 else pc.MIN_DETERMINED)
    chunk = max(2, pc.CHUNK * 224 * 224 // (h * w))
    ran = pc.check_plan(plan, descs, weights, dtype, x.float().cpu().numpy(), x, y, range(n), chk, OPTIONS,
                        stream=torch.cuda.current_stream().cuda_stream, chunk=chunk, only=only, rerun_all=False)
    secs = time.perf_counter() - t0
    kern = {}
    for s in ran[0]:
        kern.setdefault(s['stage'], s['kernel'])
    print('\n%s: %d images, checked in %.1f s' % (cfg, n, secs))
    for what, f, strict in chk.results:
        st = int(what.split()[1].split('-')[0]) if what.split()[0] in ('stage', 'chain', 'block') else \
            {'stem': 0}.get(what, ns - 1)
        print('  %-15s %-9s determined %.4f  %s' % (what, 'strict' if strict else 'contained', f, kern.get(st, '')))
    # every stage in scope was held to the strict rule on its own
    strict = {what for what, _, s in chk.results if s}
    want = {'stage %d' % i for i in (only - {ns - 1} if dense else range(1, ns - 1))} | {'head'}
    want |= set() if dense else {'stem'}
    assert want <= strict, sorted(want - strict)
    kernels = ' '.join(s['kernel'] for steps in ran for s in steps)
    for k in c['must']:
        assert k in kernels, (cfg, k, kernels)
    if dense:
        assert sum(s['kernel'].startswith('conv_tc_kernel<k5') for s in ran[0]) == 5, kernels
    if c.get('lanes'):
        _lanes_match_plan(m, plan, c)


def _lanes_match_plan(m, plan, c):
    """bench.py's `value` comes from engine.ForwardLanes: three plan copies on three streams.  Their depth maps for
    batches in flight must equal the checked plan's, bit for bit, on the same inputs (bench.py's rotating batches)."""
    n, h, w, dtype = c['n'], c['h'], c['w'], c['dtype']
    xs = [synthetic.synthetic_input(n, h, w, seed=i).cuda().to(dtype) for i in range(4)]
    ref = []
    for x in xs:
        ref.append(torch.empty((n, 1, h, w), dtype=dtype, device='cuda'))
        plan.forward(x, ref[-1], torch.cuda.current_stream().cuda_stream)
    lanes = ForwardLanes(m, lanes=3, options=OPTIONS)
    outs = [lanes.forward(xs[i % 4])[0] for i in range(8)]
    lanes.synchronize()
    torch.cuda.synchronize()
    for i, yl in enumerate(outs):
        assert torch.equal(yl, ref[i % 4]), i
