"""A/B of the plan option ``front`` on the bench workload (stock MobileNet-NNConv5(dw)+skipadd, b64, 224x224): the stem,
conv1 and conv2 as one front_tc_kernel step (1) against the three kernels (0).  The variants alternate in one process,
``--repeats`` times each.

Printed: the card, its power limit and max SM clock; the launch counts; per stage the min-max of ``plan.time_steps``
without and with the L2 flush before every launch (the front step is reported under conv2, so the conv0..conv2 row is
the one to compare); the whole forward as graph replay on one stream and through three ``ForwardLanes``; the depth maps'
equality with ``front`` 0.
usage: python tools/bench_front.py [--dtype f16|bf16] [--repeats 3] [--forwards 200]"""
import argparse
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import models  # noqa: E402
from fastdepth_b200 import synthetic  # noqa: E402
from fastdepth_b200.engine import ForwardLanes, SkipAddEngine  # noqa: E402

STAGES = ('conv0', 'conv1', 'conv2', 'conv3', 'conv6', 'decode_conv4', 'decode_conv5')
N, H, W = 64, 224, 224


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def timed(fn, forwards, join=None):
    """us per forward between two CUDA events on the current stream; ``join`` makes it wait for the lanes' streams first."""
    for _ in range(20):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(forwards):
        fn()
    if join is not None:
        join()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / forwards * 1e3          # us per forward


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--dtype', default='f16', choices=('f16', 'bf16'))
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--forwards', type=int, default=200)
    a = ap.parse_args()
    dtype = torch.float16 if a.dtype == 'f16' else torch.bfloat16
    print('card: %s   dtype %s   b%d %dx%d' % (card(), a.dtype, N, H, W))
    m = models.MobileNetSkipAdd((H, W), pretrained=False)
    m.load_state_dict(synthetic.synthetic_state_dict(seed=1))
    m = m.eval().cuda().to(dtype)
    xs = [synthetic.synthetic_input(N, H, W, seed=i).cuda().to(dtype) for i in range(4)]
    ys = [torch.empty((N, 1, H, W), dtype=dtype, device='cuda') for _ in range(4)]
    sp = torch.cuda.current_stream().cuda_stream
    variants = (0, 1)
    engines = {}
    for v in variants:
        engines[v] = SkipAddEngine(m)
        engines[v].set_option('front', v)
    lanes = {v: ForwardLanes(m, lanes=3, options={'front': v}) for v in variants}
    res = {v: dict(flush={s: [] for s in STAGES}, warm={s: [] for s in STAGES}, graph=[], lanes=[]) for v in variants}
    ref = None
    for rep in range(a.repeats):
        for v in variants:
            plan = engines[v].plan_for(xs[0])
            if rep == 0:
                print('front=%d: %d launches' % (v, plan.launches_per_forward()))
                for s in plan.steps():
                    if s['stage_name'] in STAGES:
                        print('    %-13s %s' % (s['stage_name'], s['kernel']))
                plan.forward(xs[0], ys[0], sp)
                torch.cuda.synchronize()
                if ref is None:
                    ref = ys[0].clone()
                print('    depth map equals front=0: %s' % torch.equal(ys[0], ref))
            for key, flush in (('flush', True), ('warm', False)):
                per = {}
                for s in plan.time_steps(xs[0], ys[0], sp, warmup=3, iters=20, flush_l2=flush):
                    per[s['stage_name']] = per.get(s['stage_name'], 0.0) + s['ms'] * 1e3
                for s in STAGES:
                    res[v][key][s].append(per.get(s, float('nan')))
            k = [0]

            def one():
                plan.forward(xs[k[0] & 3], ys[k[0] & 3], sp)
                k[0] += 1

            def three():
                lanes[v].forward(xs[k[0] & 3], ys[k[0] & 3])
                k[0] += 1

            def join():
                for st in lanes[v].streams_for(xs[0].device):
                    torch.cuda.current_stream().wait_stream(st)
            res[v]['graph'].append(timed(one, a.forwards))
            res[v]['lanes'].append(timed(three, a.forwards, join))
            lanes[v].synchronize()

    def rng(t):
        return '%6.1f-%-6.1f' % (min(t), max(t))
    for key, title in (('warm', 'step time per stage, us, NO L2 flush (min-max over %d repeats)' % a.repeats),
                       ('flush', 'step time per stage, us, L2 flushed before every launch')):
        print('\n' + title)
        print('%-14s' % 'stage' + ''.join('  front=%d       ' % v for v in variants))
        for s in STAGES:
            print('%-14s' % s + ''.join('  ' + rng(res[v][key][s]) + ' ' for v in variants))
        tail = ('conv0', 'conv1', 'conv2')
        print('%-14s' % 'conv0..conv2' + ''.join(
            '  ' + rng([sum(res[v][key][s][r] for s in tail) for r in range(a.repeats)]) + ' ' for v in variants))
    print('\nwhole forward, us per batch of %d (%d forwards per window, rotating inputs)' % (N, a.forwards))
    for v in variants:
        g, ln = res[v]['graph'], res[v]['lanes']
        print('front=%d  graph replay, one stream %s (%.0f img/s best)   three lanes %s (%.0f img/s best)' %
              (v, rng(g), N / min(g) * 1e6, rng(ln), N / min(ln) * 1e6))


if __name__ == '__main__':
    main()
