"""What a new input resolution costs: a new plan per shape (the engine before one plan served every shape that fits its
pixel capacity) against a new step set on the plan that is already live.

1. First-call latency at a new shape (host clock around the call, ending in a device synchronise):
   - new plan: create a plan for the shape, upload the weights, build its steps, capture its graph and run it;
   - new step set: ``fd_forward_shape`` at that shape on a live plan of 64 @ 224x224 (steps, graph capture, run);
   - steady state: the same call again (graph replay).
2. Peak device memory (``torch.cuda.max_memory_allocated`` does not see the plan's own cudaMalloc; the device's used
   memory from ``cudaMemGetInfo`` does) across a loop of mixed shapes: one plan per shape against one plan of 64 @ 224x224.

    python tools/bench_resolutions.py [--dtype f16|f32] [--out results/resolutions.json]
"""
import argparse
import json
import os
import random
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from fastdepth_b200 import plan as fplan  # noqa: E402
from fastdepth_b200 import synthetic  # noqa: E402

LIVE = (64, 224, 224)
NEW_SHAPES = ((8, 480, 640), (32, 256, 320), (64, 64, 96))


def used_bytes():
    free, total = torch.cuda.mem_get_info()
    return total - free


def sync_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def card():
    q = 'name,power.limit,clocks.max.sm'
    return subprocess.run(['nvidia-smi', '--query-gpu=' + q, '--format=csv,noheader'], capture_output=True,
                          text=True).stdout.strip()


def label(s):
    return '%d @ %dx%d' % s


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--dtype', default='f16', choices=('f16', 'f32'))
    ap.add_argument('--loop', type=int, default=40)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'needs a GPU'
    import models
    dtype = torch.float16 if a.dtype == 'f16' else torch.float32
    m = models.MobileNetSkipAdd(LIVE[1:], pretrained=False)
    m.load_state_dict(synthetic.synthetic_state_dict(seed=1))
    m = m.eval()
    descs, weights, names = fplan.describe(m)
    tf32x3 = int(dtype == torch.float32)
    shapes = NEW_SHAPES + (LIVE,)
    xs = {s: synthetic.synthetic_input(*s, seed=i).cuda().to(dtype) for i, s in enumerate(shapes)}
    ys = {s: torch.empty((s[0], 1) + s[1:], dtype=dtype, device='cuda') for s in shapes}
    st = torch.cuda.current_stream().cuda_stream

    def new_plan(s):
        p = fplan.Plan(descs, weights, names, *s, dtype, 0)
        if dtype == torch.float32:
            p.set_option('tf32x3', tf32x3)
        return p

    # warm the module loads and the first-launch costs of every kernel with one plan per shape
    for s in shapes:
        warm = new_plan(s)
        warm.forward(xs[s], ys[s], st)
        torch.cuda.synchronize()
        warm.close()

    lat = []
    for s in NEW_SHAPES:
        holder = {}
        t_plan = sync_ms(lambda: holder.setdefault('p', new_plan(s)).forward(xs[s], ys[s], st))
        holder['p'].close()
        live = new_plan(LIVE)
        live.forward(xs[LIVE], ys[LIVE], st)
        t_set = sync_ms(lambda: live.forward(xs[s], ys[s], st))
        t_again = min(sync_ms(lambda: live.forward(xs[s], ys[s], st)) for _ in range(5))
        live.close()
        lat.append(dict(shape=list(s), new_plan_ms=round(t_plan, 2), new_step_set_ms=round(t_set, 2),
                        replay_ms=round(t_again, 3)))
        print('%-16s new plan %8.2f ms   new step set %7.2f ms   replay %6.3f ms' % (label(s), t_plan, t_set, t_again))

    rng = random.Random(0)
    loop = [rng.choice(shapes) for _ in range(a.loop)]
    torch.cuda.synchronize()
    base = used_bytes()
    plans, peak_per_shape = {}, 0
    for s in loop:                                  # one plan per shape, kept (the engine's old policy)
        if s not in plans:
            plans[s] = new_plan(s)
        plans[s].forward(xs[s], ys[s], st)
        torch.cuda.synchronize()
        peak_per_shape = max(peak_per_shape, used_bytes() - base)
    for p in plans.values():
        p.close()
    torch.cuda.synchronize()
    base = used_bytes()
    one, peak_one = new_plan(LIVE), 0
    for s in loop:
        one.forward(xs[s], ys[s], st)
        torch.cuda.synchronize()
        peak_one = max(peak_one, used_bytes() - base)
    one.close()
    print('mixed loop of %d calls over %s: peak device memory  one plan per shape %.0f MB   one plan of %s %.0f MB'
          % (a.loop, ', '.join(label(s) for s in sorted(set(loop))), peak_per_shape / 2**20, label(LIVE),
             peak_one / 2**20))

    gpu = card()
    print('card (name, power limit, max SM clock): %s' % gpu)
    res = dict(gpu=gpu, dtype=a.dtype, live=list(LIVE), first_call=lat, loop_shapes=[list(s) for s in loop],
               peak_mb_plan_per_shape=round(peak_per_shape / 2**20), peak_mb_one_plan=round(peak_one / 2**20))
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
