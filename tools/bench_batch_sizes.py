"""What a new batch size costs: a new plan per size (the engine before one plan served every size up to its capacity)
against a new step set on the plan that is already live.

1. First-call latency at a new batch size n (host clock around the call, ending in a device synchronise):
   - new plan: create a plan for n, upload the weights, build its steps, capture its graph and run it;
   - new step set: ``fd_forward_batch`` at n on a live plan of capacity 64 (steps for n, graph capture, run);
   - steady state: the same call again (graph replay).
2. Peak device memory (``torch.cuda.max_memory_allocated`` does not see the plan's own cudaMalloc; the device's used
   memory from ``cudaMemGetInfo`` does) across a loop of mixed batch sizes: one plan per size against one plan of 64.

    python tools/bench_batch_sizes.py [--dtype f16|f32] [--out results/batch_sizes.json]
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

H = W = 224
CAP = 64
NEW_SIZES = (1, 5, 14, 32, 63)


def used_bytes():
    free, total = torch.cuda.mem_get_info()
    return total - free


def sync_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--dtype', default='f16', choices=('f16', 'f32'))
    ap.add_argument('--loop', type=int, default=40)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'needs a GPU'
    import models
    dtype = torch.float16 if a.dtype == 'f16' else torch.float32
    m = models.MobileNetSkipAdd((H, W), pretrained=False)
    m.load_state_dict(synthetic.synthetic_state_dict(seed=1))
    m = m.eval()
    descs, weights, names = fplan.describe(m)
    tf32x3 = int(dtype == torch.float32)
    x = synthetic.synthetic_input(CAP, H, W, seed=0).cuda().to(dtype)
    ys = {n: torch.empty((n, 1, H, W), dtype=dtype, device='cuda') for n in NEW_SIZES + (CAP,)}
    xs = {n: x[:n].contiguous() for n in NEW_SIZES + (CAP,)}
    st = torch.cuda.current_stream().cuda_stream

    def new_plan(n):
        p = fplan.Plan(descs, weights, names, n, H, W, dtype, 0)
        if dtype == torch.float32:
            p.set_option('tf32x3', tf32x3)
        return p

    # warm the module loads and the first-launch costs of every kernel with one full plan
    warm = new_plan(CAP)
    warm.forward(xs[CAP], ys[CAP], st)
    torch.cuda.synchronize()
    warm.close()

    lat = []
    for n in NEW_SIZES:
        holder = {}
        t_plan = sync_ms(lambda: holder.setdefault('p', new_plan(n)).forward(xs[n], ys[n], st))
        holder['p'].close()
        live = new_plan(CAP)
        live.forward(xs[CAP], ys[CAP], st)
        t_set = sync_ms(lambda: live.forward(xs[n], ys[n], st))
        t_again = min(sync_ms(lambda: live.forward(xs[n], ys[n], st)) for _ in range(5))
        live.close()
        lat.append(dict(n=n, new_plan_ms=round(t_plan, 2), new_step_set_ms=round(t_set, 2), replay_ms=round(t_again, 3)))
        print('n=%2d  new plan %8.2f ms   new step set %7.2f ms   replay %6.3f ms' % (n, t_plan, t_set, t_again))

    rng = random.Random(0)
    sizes = [rng.choice(NEW_SIZES + (CAP,)) for _ in range(a.loop)]
    torch.cuda.synchronize()
    base = used_bytes()
    plans, peak_per_size = {}, 0
    for n in sizes:                                 # one plan per size, kept (the engine's old policy)
        if n not in plans:
            plans[n] = new_plan(n)
        plans[n].forward(xs[n], ys[n], st)
        torch.cuda.synchronize()
        peak_per_size = max(peak_per_size, used_bytes() - base)
    for p in plans.values():
        p.close()
    torch.cuda.synchronize()
    base = used_bytes()
    one, peak_one = new_plan(CAP), 0
    for n in sizes:
        one.forward(xs[n], ys[n], st)
        torch.cuda.synchronize()
        peak_one = max(peak_one, used_bytes() - base)
    one.close()
    print('mixed loop of %d calls over sizes %s: peak device memory  one plan per size %.0f MB   one plan of %d %.0f MB'
          % (a.loop, sorted(set(sizes)), peak_per_size / 2**20, CAP, peak_one / 2**20))

    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                         text=True).stdout.strip()
    res = dict(gpu=gpu, dtype=a.dtype, hw=[H, W], capacity=CAP, first_call=lat, loop_sizes=sizes,
               peak_mb_plan_per_size=round(peak_per_size / 2**20), peak_mb_one_plan=round(peak_one / 2**20))
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
