"""A/B planner experiment knobs (environment variables read when a plan is built) on the bench workload.
usage: python tools/ab_env.py "FD_TC_MAX_NCTA=64,FD_TC_CLUSTER=1" "FD_TC_MAX_NCTA=64" "" """
import sys, os
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import models
from fastdepth_b200 import synthetic
from fastdepth_b200.engine import SkipAddEngine

sd = synthetic.synthetic_state_dict()
m = models.MobileNetSkipAdd((224, 224), pretrained=False); m.load_state_dict(sd); m = m.eval().cuda().half()
x = synthetic.synthetic_input(64, 224, 224).cuda().half()
y = torch.empty((64, 1, 224, 224), dtype=torch.half, device='cuda')
sp = torch.cuda.current_stream().cuda_stream
ref = None
for cfg in sys.argv[1:]:
    for k in ('FD_TC_MAX_NCTA', 'FD_TC_CLUSTER'):
        os.environ.pop(k, None)
    for kv in filter(None, cfg.split(',')):
        k, v = kv.split('='); os.environ[k] = v
    eng = SkipAddEngine(m)
    plan = eng.plan_for(x)
    for _ in range(5): plan.forward(x, y, sp)
    torch.cuda.synchronize()
    if ref is None: ref = y.clone()
    err = (y.float() - ref.float()).abs().max().item()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(50): plan.forward(x, y, sp)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 50
    print(f'[{cfg or "default"}] forward {ms*1e3:.1f} us  ({64/ms*1e3:.0f} img/s)  max|y - y_first_cfg| = {err:.3g}')
    t = plan.time_steps(x, y, sp, warmup=2, iters=5, flush_l2=True)
    print('   ', ' '.join(f"{s['stage_name'].replace('decode_conv','d').replace('conv','c')}:{s['ms']*1e3:.0f}" for s in t))
    print('   ', ' '.join(s['kernel'].split('[')[1].rstrip(']') for s in t if '[' in s['kernel']))
