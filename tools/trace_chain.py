"""Timeline of the chain kernel (CTA 0 of cluster 0, first image): per-layer SM-clock stamps of the roles."""
import os, sys
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import models
from fastdepth_b200 import synthetic
from fastdepth_b200.engine import SkipAddEngine
widths = synthetic.PRUNED_WIDTHS if (len(sys.argv) > 1 and sys.argv[1] == 'pruned') else synthetic.STOCK_WIDTHS
sd = synthetic.synthetic_state_dict(widths)
m = models.MobileNetSkipAdd((224, 224), pretrained=False, widths=widths); m.load_state_dict(sd); m = m.eval().cuda().half()
eng = SkipAddEngine(m); eng.set_option('graph', 0); m.__dict__['_fd_engine'] = eng
x = synthetic.synthetic_input(64, 224, 224).cuda().half()
plan = eng.plan_for(x)
y = torch.empty((64, 1, 224, 224), dtype=torch.half, device='cuda')
sp = torch.cuda.current_stream().cuda_stream
plan.forward(x, y, sp); torch.cuda.synchronize()
st = [s for s in plan.steps() if 'chain_tc' in s['kernel']][0]
first = int(st['kernel'].split('{stages ')[1].split('-')[0])
for rep in range(2):
    tr = plan.trace_stage(first, y, sp)
t0 = min(v.min() for v in tr.values() if len(v))
print(st['kernel'])
for k, v in tr.items():
    print('%-22s %s' % (k, ' '.join('%7d' % (a - t0) for a in v)))
ls, le = tr['layer_start'] - t0, tr['halo_received'] - t0
print('per layer (cycles):', ' '.join('%d' % (b - a) for a, b in zip(ls, le)))
for a, b, n in (('layer_start', 'dw_done_grp0', 'dw phase grp0'), ('dw_done_grp0', 'pointwise_done', 'pointwise passes'),
                ('pointwise_done', 'epilogue_done', 'epilogue'), ('epilogue_done', 'local_barrier', 'zero list + local barrier'),
                ('local_barrier', 'halo_received', 'halo wait')):
    n_ = min(len(tr[a]), len(tr[b]))
    print('%-28s %s' % (n, ' '.join('%6d' % d for d in (tr[b][:n_] - tr[a][:n_]))))
