"""Small-shape workload for compute-sanitizer (memcheck / racecheck / synccheck / initcheck) over every kernel organisation
of the fused path: stock and pruned widths, fp16 and bf16, TMA and LSU epilogues, in-place skip accumulation on and off, head
folded and not, the planner's output-channel splits (environment knobs), graph replay and direct launches.
usage (on a machine with an H100 and compute-sanitizer): compute-sanitizer --tool memcheck python tools/sanitize_run.py [quick]"""
import itertools
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import models  # noqa: E402
from fastdepth_b200 import synthetic  # noqa: E402
from fastdepth_b200.engine import SkipAddEngine  # noqa: E402

quick = len(sys.argv) > 1 and sys.argv[1] == 'quick'
ran = 0
for widths, wname in ((synthetic.STOCK_WIDTHS, 'stock'), (synthetic.PRUNED_WIDTHS, 'pruned')):
    sd = synthetic.synthetic_state_dict(widths)
    for dtype in (torch.float16,) if quick else (torch.float16, torch.bfloat16):
        for (h, w, n) in ((64, 96, 2),) if quick else ((64, 96, 2), (224, 224, 3)):
            m = models.MobileNetSkipAdd((h, w), pretrained=False, widths=widths)
            m.load_state_dict(sd)
            m = m.eval().cuda().to(dtype)
            x = synthetic.synthetic_input(n, h, w, seed=3).cuda().to(dtype)
            ref = {}
            envs = ({}, {'FD_TC_MAX_NCTA': '64', 'FD_TC_CLUSTER': '1'})
            for env, (tma, inpl, fold, graph) in itertools.product(envs if not quick else envs[:1],
                                                                   ((1, 1, 1, 0), (1, 0, 0, 0), (0, 0, 1, 0), (1, 1, 1, 1))):
                for k in ('FD_TC_MAX_NCTA', 'FD_TC_CLUSTER'):
                    os.environ.pop(k, None)
                os.environ.update(env)
                eng = SkipAddEngine(m)
                for k, v in (('tma_epilogue', tma), ('inplace_skip', inpl), ('fold_head', fold), ('graph', graph)):
                    eng.set_option(k, v)
                with torch.no_grad():
                    y = eng(x)
                    y2 = eng(x)                      # second call: graph replay / steady state
                torch.cuda.synchronize()
                assert torch.isfinite(y.float()).all() and torch.equal(y, y2)
                if fold not in ref:                  # the folded head sums its 32 products in another order than head_kernel
                    ref[fold] = y.clone()
                else:
                    assert torch.equal(ref[fold], y), (wname, dtype, h, w, env, tma, inpl, fold, graph)
                eng.refresh()
                ran += 1
print('sanitize_run: %d configurations ran, outputs finite and bit-identical across organisations' % ran)
