"""MobileNet-UpConv and MobileNet-DeConv{3,5,7,9} on the H100: our path against cuDNN eager, one command.

    python tools/bench_convt.py [--out DIR] [--iters N] [--warmup W] [--decoders upconv,deconv5,...]

* ours: models.MobileNet(decoder) through the C-ABI at b64 224^2 in fp16 and bf16 (one fd_forward per batch, CUDA graph
  replay), timed with CUDA events after a warm-up;
* cuDNN eager (cudnn.benchmark=True) on the same model, NCHW and channels_last;
* a per-step table from Plan.time_steps (L2 flushed between launches): kernel, tile, achieved TFLOP/s (MACs the
  algorithm needs: k*k*c_in*c_out per input pixel for a DECONV / UPCONV stage) and its share of the 989 TFLOP/s dense
  16-bit data-sheet peak, HBM share of 3.35 TB/s;
* the card name and power limit, read in the same run; everything goes to DIR/bench_convt.json (default: a directory
  under the system temp dir, so the tree is never written).
"""
import argparse
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import torch  # noqa: E402

from bench_nnconv5 import PEAK_HBM, PEAK_TFLOPS, card, timed  # noqa: E402

DECODERS = ('upconv', 'deconv3', 'deconv5', 'deconv7', 'deconv9')


def model(decoder, dtype, channels_last=False):
    import models
    from fastdepth_b200 import synthetic
    m = models.MobileNet(decoder, (224, 224), pretrained=False)
    m.load_state_dict(synthetic.synthetic_convt_state_dict(decoder, seed=1))
    m = m.eval().cuda().to(dtype)
    return m.to(memory_format=torch.channels_last) if channels_last else m


def ours(decoder, dtype, n, h, w, warmup, iters):
    from fastdepth_b200 import plan as _plan
    p = _plan.Plan.from_module(model(decoder, dtype), n, h, w, dtype, 0)
    x = torch.rand(n, 3, h, w, device='cuda').to(dtype)
    y = torch.empty(n, 1, h, w, device='cuda', dtype=dtype)
    st = torch.cuda.current_stream().cuda_stream
    ms = timed(lambda: p.forward(x, y, st), warmup, iters)
    steps = p.time_steps(x, y, st, warmup=2, iters=max(3, iters // 4), flush_l2=True)
    rows = []
    for s in steps:
        tf = 2 * s['macs'] / (s['ms'] * 1e-3) / 1e12 if s['ms'] > 0 else 0.0
        rows.append(dict(stage=s['stage_name'], kernel=s['kernel'], ms=round(s['ms'], 4), tflops=round(tf, 1),
                         peak_share=round(tf / PEAK_TFLOPS, 3),
                         hbm_share=round(s['alg_bytes'] / (s['ms'] * 1e-3) / PEAK_HBM, 3) if s['ms'] > 0 else 0.0))
    p.close()
    return ms, rows


def cudnn(decoder, dtype, n, h, w, warmup, iters, channels_last):
    torch.backends.cudnn.benchmark = True
    m = model(decoder, dtype, channels_last)
    x = torch.rand(n, 3, h, w, device='cuda').to(dtype)
    if channels_last:
        x = x.to(memory_format=torch.channels_last)
    with torch.no_grad():
        return timed(lambda: m.decoder(m.mobilenet(x)), warmup, iters)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=os.path.join(tempfile.gettempdir(), 'bench_convt'),
                    help='directory for bench_convt.json (default: a directory under the system temp dir)')
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=10)
    ap.add_argument('--decoders', default=','.join(DECODERS))
    a = ap.parse_args()
    from fastdepth_b200 import build
    build.build()
    res = dict(card=card(), configs=[])
    n, h, w = 64, 224, 224
    for decoder in a.decoders.split(','):
        for dtype in (torch.float16, torch.bfloat16):
            with torch.no_grad():
                ms, rows = ours(decoder, dtype, n, h, w, a.warmup, a.iters)
            cfg = dict(decoder=decoder, dtype=str(dtype).replace('torch.', ''), n=n, h=h, w=w, ours_ms=round(ms, 3),
                       ours_img_s=round(n / ms * 1e3, 1), steps=rows)
            for cl in (False, True):
                t = cudnn(decoder, dtype, n, h, w, a.warmup, a.iters, cl)
                cfg['cudnn_%s_ms' % ('nhwc' if cl else 'nchw')] = round(t, 3)
            res['configs'].append(cfg)
            print(json.dumps({k: v for k, v in cfg.items() if k != 'steps'}))
            print('  %-22s %-58s %8s %8s %6s %6s' % ('stage', 'kernel', 'ms', 'TFLOP/s', 'peak', 'HBM'))
            for r in rows:
                print('  %-22s %-58s %8.4f %8.1f %6.3f %6.3f' % (r['stage'][:22], r['kernel'][:58], r['ms'], r['tflops'],
                                                              r['peak_share'], r['hbm_share']))
    res['card_after'] = card()
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, 'bench_convt.json'), 'w') as f:
        json.dump(res, f, indent=1)
    print('card:', res['card'])
    print('wrote', os.path.join(a.out, 'bench_convt.json'))


if __name__ == '__main__':
    main()
