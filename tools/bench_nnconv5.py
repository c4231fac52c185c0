"""MobileNet-NNConv5 (dense 5x5 decoder) on the H100: our path against cuDNN eager, one command.

    python tools/bench_nnconv5.py [--out DIR] [--iters N] [--warmup W]

* ours: models.MobileNet('nnconv5') through the C-ABI at b64 224^2 fp16 and bf16 and b16 480x640 fp16 (one fd_forward per
  batch, CUDA graph replay), timed with CUDA events after a warm-up;
* cuDNN eager (cudnn.benchmark=True) on the same model, NCHW and channels_last;
* a per-step table from Plan.time_steps (L2 flushed between launches): kernel, tile, achieved TFLOP/s and its share of the
  989 TFLOP/s dense 16-bit data-sheet peak, HBM share of 3.35 TB/s;
* fp32: stock PyTorch (cuDNN, TF32 allowed as PyTorch's default for convolutions) against path 0 through the C-ABI, the
  measurement behind keeping the fp32 dense decoder on stock PyTorch;
* the card name and power limit, read in the same run; everything goes to DIR/bench_nnconv5.json (default: a
  directory under the system temp dir, so the tree is never written).
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

PEAK_TFLOPS = 989.0
PEAK_HBM = 3.35e12


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                       capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name(0)


def timed(fn, warmup, iters):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def model(dtype, channels_last=False):
    import models
    from fastdepth_b200 import synthetic
    m = models.MobileNet('nnconv5', (224, 224), pretrained=False)
    m.load_state_dict(synthetic.synthetic_nnconv_state_dict(5, seed=1))
    m = m.eval().cuda().to(dtype)
    return m.to(memory_format=torch.channels_last) if channels_last else m


def ours(dtype, n, h, w, warmup, iters, path=1):
    from fastdepth_b200 import plan as _plan
    m = model(dtype)
    p = _plan.Plan.from_module(m, n, h, w, dtype, 0)
    p.set_option('path', path)
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


def cudnn(dtype, n, h, w, warmup, iters, channels_last):
    torch.backends.cudnn.benchmark = True
    m = model(dtype, channels_last)
    x = torch.rand(n, 3, h, w, device='cuda').to(dtype)
    if channels_last:
        x = x.to(memory_format=torch.channels_last)
    with torch.no_grad():
        return timed(lambda: m.decoder(m.mobilenet(x)), warmup, iters)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=os.path.join(tempfile.gettempdir(), 'bench_nnconv5'),
                    help='directory for bench_nnconv5.json (default: a directory under the system temp dir)')
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=10)
    a = ap.parse_args()
    from fastdepth_b200 import build
    build.build()
    res = dict(card=card(), configs=[])
    for dtype, n, h, w in ((torch.float16, 64, 224, 224), (torch.bfloat16, 64, 224, 224), (torch.float16, 16, 480, 640)):
        with torch.no_grad():
            ms, rows = ours(dtype, n, h, w, a.warmup, a.iters)
        cfg = dict(dtype=str(dtype).replace('torch.', ''), n=n, h=h, w=w, ours_ms=round(ms, 3),
                   ours_img_s=round(n / ms * 1e3, 1), steps=rows)
        for cl in (False, True):
            t = cudnn(dtype, n, h, w, a.warmup, a.iters, cl)
            cfg['cudnn_%s_ms' % ('nhwc' if cl else 'nchw')] = round(t, 3)
            cfg['cudnn_%s_img_s' % ('nhwc' if cl else 'nchw')] = round(n / t * 1e3, 1)
        res['configs'].append(cfg)
        print(json.dumps({k: v for k, v in cfg.items() if k != 'steps'}))
        print('  %-22s %-58s %8s %8s %6s %6s' % ('stage', 'kernel', 'ms', 'TFLOP/s', 'peak', 'HBM'))
        for r in rows:
            print('  %-22s %-58s %8.4f %8.1f %6.3f %6.3f' % (r['stage'][:22], r['kernel'][:58], r['ms'], r['tflops'],
                                                          r['peak_share'], r['hbm_share']))
    # fp32: stock (cuDNN, TF32 per PyTorch's conv default) against path 0 through the C-ABI
    n = 16
    with torch.no_grad():
        ms0, _ = ours(torch.float32, n, 224, 224, 2, 5, path=0)
    t32 = cudnn(torch.float32, n, 224, 224, 3, 10, False)
    res['fp32'] = dict(n=n, path0_ms=round(ms0, 3), stock_ms=round(t32, 3),
                       allow_tf32_conv=bool(torch.backends.cudnn.allow_tf32))
    print(json.dumps(res['fp32']))
    res['card_after'] = card()
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, 'bench_nnconv5.json'), 'w') as f:
        json.dump(res, f, indent=1)
    print('card:', res['card'])
    print('wrote', os.path.join(a.out, 'bench_nnconv5.json'))


if __name__ == '__main__':
    main()
