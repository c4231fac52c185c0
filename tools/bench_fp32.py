"""fp32 MobileNetSkipAdd on the H100: the split-TF32 pointwise steps ('high') against the fp32 SIMT path ('highest') and
cuDNN eager, one command.

    python tools/bench_fp32.py [--out DIR] [--iters N] [--warmup W] [--runs R]

* ours: stock MobileNetSkipAdd in fp32 at b64 and b1 224^2 through the module's own engine, under
  torch.set_float32_matmul_precision('highest') and ('high'), alternating, R runs each (CUDA events, after a warm-up);
* per-step times from Plan.time_steps (L2 flushed between launches) for both settings; for the split-TF32 steps their
  share of the 495 TFLOP/s dense TF32 data-sheet peak, counting all three products (3 x 2 x MACs);
* cuDNN eager (the same module run layer by layer in PyTorch, cudnn.benchmark) with cudnn.conv.fp32_precision 'tf32'
  (torch's default) and 'ieee', NCHW and channels_last;
* every variant's rel error (tests/conftest.py's rel_err) against the fp32 CPU forward of the same module on 2 images;
* the card name and power limit, read in the same run; everything goes to DIR/bench_fp32.json (default: a directory
  under the system temp dir, so the tree is never written).
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
import torch.nn.functional as F  # noqa: E402

PEAK_TF32 = 495.0          # TFLOP/s, dense, H100 SXM data sheet
PEAK_FP32 = 67.0
CHECK = 2                  # images checked against the CPU forward


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
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


def rel_err(got, want):
    got, want = got.double(), want.double()
    denom = torch.maximum(want.abs(), want.abs().mean())
    return ((got - want).abs() / denom).max().item()


def model():
    import models
    from fastdepth_b200 import synthetic
    m = models.MobileNetSkipAdd((224, 224), pretrained=False, widths=synthetic.STOCK_WIDTHS)
    m.load_state_dict(synthetic.synthetic_state_dict(synthetic.STOCK_WIDTHS, seed=1))
    return m.eval()


def eager(m, x):
    """MobileNetSkipAdd's forward as plain PyTorch layers (encoder, decoder with nearest x2 upsampling, skips added after
    decoder stages 2, 3, 4 from encoder blocks 5, 3, 1)."""
    keep = {}
    for i in range(14):
        x = getattr(m, 'conv%d' % i)(x)
        if i in (1, 3, 5):
            keep[i] = x
    for j, src in ((1, None), (2, 5), (3, 3), (4, 1), (5, None)):
        x = F.interpolate(getattr(m, 'decode_conv%d' % j)(x), scale_factor=2, mode='nearest')
        if src is not None:
            x = x + keep[src]
    return m.decode_conv6(x)


def ours_steps(m, x, prec, iters):
    torch.set_float32_matmul_precision(prec)
    with torch.no_grad():
        m(x)
    p = m.__dict__['_fd_engine'].plan_for(x)
    steps = p.time_steps(x, torch.empty(x.shape[0], 1, 224, 224, device='cuda'), torch.cuda.current_stream().cuda_stream,
                         warmup=2, iters=iters, flush_l2=True)
    rows = []
    for s in steps:
        if s['kernel'] == 'pw_kernel' or s['kernel'].startswith('dw_kernel') or 'tf32x3' in s['kernel']:
            r = dict(stage=s['stage_name'], kernel=s['kernel'], ms=round(s['ms'], 4))
            if 'tf32x3' in s['kernel']:
                tf = 3 * 2 * s['macs'] / (s['ms'] * 1e-3) / 1e12
                r.update(tf32_tflops_3products=round(tf, 1), tf32_peak_share=round(tf / PEAK_TF32, 3))
            elif s['kernel'] == 'pw_kernel':
                tf = 2 * s['macs'] / (s['ms'] * 1e-3) / 1e12
                r.update(fp32_tflops=round(tf, 1), fp32_peak_share=round(tf / PEAK_FP32, 3))
            rows.append(r)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=os.path.join(tempfile.gettempdir(), 'bench_fp32'),
                    help='directory for bench_fp32.json (default: a directory under the system temp dir)')
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--runs', type=int, default=3)
    a = ap.parse_args()
    from fastdepth_b200 import build, synthetic
    build.build()
    res = dict(card=card(), configs=[])
    m_cpu = model()
    prec0 = torch.get_float32_matmul_precision()
    for n in (64, 1):
        x = synthetic.synthetic_input(n, 224, 224, seed=0)
        with torch.no_grad():
            want = eager(m_cpu, x[:CHECK])
        xg = x.cuda()
        m = model().cuda()
        cfg = dict(n=n, h=224, w=224)
        times = {'highest': [], 'high': []}
        for prec in ('highest', 'high'):
            torch.set_float32_matmul_precision(prec)
            with torch.no_grad():
                cfg['rel_err_%s' % prec] = rel_err(m(xg)[:CHECK].cpu(), want)
        for _ in range(a.runs):
            for prec in ('highest', 'high'):
                torch.set_float32_matmul_precision(prec)
                with torch.no_grad():
                    times[prec].append(timed(lambda: m(xg), a.warmup, a.iters))
        for prec, ts in times.items():
            cfg['ours_%s_ms' % prec] = [round(t, 3) for t in ts]
            cfg['ours_%s_img_s' % prec] = round(n / min(ts) * 1e3, 1)
        for prec in ('highest', 'high'):
            cfg['steps_%s' % prec] = ours_steps(m, xg, prec, max(3, a.iters // 2))
        torch.set_float32_matmul_precision(prec0)
        torch.backends.cudnn.benchmark = True
        for conv_prec in ('tf32', 'ieee'):
            torch.backends.cudnn.conv.fp32_precision = conv_prec
            for cl in (False, True):
                me = model().cuda()
                xe = xg
                if cl:
                    me = me.to(memory_format=torch.channels_last)
                    xe = xg.to(memory_format=torch.channels_last)
                key = 'cudnn_%s_%s' % (conv_prec, 'nhwc' if cl else 'nchw')
                with torch.no_grad():
                    t = timed(lambda: eager(me, xe), a.warmup, a.iters)
                    cfg[key + '_ms'] = round(t, 3)
                    cfg[key + '_img_s'] = round(n / t * 1e3, 1)
                    cfg[key + '_rel_err'] = rel_err(eager(me, xe)[:CHECK].float().cpu(), want)
        torch.backends.cudnn.conv.fp32_precision = 'tf32'
        res['configs'].append(cfg)
        print(json.dumps({k: v for k, v in cfg.items() if not k.startswith('steps')}))
        for prec in ('highest', 'high'):
            print('  steps under %r (L2 flushed):' % prec)
            for r in cfg['steps_%s' % prec]:
                extra = {k: v for k, v in r.items() if k not in ('stage', 'kernel', 'ms')}
                print('    %-16s %-64s %8.4f ms  %s' % (r['stage'][:16], r['kernel'][:64], r['ms'], extra or ''))
    res['card_after'] = card()
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, 'bench_fp32.json'), 'w') as f:
        json.dump(res, f, indent=1)
    print('card:', res['card'], '| after:', res['card_after'])
    print('wrote', os.path.join(a.out, 'bench_fp32.json'))


if __name__ == '__main__':
    main()
