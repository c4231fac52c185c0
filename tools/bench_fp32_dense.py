"""fp32 dense decoders on the H100: the split-TF32 engine ('high') against cuDNN eager, one command.

    python tools/bench_fp32_dense.py [--out DIR] [--iters N] [--warmup W] [--runs R] [--decoders a,b,...]

* ours: MobileNet('nnconv5'), ('deconv3' / '5' / '7' / '9') and ('upconv') in fp32 at b64 and b1 224^2 through the module's
  own engine under torch.set_float32_matmul_precision('high'), R runs (CUDA events, after a warm-up);
* per-step times from Plan.time_steps (L2 flushed between launches); for the split-TF32 steps their share of the
  495 TFLOP/s dense TF32 data-sheet peak, counting all three products (3 x 2 x MACs);
* cuDNN eager (the same module's encoder and decoder in PyTorch, cudnn.benchmark) with cudnn.conv.fp32_precision 'tf32'
  (torch's default) and 'ieee', NCHW and channels_last;
* every variant's rel error (tests/conftest.py's rel_err) against the fp32 CPU forward of the same module on 2 images;
* the card name and power limit, read in the same run; everything goes to DIR/bench_fp32_dense.json (default: a
  directory under the system temp dir, so the tree is never written).
"""
import argparse
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch  # noqa: E402

from bench_fp32 import CHECK, PEAK_TF32, card, rel_err, timed  # noqa: E402

DECODERS = ('nnconv5', 'deconv3', 'deconv5', 'deconv7', 'deconv9', 'upconv')


def model(decoder):
    import models
    from fastdepth_b200 import synthetic
    m = models.MobileNet(decoder, (224, 224), pretrained=False)
    if decoder == 'nnconv5':
        m.load_state_dict(synthetic.synthetic_nnconv_state_dict(5, seed=1))
    else:
        m.load_state_dict(synthetic.synthetic_convt_state_dict(decoder, seed=1))
    return m.eval()


def eager(m, x):
    """The module's stock PyTorch forward, whatever the matmul precision."""
    return m.decoder(m.mobilenet(x))


def ours_steps(m, x, iters):
    p = m.__dict__['_fd_engine'].plan_for(x)
    steps = p.time_steps(x, torch.empty(x.shape[0], 1, 224, 224, device='cuda'), torch.cuda.current_stream().cuda_stream,
                         warmup=2, iters=iters, flush_l2=True)
    rows = []
    for s in steps:
        r = dict(stage=s['stage_name'], kernel=s['kernel'], ms=round(s['ms'], 4))
        if 'tf32x3' in s['kernel']:
            tf = 3 * 2 * s['macs'] / (s['ms'] * 1e-3) / 1e12
            r.update(tf32_tflops_3products=round(tf, 1), tf32_peak_share=round(tf / PEAK_TF32, 3))
        rows.append(r)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=os.path.join(tempfile.gettempdir(), 'bench_fp32_dense'),
                    help='directory for bench_fp32_dense.json (default: a directory under the system temp dir)')
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--decoders', default=','.join(DECODERS))
    a = ap.parse_args()
    from fastdepth_b200 import build, synthetic
    build.build()
    res = dict(card=card(), configs=[])
    prec0 = torch.get_float32_matmul_precision()
    for dec in a.decoders.split(','):
        m_cpu = model(dec)
        for n in (64, 1):
            x = synthetic.synthetic_input(n, 224, 224, seed=0)
            with torch.no_grad():
                want = eager(m_cpu, x[:CHECK])
            xg = x.cuda()
            m = model(dec).cuda()
            cfg = dict(decoder=dec, n=n, h=224, w=224)
            torch.set_float32_matmul_precision('high')
            with torch.no_grad():
                cfg['ours_high_rel_err'] = rel_err(m(xg)[:CHECK].cpu(), want)
                ts = [timed(lambda: m(xg), a.warmup, a.iters) for _ in range(a.runs)]
            cfg['ours_high_ms'] = [round(t, 3) for t in ts]
            cfg['ours_high_img_s'] = round(n / min(ts) * 1e3, 1)
            cfg['steps_high'] = ours_steps(m, xg, max(3, a.iters // 2))
            torch.set_float32_matmul_precision(prec0)
            del m
            torch.backends.cudnn.benchmark = True
            for conv_prec in ('tf32', 'ieee'):
                torch.backends.cudnn.conv.fp32_precision = conv_prec
                for cl in (False, True):
                    me = model(dec).cuda()
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
                    del me
            torch.backends.cudnn.conv.fp32_precision = 'tf32'
            torch.backends.cudnn.benchmark = False
            res['configs'].append(cfg)
            print(json.dumps({k: v for k, v in cfg.items() if not k.startswith('steps')}))
            print("  steps under 'high' (L2 flushed):")
            for r in cfg['steps_high']:
                extra = {k: v for k, v in r.items() if k not in ('stage', 'kernel', 'ms')}
                print('    %-16s %-64s %8.4f ms  %s' % (r['stage'][:16], r['kernel'][:64], r['ms'], extra or ''))
            torch.cuda.empty_cache()
    res['card_after'] = card()
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, 'bench_fp32_dense.json'), 'w') as f:
        json.dump(res, f, indent=1)
    print('card:', res['card'], '| after:', res['card_after'])
    print('wrote', os.path.join(a.out, 'bench_fp32_dense.json'))


if __name__ == '__main__':
    main()
