"""In-channel counts on the engine: MobileNet(decoder, in_channels=k) at b64 224x224 against stock cuDNN eager.

For every (decoder, c_in) of the sweep (nnconv5dw with c_in 1, 3, 4, 7 and upconv with c_in 4), in fp16 and bf16:
* the engine's forward (graph replay, CUDA events) and the best of stock PyTorch eager in NCHW and ``channels_last``
  (cuDNN, ``torch.backends.cudnn.benchmark`` on), us per batch;
* the step times of conv0..conv2 through ``plan.time_steps`` (L2 flushed before every launch), with ``front`` 1 and 0
  alternating where the front route can take that c_in (1..4), and the kernels that ran;
* that ``front`` 1 and 0 give the same depth map.
The card name, power limit and max SM clock are read in the same run.
usage: python tools/bench_in_channels.py [--repeats 3] [--forwards 100] [--dtypes f16,bf16]"""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import models  # noqa: E402
from fastdepth_b200 import synthetic  # noqa: E402
from fastdepth_b200.engine import SkipAddEngine  # noqa: E402

N, H, W = 64, 224, 224
SWEEP = (('nnconv5dw', 1), ('nnconv5dw', 3), ('nnconv5dw', 4), ('nnconv5dw', 7), ('upconv', 4))
FRONT = ('mobilenet.0', 'mobilenet.1', 'mobilenet.2')      # conv0..conv2


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def timed(fn, forwards):
    for _ in range(10):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(forwards):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / forwards * 1e3


def state_dict(decoder, c_in):
    if decoder == 'nnconv5dw':
        return synthetic.to_mobilenet_keys(synthetic.synthetic_state_dict(synthetic.STOCK_WIDTHS, seed=1, in_channels=c_in))
    return synthetic.synthetic_convt_state_dict(decoder, seed=1, in_channels=c_in)


def rng(t):
    return '%7.1f-%-7.1f' % (min(t), max(t))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--forwards', type=int, default=100)
    ap.add_argument('--dtypes', default='f16,bf16')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_in_channels needs a GPU')
    torch.backends.cudnn.benchmark = True
    print('card: %s   b%d %dx%d' % (card(), N, H, W))
    sp = torch.cuda.current_stream().cuda_stream
    for dn in a.dtypes.split(','):
        dtype = {'f16': torch.float16, 'bf16': torch.bfloat16}[dn]
        for decoder, c_in in SWEEP:
            m = models.MobileNet(decoder, (H, W), in_channels=c_in, pretrained=False)
            m.load_state_dict(state_dict(decoder, c_in))
            m = m.eval().cuda().to(dtype)
            xs = [synthetic.synthetic_input(N, H, W, seed=i, channels=c_in).cuda().to(dtype) for i in range(2)]
            ys = [torch.empty((N, 1, H, W), dtype=dtype, device='cuda') for _ in range(2)]
            fronts = (1, 0) if c_in <= 4 else (1,)
            engines = {}
            for f in fronts:
                engines[f] = SkipAddEngine(m)
                engines[f].set_option('front', f)
            res = {f: dict(graph=[], steps=[]) for f in fronts}
            eager = {'nchw': [], 'channels_last': []}
            m_cl = models.MobileNet(decoder, (H, W), in_channels=c_in, pretrained=False)
            m_cl.load_state_dict(state_dict(decoder, c_in))
            m_cl = m_cl.eval().cuda().to(dtype).to(memory_format=torch.channels_last)
            xs_cl = [x.contiguous(memory_format=torch.channels_last) for x in xs]
            names, same = {}, None
            for rep in range(a.repeats):
                for f in fronts:
                    p = engines[f].plan_for(xs[0])
                    if rep == 0:
                        names[f] = [s['kernel'] for s in p.steps() if s['stage_name'] in FRONT]
                        p.forward(xs[0], ys[0], sp)
                        torch.cuda.synchronize()
                        if f == fronts[0]:
                            ref = ys[0].clone()
                        else:
                            same = torch.equal(ref, ys[0])
                    per = sum(s['ms'] * 1e3 for s in p.time_steps(xs[0], ys[0], sp, warmup=3, iters=20, flush_l2=True)
                              if s['stage_name'] in FRONT)
                    res[f]['steps'].append(per)
                    k = [0]

                    def one():
                        p.forward(xs[k[0] & 1], ys[k[0] & 1], sp)
                        k[0] += 1
                    res[f]['graph'].append(timed(one, a.forwards))
                with torch.no_grad():
                    k = [0]

                    def nchw():
                        m.decoder(m.mobilenet(xs[k[0] & 1]))      # stock PyTorch layers, bypassing the engine
                        k[0] += 1

                    def cl():
                        m_cl.decoder(m_cl.mobilenet(xs_cl[k[0] & 1]))
                        k[0] += 1
                    eager['nchw'].append(timed(nchw, max(10, a.forwards // 4)))
                    eager['channels_last'].append(timed(cl, max(10, a.forwards // 4)))
            best = min(eager, key=lambda v: min(eager[v]))
            print('\n%s %s in_channels=%d' % (dn, decoder, c_in))
            for f in fronts:
                print('  front=%d  conv0..conv2 steps %s us: %s' % (f, rng(res[f]['steps']), ' | '.join(names[f])))
                print('  front=%d  engine forward   %s us  (%.0f img/s best)' %
                      (f, rng(res[f]['graph']), N / min(res[f]['graph']) * 1e6))
            print('  eager    %-13s %s us  (%.0f img/s best); other layout %s us' %
                  (best, rng(eager[best]), N / min(eager[best]) * 1e6, rng(eager['nchw' if best != 'nchw' else 'channels_last'])))
            print('  engine / best eager: %.2fx' % (min(eager[best]) / min(res[1]['graph'])))
            if same is not None:
                print('  depth map front=1 equals front=0: %s' % same)
            for e in engines.values():
                e.refresh()
            del m, m_cl
            torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
