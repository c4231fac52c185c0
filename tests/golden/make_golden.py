"""Generate the golden fixtures in this directory FROM THE LIVE REFERENCE.

Run with a checkout of the reference (dwofk/fast-depth) at hand:

    python tests/golden/make_golden.py /path/to/fast-depth

It imports the reference's own ``models.py`` / ``metrics.py`` read-only under alias module
names (the repo has same-named top-level modules), instantiates the reference's
``MobileNetSkipAdd`` (models.py:654-732), loads the seeded synthetic state_dict from
``fastdepth_b200.synthetic`` and records the reference forward's outputs.  Nothing from the
reference is copied: only numbers it computed.  The tests read the committed .npz files and
never need the reference itself.
"""
import importlib.util
import os
import sys

import numpy as np
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.path.abspath(sys.argv[1]) if len(sys.argv) > 1 else None
sys.path.insert(0, ROOT)

from fastdepth_b200 import synthetic  # noqa: E402

STAGE_NAMES = ['conv%d' % i for i in range(14)] + ['decode_conv%d' % j for j in range(1, 7)]
N_SAMPLE = 96


def load_reference():
    """Load the reference's {models,metrics}.py as ref_models / ref_metrics.  The reference does
    ``import imagenet.mobilenet`` (models.py:8), so point those names at ITS copies meanwhile."""
    saved = {k: sys.modules.get(k) for k in ('imagenet', 'imagenet.mobilenet', 'models', 'metrics')}
    for k in saved:
        sys.modules.pop(k, None)
    sys.path.insert(0, REF)
    try:
        spec = importlib.util.spec_from_file_location('ref_models', os.path.join(REF, 'models.py'))
        ref_models = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(ref_models)
        spec = importlib.util.spec_from_file_location('ref_metrics', os.path.join(REF, 'metrics.py'))
        ref_metrics = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(ref_metrics)
    finally:
        sys.path.remove(REF)
        for k in ('imagenet', 'imagenet.mobilenet'):
            sys.modules.pop(k, None)
        for k, v in saved.items():
            if v is not None:
                sys.modules[k] = v
    return ref_models, ref_metrics


def reference_module(ref_models, widths):
    """The reference's MobileNetSkipAdd; for pruned widths its children are re-built with the
    reference's OWN builders (models.depthwise / models.pointwise) and stock nn layers in the
    conv_dw pattern (imagenet/mobilenet.py:29-38) -- forward() is width-agnostic."""
    m = ref_models.MobileNetSkipAdd((224, 224), pretrained=False)
    enc, dec = widths
    if tuple(enc) != synthetic.STOCK_ENCODER or tuple(dec) != synthetic.STOCK_DECODER:
        strides = (2, 1, 2, 1, 2, 1, 2, 1, 1, 1, 1, 1, 2, 1)
        m.conv0 = nn.Sequential(nn.Conv2d(3, enc[0], 3, 2, 1, bias=False), nn.BatchNorm2d(enc[0]),
                                nn.ReLU6(inplace=True))
        for i in range(1, 14):
            ci, co = enc[i - 1], enc[i]
            setattr(m, 'conv%d' % i, nn.Sequential(
                nn.Conv2d(ci, ci, 3, strides[i], 1, groups=ci, bias=False), nn.BatchNorm2d(ci),
                nn.ReLU6(inplace=True),
                nn.Conv2d(ci, co, 1, 1, 0, bias=False), nn.BatchNorm2d(co), nn.ReLU6(inplace=True)))
        c = enc[13]
        for j, co in enumerate(dec, start=1):
            setattr(m, 'decode_conv%d' % j,
                    nn.Sequential(ref_models.depthwise(c, 5), ref_models.pointwise(c, co)))
            c = co
        m.decode_conv6 = ref_models.pointwise(c, 1)
    return m.eval()


def sample_index(numel, seed):
    rng = np.random.Generator(np.random.PCG64(seed))
    return np.sort(rng.choice(numel, size=min(N_SAMPLE, numel), replace=False))


def make_forward_fixture(ref_models, name, widths, n, h, w, wseed=1, xseed=0):
    sd = synthetic.synthetic_state_dict(widths, seed=wseed)
    m = reference_module(ref_models, widths)
    missing = m.load_state_dict(sd, strict=True)
    x = synthetic.synthetic_input(n, h, w, seed=xseed)
    outs = {}
    hooks = [getattr(m, s).register_forward_hook(
        lambda mod, inp, out, s=s: outs.__setitem__(s, out.detach().clone())) for s in STAGE_NAMES]
    with torch.no_grad():
        y = m(x)
    for hk in hooks:
        hk.remove()
    # decode_conv1..5 hooks see the block output BEFORE interpolate/add; record that (".pw")
    fix = {'widths_enc': np.asarray(widths[0]), 'widths_dec': np.asarray(widths[1]),
           'shape': np.asarray([n, h, w]), 'wseed': np.asarray(wseed), 'xseed': np.asarray(xseed),
           'output': y.numpy()}
    print('== %s: out range %.4g..%.4g mean %.4g frac_zero %.3f' %
          (name, y.min(), y.max(), y.mean(), (y == 0).float().mean()))
    for k, s in enumerate(STAGE_NAMES):
        t = outs[s]
        key = s if not s.startswith('decode_conv') or s == 'decode_conv6' else s + '.pw'
        idx = sample_index(t.numel(), seed=100 + k)
        fix['stage/%s/shape' % key] = np.asarray(t.shape)
        fix['stage/%s/idx' % key] = idx
        fix['stage/%s/val' % key] = t.reshape(-1)[idx].numpy()
        fix['stage/%s/absmean' % key] = np.asarray(t.abs().double().mean().item())
        sat = (t >= 6.0).float().mean().item() if s.startswith('conv') else 0.0
        print('   %-14s %-22s absmean %.4g max %.4g zero %.3f sat6 %.4f' %
              (key, tuple(t.shape), t.abs().mean(), t.max(), (t == 0).float().mean(), sat))
    assert (y == 0).float().mean() < 0.5, 'dead output: parity would be vacuous'
    np.savez_compressed(os.path.join(HERE, name + '.npz'), **fix)


def make_nnconv_dw_fixture(ref_models, name, n, h, w, wseed=1, xseed=0):
    """reference models.MobileNet(decoder='nnconv5dw') (models.py:420-460 with NNConv(5, dw=True), l.229-244,
    253-270): the SkipAdd topology without skips -- SURVEY.md section 8f row 2."""
    sd = synthetic.to_mobilenet_keys(synthetic.synthetic_state_dict(synthetic.STOCK_WIDTHS, seed=wseed))
    m = ref_models.MobileNet('nnconv5dw', (224, 224), pretrained=False)
    m.load_state_dict(sd, strict=True)
    m.eval()
    x = synthetic.synthetic_input(n, h, w, seed=xseed)
    with torch.no_grad():
        y = m(x)
    print('== %s: out range %.4g..%.4g mean %.4g frac_zero %.3f' % (name, y.min(), y.max(), y.mean(), (y == 0).float().mean()))
    assert (y == 0).float().mean() < 0.5
    np.savez_compressed(os.path.join(HERE, name + '.npz'), shape=np.asarray([n, h, w]), wseed=np.asarray(wseed),
                        xseed=np.asarray(xseed), output=y.numpy())


def make_skipconcat_fixture(ref_models, name, n, h, w, wseed=1, xseed=0):
    """reference models.MobileNetSkipConcat (models.py:734-814) -- SURVEY.md section 8f row 1."""
    sd = synthetic.synthetic_state_dict(synthetic.STOCK_WIDTHS, seed=wseed, skip='concat')
    m = ref_models.MobileNetSkipConcat((224, 224), pretrained=False)
    m.load_state_dict(sd, strict=True)
    m.eval()
    x = synthetic.synthetic_input(n, h, w, seed=xseed)
    with torch.no_grad():
        y = m(x)
    print('== %s: out range %.4g..%.4g mean %.4g frac_zero %.3f' % (name, y.min(), y.max(), y.mean(), (y == 0).float().mean()))
    assert (y == 0).float().mean() < 0.5
    np.savez_compressed(os.path.join(HERE, name + '.npz'), shape=np.asarray([n, h, w]), wseed=np.asarray(wseed),
                        xseed=np.asarray(xseed), output=y.numpy())


def make_metrics_fixture(ref_metrics):
    """Known answer for metrics.Result.evaluate (reference metrics.py:31-55) on the reference's own
    sample (deploy/data/pred.npy vs depth.npy), subsampled 4x so the fixture stays small, plus a
    synthetic multi-image case that pins the per-image AverageMeter semantics (metrics.py:71-95)."""
    pred = np.load(os.path.join(REF, 'deploy/data/pred.npy')).reshape(224, 224)
    depth = np.load(os.path.join(REF, 'deploy/data/depth.npy')).reshape(224, 224)
    fix = {}
    names = ('irmse', 'imae', 'mse', 'rmse', 'mae', 'absrel', 'lg10', 'delta1', 'delta2', 'delta3')

    def run(o, t):
        r = ref_metrics.Result()
        r.evaluate(torch.from_numpy(np.ascontiguousarray(o)), torch.from_numpy(np.ascontiguousarray(t)))
        return np.asarray([getattr(r, k) for k in names], dtype=np.float64)

    full = run(pred, depth)
    print('metrics full  :', dict(zip(names, np.round(full, 4))))
    fix['names'] = np.asarray(names)
    fix['full_values'] = full                      # RMSE 618.001 etc. (SURVEY.md section 4)
    p4, d4 = pred[::4, ::4].copy(), depth[::4, ::4].copy()
    fix['pred_sub4'] = p4.astype(np.float32)
    fix['depth_sub4'] = d4.astype(np.float32)
    fix['sub4_values'] = run(p4, d4)
    # per-image averaging: 3 images, one with zero-target holes (exercises the OR mask)
    rng = np.random.Generator(np.random.PCG64(7))
    outs = (rng.random((3, 1, 24, 32), dtype=np.float32) * 4 + 0.5).astype(np.float32)
    tgts = (outs * (1 + 0.2 * rng.standard_normal(outs.shape).astype(np.float32))).clip(1e-3, None).astype(np.float32)
    tgts[1, 0, :4, :] = 0.0
    outs[1, 0, :2, :] = 0.0                         # both zero on 2 rows -> masked out
    meter = ref_metrics.AverageMeter()
    for i in range(3):
        r = ref_metrics.Result()
        r.evaluate(torch.from_numpy(outs[i:i + 1]), torch.from_numpy(tgts[i:i + 1]))
        meter.update(r, 0.0, 0.0, 1)
    avg = meter.average()
    fix['multi_out'] = outs
    fix['multi_tgt'] = tgts
    fix['multi_avg'] = np.asarray([getattr(avg, k) for k in names], dtype=np.float64)
    np.savez_compressed(os.path.join(HERE, 'metrics_known_answer.npz'), **fix)


if __name__ == '__main__':
    if REF is None:
        raise SystemExit('usage: make_golden.py <path of a dwofk/fast-depth checkout>')
    torch.manual_seed(0)
    torch.set_num_threads(8)
    ref_models, ref_metrics = load_reference()
    make_forward_fixture(ref_models, 'skipadd_stock_2x64x96', synthetic.STOCK_WIDTHS, 2, 64, 96)
    make_forward_fixture(ref_models, 'skipadd_pruned_2x64x96', synthetic.PRUNED_WIDTHS, 2, 64, 96)
    make_forward_fixture(ref_models, 'skipadd_stock_1x224x224', synthetic.STOCK_WIDTHS, 1, 224, 224)
    make_nnconv_dw_fixture(ref_models, 'nnconv5dw_stock_2x64x96', 2, 64, 96)
    make_skipconcat_fixture(ref_models, 'skipconcat_stock_2x64x96', 2, 64, 96)
    make_metrics_fixture(ref_metrics)
    print('wrote fixtures to', HERE)
