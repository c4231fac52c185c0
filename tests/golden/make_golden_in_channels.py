"""Generate the in_channels golden fixtures (``nnconv5dw_cin{1,4}_*.npz``, ``upconv5_cin4_*.npz``) FROM THE LIVE REFERENCE.

    python tests/golden/make_golden_in_channels.py /path/to/fast-depth

Loads the reference's own ``models.py`` the way ``make_golden.py`` does, instantiates its
``MobileNet(decoder, (224, 224), in_channels=k, pretrained=False)`` (models.py:420-460; for k != 3 the stem is its own
``conv_bn(k, 32, 2)``, l.443-453), loads the seeded, BN-calibrated synthetic weights of ``tests/in_channels_ref.py`` and
records the reference forward's output on ``synthetic_input(..., channels=k)`` (image channels plus a sparse depth
channel).  It prints each golden's storage-emulated conditioning (fp16 / bf16 forward against fp32).  Only these fixtures
are written.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import make_golden  # noqa: E402
import in_channels_ref as icr  # noqa: E402


def make_fixture(ref_models, name):
    decoder, c, n, h, w = icr.GOLDENS[name]
    sd = icr.state_dict(decoder, c)
    m = ref_models.MobileNet(decoder, (224, 224), in_channels=c, pretrained=False)
    m.load_state_dict(sd, strict=True)
    m.eval()
    x = icr.golden_input(name)
    with torch.no_grad():
        y = m(x)
    print('== %s: out range %.4g..%.4g mean %.4g frac_zero %.3f  conditioning %s' %
          (name, y.min(), y.max(), y.mean(), (y == 0).float().mean(), icr.conditioning(name)))
    assert (y == 0).float().mean() < 0.5
    keys = sorted(m.state_dict().keys())
    shapes = [','.join(str(d) for d in m.state_dict()[k].shape) for k in keys]
    np.savez_compressed(os.path.join(HERE, name + '.npz'), shape=np.asarray([n, h, w]), in_channels=np.asarray(c),
                        wseed=np.asarray(1), xseed=np.asarray(0), decoder=np.asarray(decoder), output=y.numpy(),
                        state_dict_keys=np.asarray(keys), state_dict_shapes=np.asarray(shapes))


if __name__ == '__main__':
    if make_golden.REF is None:
        raise SystemExit('usage: make_golden_in_channels.py <path of a dwofk/fast-depth checkout>')
    torch.manual_seed(0)
    torch.set_num_threads(8)
    ref_models, _ = make_golden.load_reference()
    for name in icr.GOLDENS:
        make_fixture(ref_models, name)
    print('wrote fixtures to', HERE)
