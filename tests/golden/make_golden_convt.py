"""Generate the DeConv / UpConv golden fixtures (``{upconv5,deconv3,deconv5,deconv7,deconv9}_stock_*.npz``) FROM THE LIVE
REFERENCE.

    python tests/golden/make_golden_convt.py /path/to/fast-depth

Loads the reference's own ``models.py`` the way ``make_golden.py`` does, instantiates its ``MobileNet('upconv')`` /
``MobileNet('deconv<k>')`` (models.py:420-460 with UpConv, l.183-201, or DeConv(k, dw=False), l.145-180), loads
``fastdepth_b200.synthetic.synthetic_convt_state_dict`` and records the reference forward's output, plus the reference
module's state_dict keys and shapes (the schema the tests hold models.MobileNet to).  Only these fixtures are written.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden  # noqa: E402
from fastdepth_b200 import synthetic  # noqa: E402


def make_convt_fixture(ref_models, decoder, name, n, h, w, wseed=1, xseed=0):
    sd = synthetic.synthetic_convt_state_dict(decoder, seed=wseed)
    m = ref_models.MobileNet(decoder, (224, 224), pretrained=False)
    m.load_state_dict(sd, strict=True)
    m.eval()
    x = synthetic.synthetic_input(n, h, w, seed=xseed)
    with torch.no_grad():
        y = m(x)
    print('== %s: out range %.4g..%.4g mean %.4g frac_zero %.3f' % (name, y.min(), y.max(), y.mean(), (y == 0).float().mean()))
    assert (y == 0).float().mean() < 0.5
    keys = sorted(m.state_dict().keys())
    shapes = [','.join(str(d) for d in m.state_dict()[k].shape) for k in keys]
    np.savez_compressed(os.path.join(HERE, name + '.npz'), shape=np.asarray([n, h, w]), wseed=np.asarray(wseed),
                        xseed=np.asarray(xseed), decoder=np.asarray(decoder), output=y.numpy(),
                        state_dict_keys=np.asarray(keys), state_dict_shapes=np.asarray(shapes))


if __name__ == '__main__':
    if make_golden.REF is None:
        raise SystemExit('usage: make_golden_convt.py <path of a dwofk/fast-depth checkout>')
    torch.manual_seed(0)
    torch.set_num_threads(8)
    ref_models, _ = make_golden.load_reference()
    for dec, tag in (('upconv', 'upconv5'), ('deconv3', 'deconv3'), ('deconv5', 'deconv5'), ('deconv7', 'deconv7'),
                     ('deconv9', 'deconv9')):
        make_convt_fixture(ref_models, dec, '%s_stock_2x64x96' % tag, 2, 64, 96)
    make_convt_fixture(ref_models, 'upconv', 'upconv5_stock_1x224x224', 1, 224, 224)
    make_convt_fixture(ref_models, 'deconv5', 'deconv5_stock_1x224x224', 1, 224, 224)
    print('wrote fixtures to', HERE)
