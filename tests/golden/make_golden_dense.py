"""Generate the dense-decoder golden fixtures (``nnconv5_stock_*.npz``) FROM THE LIVE REFERENCE.

    python tests/golden/make_golden_dense.py /path/to/fast-depth

Loads the reference's own ``models.py`` the way ``make_golden.py`` does, instantiates its ``MobileNet('nnconv5')``
(models.py:420-460 with NNConv(5, dw=False), l.245-270), loads ``fastdepth_b200.synthetic.synthetic_nnconv_state_dict``
and records the reference forward's output.  Only the two new fixtures are written; the others stay as they are.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden  # noqa: E402
from fastdepth_b200 import synthetic  # noqa: E402


def make_nnconv_dense_fixture(ref_models, name, n, h, w, wseed=1, xseed=0):
    sd = synthetic.synthetic_nnconv_state_dict(5, seed=wseed)
    m = ref_models.MobileNet('nnconv5', (224, 224), pretrained=False)
    m.load_state_dict(sd, strict=True)
    m.eval()
    x = synthetic.synthetic_input(n, h, w, seed=xseed)
    with torch.no_grad():
        y = m(x)
    print('== %s: out range %.4g..%.4g mean %.4g frac_zero %.3f' % (name, y.min(), y.max(), y.mean(), (y == 0).float().mean()))
    assert (y == 0).float().mean() < 0.5
    np.savez_compressed(os.path.join(HERE, name + '.npz'), shape=np.asarray([n, h, w]), wseed=np.asarray(wseed),
                        xseed=np.asarray(xseed), kernel_size=np.asarray(5), output=y.numpy())


if __name__ == '__main__':
    if make_golden.REF is None:
        raise SystemExit('usage: make_golden_dense.py <path of a dwofk/fast-depth checkout>')
    torch.manual_seed(0)
    torch.set_num_threads(8)
    ref_models, _ = make_golden.load_reference()
    make_nnconv_dense_fixture(ref_models, 'nnconv5_stock_2x64x96', 2, 64, 96)
    make_nnconv_dense_fixture(ref_models, 'nnconv5_stock_1x224x224', 1, 224, 224)
    print('wrote fixtures to', HERE)
