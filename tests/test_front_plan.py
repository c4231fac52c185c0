"""Eligibility and budget of the front kernel (plan option ``front``: the stem, conv1 and conv2 as one step), without a GPU.

The route is taken only by 16-bit plans whose stem and first two blocks have the stock MobileNet shapes (3 -> 32 -> 64 ->
128, strides 2, 1, 2), with no skip into those blocks and no concatenation onto their outputs.  The pruned widths,
SkipConcat (conv1 is a channel slice of decode_conv4's buffer) and every kernel-sweep topology keep three steps."""
import ctypes

import pytest
import torch

import test_kernel_sweep as ks
from fastdepth_b200 import _lib
from fastdepth_b200 import plan as fplan
from fastdepth_b200 import synthetic

KEYS = ('ok', 'items', 'smem_bytes', 'ctas_per_sm', 'threads', 'param_bytes', 'a_bytes', 'tile_bytes')
SM_SMEM = 228 * 1024                 # shared memory of one H100 SM
CTA_RESERVED = 1024                  # the runtime's reservation per resident CTA
DT = {torch.float16: 1, torch.bfloat16: 2, torch.float32: 0}


@pytest.fixture(scope='module')
def lib():
    return _lib.load()


def front(lib, descs, n, h, w, dtype=torch.float16):
    arr = (_lib.StageDesc * len(descs))(*[_lib.StageDesc(**d) for d in descs])
    out = (ctypes.c_int * 8)()
    assert lib.fd_debug_front_plan(arr, len(descs), DT[dtype], n, h, w, out, 8) == 0
    return dict(zip(KEYS, out))


def _descs(net):
    import models
    if net in ('stock', 'pruned'):
        widths = synthetic.STOCK_WIDTHS if net == 'stock' else synthetic.PRUNED_WIDTHS
        m = models.MobileNetSkipAdd((224, 224), pretrained=False, widths=widths)
    elif net == 'concat':
        m = models.MobileNetSkipConcat((224, 224), pretrained=False)
    else:
        m = models.MobileNet(net, (224, 224), pretrained=False)
    return fplan.describe(m)[0]


@pytest.mark.parametrize('net,want', [('stock', 1), ('nnconv5', 1), ('nnconv5dw', 1), ('pruned', 0), ('concat', 0)])
def test_eligibility_of_the_networks(lib, net, want):
    d = _descs(net)
    for dtype in (torch.float16, torch.bfloat16):
        q = front(lib, d, 64, 224, 224, dtype)
        assert q['ok'] == want, (net, dtype)
        assert q['items'] == (64 * 7 * 7 if want else 0)
    assert front(lib, d, 64, 224, 224, torch.float32)['ok'] == 0
    if want:
        assert front(lib, d, 16, 480, 640)['items'] == 16 * 15 * 20
        assert front(lib, d, 1, 32, 32)['items'] == 1


def test_other_widths_and_acts_fall_back(lib):
    base = ks.enc_dec((32, 64, 128, 128, 256, 32))
    assert front(lib, base, 2, 64, 96)['ok'] == 1
    assert front(lib, ks.enc_dec((32, 64, 128, 128, 256, 32), acts=(ks.R6, ks.R, ks.R, ks.R6, ks.R6, ks.R, ks.R, ks.R)), 2, 64, 96)['ok'] == 1
    for c in ((32, 64, 136, 128, 256, 32), (32, 72, 128, 128, 256, 32), (24, 64, 128, 128, 256, 32)):
        assert front(lib, ks.enc_dec(c), 2, 64, 96)['ok'] == 0, c
    mixed = ks.enc_dec((32, 64, 128, 128, 256, 32), acts=(ks.R6, ks.R, ks.R6, ks.R6, ks.R6, ks.R, ks.R, ks.R))
    assert front(lib, mixed, 2, 64, 96)['ok'] == 0           # one act for both blocks
    stem_relu = ks.enc_dec((32, 64, 128, 128, 256, 32), acts=(ks.R, ks.R6, ks.R6, ks.R6, ks.R6, ks.R, ks.R, ks.R))
    assert front(lib, stem_relu, 2, 64, 96)['ok'] == 0        # the stem kernel is ReLU6 only


@pytest.mark.parametrize('case', list(ks.CASES))
def test_every_sweep_topology_falls_back(lib, case):
    c = ks.CASES[case]
    assert front(lib, c['descs'](), c['n'], c['h'], c['w'], c['dtype'] if c['dtype'] in DT else torch.float16)['ok'] == 0


def test_budget_fits_two_ctas_per_sm(lib):
    q = front(lib, _descs('stock'), 64, 224, 224)
    assert q['ctas_per_sm'] == 2 and q['threads'] == 256
    assert q['smem_bytes'] <= 227 * 1024
    assert q['ctas_per_sm'] * (q['smem_bytes'] + CTA_RESERVED) <= SM_SMEM
    # weights 224 rows x 128 B + parameters; A: 320 rows x 128 B; tiles: T1 = 289 px x 128 B (T0 + x box and the 16 KB
    # conv2 staging fit inside it)
    assert q['param_bytes'] >= 224 * 128 and q['a_bytes'] == 320 * 128 and q['tile_bytes'] >= 289 * 128
    assert q['param_bytes'] + q['a_bytes'] + q['tile_bytes'] + 1024 <= q['smem_bytes']
