"""CPU tests of the DECONV / UPCONV stages: the four-phase algebra for every k, the planner's phase tables and grouping
(through fd_debug_convt_plan), the model surface (models.MobileNet('deconv<k>' / 'upconv'), state_dict schema, pickles,
describe / supports), the three references against the reference's goldens, and the interval stage against the
storage-emulated stage."""
import ctypes
import io
import os
import pickle

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import convt_ref as cr
from conftest import GOLDEN, rel_err
from fastdepth_b200 import _lib, plan, synthetic
from oracle import stage_ref as sr

STAGES = ((1024, 512), (512, 256), (256, 128), (128, 64), (64, 32))
KINDS = [(cr.DECONV, 3), (cr.DECONV, 5), (cr.DECONV, 7), (cr.DECONV, 9), (cr.UPCONV, 5)]
KIDS = ['deconv3', 'deconv5', 'deconv7', 'deconv9', 'upconv5']
GOLDENS = ['%s_stock_2x64x96' % d for d in ('upconv5', 'deconv3', 'deconv5', 'deconv7', 'deconv9')] + \
    ['upconv5_stock_1x224x224', 'deconv5_stock_1x224x224']


def _decoder_of(tag):
    return 'upconv' if tag.startswith('upconv') else tag


# ------------------------------------------------------------------------------------------------ phase algebra
@pytest.mark.parametrize('kind,k', KINDS, ids=KIDS)
def test_phase_algebra_matches_pytorch(kind, k):
    g = torch.Generator().manual_seed(k + 10 * kind)
    x = torch.randn(2, 5, 7, 6, dtype=torch.float64, generator=g)
    if kind == cr.DECONV:
        w = torch.randn(5, 3, k, k, dtype=torch.float64, generator=g)
        want = F.conv_transpose2d(x, w, None, 2, (k - 1) // 2, 1)
    else:
        w = torch.randn(3, 5, k, k, dtype=torch.float64, generator=g)
        want = F.conv2d(cr.unpool(x), w, None, 1, (k - 1) // 2)
    got = cr.phase_forward(kind, x, w)
    assert got.shape == want.shape == (2, 3, 14, 12)
    assert (got - want).abs().max().item() <= 2e-14 * want.abs().max().item()


def test_phase_table():
    """The per-axis (d, t) lists; the four phases partition the k*k taps and every offset stays in [-2, 2]."""
    want = {(cr.DECONV, 3): ([(0, 1)], [(0, 2), (1, 0)]),
            (cr.DECONV, 5): ([(-1, 4), (0, 2), (1, 0)], [(0, 3), (1, 1)]),
            (cr.DECONV, 7): ([(-1, 5), (0, 3), (1, 1)], [(-1, 6), (0, 4), (1, 2), (2, 0)]),
            (cr.DECONV, 9): ([(-2, 8), (-1, 6), (0, 4), (1, 2), (2, 0)], [(-1, 7), (0, 5), (1, 3), (2, 1)]),
            (cr.UPCONV, 5): ([(-1, 0), (0, 2), (1, 4)], [(0, 1), (1, 3)])}
    for (kind, k), (r0, r1) in want.items():
        assert cr.phase_taps(kind, k, 0) == r0 and cr.phase_taps(kind, k, 1) == r1
        assert sorted(t for _, t in r0 + r1) == list(range(k))
        assert all(-2 <= d <= 2 for d, _ in r0 + r1)


# ------------------------------------------------------------------------------------------------ planner
def convt_plan(kind, k, h, w, n, ci, co, sms=132):
    out = (ctypes.c_int * 44)()
    _lib.check(_lib.load().fd_debug_convt_plan(kind, k, h, w, n, ci, co, sms, out, 44))
    keys = ('ok', 'ni', 'th', 'tw', 'bn', 'stages', 'm_tiles', 'n_splits', 'items', 'waves', 'kblocks', 'smem_bytes',
            'useful_permille', 'cost', 'groups')
    q = dict(zip(keys, out[:15]))
    q['phases'] = [tuple(out[16 + 5 * i:21 + 5 * i]) for i in range(4)]
    q['group_ph'] = [tuple(out[36 + 2 * g:38 + 2 * g]) for g in range(4)]
    return q


@pytest.mark.parametrize('kind,k', KINDS, ids=KIDS)
def test_convt_planner(built_lib, kind, k):
    for n, (h, w) in ((64, (7, 7)), (1, (2, 3)), (3, (1, 1)), (2, (1, 2)), (16, (15, 20))):
        for ci, co in STAGES:
            q = convt_plan(kind, k, h, w, n, ci, co)
            assert q['ok'] == 1, (n, h, w, ci, co, q)
            assert q['ni'] * q['th'] * q['tw'] == 128 and q['bn'] in (64, 128, 256)
            assert q['smem_bytes'] <= 227 * 1024 and 2 <= q['stages'] <= 8
            assert q['m_tiles'] == -(-n // q['ni']) * -(-h // q['th']) * -(-w // q['tw'])
            assert q['n_splits'] * q['bn'] >= co and q['kblocks'] * 64 >= ci
            # the phase table: contiguous phase-major taps, offsets and taps as the algebra says
            taps = 0
            for ph, (tap0, ny, nx, dy0, dx0) in enumerate(q['phases']):
                ys, xs = cr.phase_taps(kind, k, ph >> 1), cr.phase_taps(kind, k, ph & 1)
                assert (tap0, ny, nx, dy0, dx0) == (taps, len(ys), len(xs), ys[0][0], xs[0][0])
                assert [d for d, _ in ys] == list(range(dy0, dy0 + ny)) and [d for d, _ in xs] == list(range(dx0, dx0 + nx))
                taps += ny * nx
            assert taps == k * k
            # every phase in exactly one group; items x taps = k^2 kblocks m_tiles n_splits
            groups = [tuple(p for p in g if p >= 0) for g in q['group_ph'][:q['groups']]]
            assert q['groups'] in (2, 4) and sorted(sum(groups, ())) == [0, 1, 2, 3]
            assert all(g == (-1, -1) for g in q['group_ph'][q['groups']:])
            assert q['items'] == q['m_tiles'] * q['n_splits'] * q['groups']
            per = q['m_tiles'] * q['n_splits']
            item_taps = sum(per * sum(q['phases'][p][1] * q['phases'][p][2] for p in g) for g in groups)
            assert item_taps * q['kblocks'] == k * k * q['kblocks'] * q['m_tiles'] * q['n_splits']
            if q['groups'] == 2:
                assert sorted(groups) == [(0, 3), (1, 2)]
            else:                                           # one phase per item, the heaviest first
                cost = [q['phases'][g[0]][1] * q['phases'][g[0]][2] for g in groups]
                assert cost == sorted(cost, reverse=True)


def test_convt_planner_rejects():
    assert convt_plan(cr.DECONV, 4, 7, 7, 1, 64, 64)['ok'] == 0
    assert convt_plan(cr.DECONV, 5, 7, 7, 1, 4, 64)['ok'] == 0
    out = (ctypes.c_int * 44)()
    with pytest.raises(RuntimeError):
        _lib.check(_lib.load().fd_debug_convt_plan(3, 5, 7, 7, 1, 64, 64, 132, out, 44))      # CONV is not phased
    with pytest.raises(RuntimeError):
        _lib.check(_lib.load().fd_debug_convt_plan(cr.DECONV, 5, 7, 7, 1, 64, 64, 132, out, 16))


# ------------------------------------------------------------------------------------------------ model surface
def test_choose_decoder():
    import models
    for d in ('deconv3', 'deconv5', 'deconv7', 'deconv9'):
        m = models.choose_decoder(d)
        assert isinstance(m, models.DeConv) and m.convt1[0].kernel_size == (int(d[6]),) * 2
    assert isinstance(models.choose_decoder('upconv'), models.UpConv)
    for d in ('deconv5dw', 'deconv3dw', 'upproj', 'blconv5', 'shuffle5', 'blconv3dw'):
        with pytest.raises(NotImplementedError):
            models.choose_decoder(d)
    with pytest.raises(AssertionError):
        models.choose_decoder('bogus')


@pytest.mark.parametrize('name', GOLDENS[:5])
def test_state_dict_schema_matches_reference(name):
    """Keys and shapes of models.MobileNet(decoder).state_dict() are the reference module's, recorded in the golden."""
    import models
    fx = np.load(os.path.join(GOLDEN, name + '.npz'))
    m = models.MobileNet(str(fx['decoder']), (224, 224), pretrained=False)
    sd = m.state_dict()
    assert sorted(sd.keys()) == list(fx['state_dict_keys'])
    assert [','.join(str(d) for d in sd[k].shape) for k in fx['state_dict_keys']] == list(fx['state_dict_shapes'])
    m.load_state_dict(synthetic.synthetic_convt_state_dict(str(fx['decoder']), seed=1), strict=True)


def test_pickle_round_trip_and_unpool_mask():
    import models
    m = models.MobileNet('upconv', (224, 224), pretrained=False).eval()
    m.load_state_dict(synthetic.synthetic_convt_state_dict('upconv', seed=1))
    u = m.decoder.upconv1[0]
    assert isinstance(u, models.Unpool) and 'mask' in u.__dict__ and torch.equal(u.mask, torch.tensor([[[[1., 0.], [0., 0.]]]]))
    assert not any('mask' in k for k in m.state_dict())
    buf = io.BytesIO()
    torch.save(m, buf)
    buf.seek(0)
    m2 = torch.load(buf, weights_only=False)
    x = synthetic.synthetic_input(1, 64, 64, seed=0)
    with torch.no_grad():
        assert torch.equal(m(x), m2(x))
    # an Unpool restored from a pickle carries only the reference's attributes (stride, mask) and still runs
    u2 = pickle.loads(pickle.dumps(u))
    assert u2.stride == 2 and torch.equal(u2(torch.ones(1, 1, 1, 2)), torch.tensor([[[[1., 0., 1., 0.], [0., 0., 0., 0.]]]]))


@pytest.mark.parametrize('decoder', cr.DECODERS)
def test_describe_convt_decoders(decoder):
    import models
    m = models.MobileNet(decoder, (224, 224), pretrained=False).eval()
    assert plan.supports(m) and plan.dense_decoder(m)
    descs, wts, names = plan.describe(m)
    kind = _lib.FD_STAGE_UPCONV if decoder == 'upconv' else _lib.FD_STAGE_DECONV
    k = 5 if decoder == 'upconv' else int(decoder[6])
    dec = descs[14:19]
    assert [d['kind'] for d in dec] == [kind] * 5
    assert [(d['c_in'], d['c_out']) for d in dec] == list(STAGES)
    assert all(d['ksize'] == k and d['stride'] == 2 and d['upsample'] == 0 and d['skip_src'] == -1 for d in dec)
    child = 'upconv' if decoder == 'upconv' else 'convt'
    assert names[14:] == ['decoder.%s%d' % (child, j) for j in range(1, 6)] + ['decoder.convf']
    for j, wt in enumerate(wts[14:19], start=1):
        blk = getattr(m.decoder, '%s%d' % (child, j))
        conv, bn = (blk[1], blk[2]) if decoder == 'upconv' else (blk[0], blk[1])
        np.testing.assert_array_equal(wt[3].reshape(conv.weight.shape), conv.weight.detach().numpy())
        s, b = plan.fold_bn(bn)
        np.testing.assert_array_equal(wt[4], s)
        np.testing.assert_array_equal(wt[5], b)
    assert descs[-1]['kind'] == _lib.FD_STAGE_HEAD and descs[-1]['c_in'] == 32


def test_supports_rejects_other_transposed_convs():
    import models
    m = models.MobileNet('deconv5', (224, 224), pretrained=False).eval()
    m.decoder.convt2[0] = torch.nn.ConvTranspose2d(512, 256, 5, 2, 2, 1, bias=False, dilation=1, groups=2)
    assert not plan.supports(m)
    m = models.MobileNet('upconv', (224, 224), pretrained=False).eval()
    m.decoder.upconv3[1] = torch.nn.Conv2d(256, 128, 3, 1, 1, bias=False)
    assert not plan.supports(m)
    with torch.no_grad():                               # CPU tensors stay on stock PyTorch
        assert m(torch.rand(1, 3, 64, 64)).shape == (1, 1, 64, 64)
    assert '_fd_engine' not in m.__dict__


# ------------------------------------------------------------------------------------------------ references vs goldens
@pytest.mark.parametrize('name', GOLDENS)
def test_convt_oracles_match_reference_goldens(built_lib, name):
    fx = np.load(os.path.join(GOLDEN, name + '.npz'))
    n, h, w = (int(v) for v in fx['shape'])
    dec = str(fx['decoder'])
    sd = synthetic.synthetic_convt_state_dict(dec, seed=int(fx['wseed']))
    x = synthetic.synthetic_input(n, h, w, seed=int(fx['xseed']))
    want = torch.from_numpy(fx['output'])
    assert rel_err(cr.torch_forward(sd, x, dec), want) < 1e-4
    assert rel_err(torch.from_numpy(cr.c_forward(sd, x, dec)), want) < 1e-4


def test_synthetic_convt_recipe():
    """Seeded, and the 16-bit storage noise on the small golden stays within the end-to-end tolerances."""
    for dec in cr.DECODERS:
        sd = synthetic.synthetic_convt_state_dict(dec, seed=1)
        again = synthetic.synthetic_convt_state_dict(dec, seed=1)
        assert all(torch.equal(sd[k], again[k]) for k in sd)
        x = synthetic.synthetic_input(2, 64, 96, seed=0)
        ref = cr.torch_forward(sd, x, dec)
        assert (ref == 0).float().mean() < 0.05
        assert rel_err(cr.torch_forward(sd, x, dec, storage=torch.float16), ref) < 5e-3, dec
        assert rel_err(cr.torch_forward(sd, x, dec, storage=torch.bfloat16), ref) < 5e-2, dec


# ------------------------------------------------------------------------------------------------ interval stage
@pytest.mark.parametrize('kind,k', KINDS, ids=KIDS)
@pytest.mark.parametrize('dtype', [torch.float16, torch.bfloat16])
def test_convt_interval_contains_storage_emulated_stage(kind, k, dtype):
    rng = np.random.Generator(np.random.PCG64(k + kind))
    for ci, co, h, w in ((1024, 64, 2, 3), (64, 32, 9, 7)):
        x = torch.from_numpy(rng.random((1, ci, h, w), dtype=np.float32)).to(dtype).float()
        shape = (ci, co, k, k) if kind == cr.DECONV else (co, ci, k, k)
        wq = torch.from_numpy(rng.uniform(-1, 1, shape).astype(np.float32) / np.sqrt(ci * k * k / 4)).to(dtype).float()
        s, b = rng.uniform(0.5, 1.5, co).astype(np.float32), rng.normal(0.2, 0.3, co).astype(np.float32)
        y = cr.phase_forward(kind, x, wq) * torch.from_numpy(s).view(1, -1, 1, 1) + torch.from_numpy(b).view(1, -1, 1, 1)
        y = y.clamp_min(0).to(dtype).float().permute(0, 2, 3, 1)
        iv = sr.quantize(cr.convt(sr.exact(x.permute(0, 2, 3, 1)), wq.numpy(), s, b, kind, k, sr.RELU), dtype)
        assert sr.check(y, iv, dtype, 'k%d %s' % (k, dtype)) > 0.5
        # one phase's output written to its neighbour's parity is caught
        bad = y.clone()
        bad[:, 0::2, 0::2], bad[:, 0::2, 1::2] = y[:, 0::2, 1::2], y[:, 0::2, 0::2]
        with pytest.raises(AssertionError):
            sr.check(bad, iv, dtype, 'phases swapped')
