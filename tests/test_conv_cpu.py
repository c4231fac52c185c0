"""CPU tests of the dense conv stage: the planner (through fd_debug_conv_plan), describe() / supports() / routing of
MobileNet('nnconv5' / 'nnconv3'), the three dense-decoder references against the reference's goldens, and the interval
CONV reference against the storage-emulated forward."""
import ctypes
import os

import numpy as np
import pytest
import torch

import dense_ref as dr
from conftest import GOLDEN, rel_err
from fastdepth_b200 import _lib, plan, synthetic
from oracle import stage_ref as sr

NNCONV5 = ((1024, 512), (512, 256), (256, 128), (128, 64), (64, 32))


def conv_plan(k, h, w, n, ci, co, sms=132):
    out = (ctypes.c_int * 16)()
    _lib.check(_lib.load().fd_debug_conv_plan(k, h, w, n, ci, co, sms, out, 16))
    keys = ('ok', 'ni', 'th', 'tw', 'bn', 'stages', 'm_tiles', 'n_splits', 'items', 'waves', 'kblocks', 'smem_bytes',
            'useful_permille', 'cost')
    return dict(zip(keys, out[:14]))


@pytest.mark.parametrize('hw', [(224, 224), (480, 640), (64, 96)], ids=['224', '480x640', '64x96'])
def test_conv_planner_covers_every_nnconv5_stage(built_lib, hw):
    for n in (1, 2, 3, 7, 16, 33, 64):
        h, w = hw[0] // 32, hw[1] // 32
        for ci, co in NNCONV5:
            q = conv_plan(5, h, w, n, ci, co)
            assert q['ok'] == 1, (hw, n, ci, co, q)
            assert q['ni'] * q['th'] * q['tw'] == 128
            assert q['bn'] in (64, 128, 256) and 2 <= q['stages'] <= 8
            assert q['smem_bytes'] <= 227 * 1024
            # the tiles cover every output pixel and every output channel
            tiles = -(-n // q['ni']) * -(-h // q['th']) * -(-w // q['tw'])
            assert q['m_tiles'] == tiles and q['n_splits'] * q['bn'] >= co
            assert q['items'] == tiles * q['n_splits'] and q['waves'] == -(-q['items'] // 132)
            assert q['kblocks'] * 64 >= ci
            assert q['useful_permille'] == int(1000 * n * h * w / (tiles * 128))
            h, w = 2 * h, 2 * w


def test_conv_planner_wave_and_waste_choices(built_lib):
    # stage 1 at b64 224^2: 3136 pixels on a 7x7 map; 2-image 8x8 boxes waste a quarter of the rows but one wave of bn 128
    # items beats half a machine of bn 256 items
    q = conv_plan(5, 7, 7, 64, 1024, 512)
    assert q['waves'] == 1 and q['items'] >= 100, q
    # a 1x2 map of one image: the smallest box shape
    q = conv_plan(3, 1, 2, 1, 64, 64)
    assert q['ok'] and q['ni'] * q['th'] * q['tw'] == 128
    assert conv_plan(5, 7, 7, 64, 4, 512)['ok'] == 0          # c_in < 8 is not a conv stage


def test_describe_dense_decoders():
    import models
    for k in (5, 3):
        m = models.MobileNet('nnconv%d' % k, (224, 224), pretrained=False).eval()
        assert plan.supports(m) and plan.dense_decoder(m)
        descs, wts, names = plan.describe(m)
        conv = descs[14:19]
        assert [d['kind'] for d in conv] == [_lib.FD_STAGE_CONV] * 5
        assert [(d['c_in'], d['c_out']) for d in conv] == list(NNCONV5)
        assert all(d['ksize'] == k and d['upsample'] == 1 and d['skip_src'] == -1 and d['stride'] == 1 for d in conv)
        for j, (d, wt) in enumerate(zip(conv, wts[14:19]), start=1):
            blk = getattr(m.decoder, 'conv%d' % j)
            assert wt[:3] == (None, None, None)
            assert wt[3].shape == (d['c_out'], d['c_in'] * k * k)
            np.testing.assert_array_equal(wt[3], blk[0].weight.detach().numpy().reshape(d['c_out'], -1))
            s, b = plan.fold_bn(blk[1])
            np.testing.assert_array_equal(wt[4], s)
            np.testing.assert_array_equal(wt[5], b)
        assert descs[-1]['kind'] == _lib.FD_STAGE_HEAD and descs[-1]['c_in'] == 32


def test_supports_and_routing_truth_table():
    import models
    dense = models.MobileNet('nnconv5', (224, 224), pretrained=False).eval()
    dw = models.MobileNet('nnconv5dw', (224, 224), pretrained=False).eval()
    assert plan.supports(dense) and plan.dense_decoder(dense)
    assert plan.supports(dw) and not plan.dense_decoder(dw)
    # a 7x7 decoder conv is not a kernel target
    odd = models.MobileNet('nnconv5', (224, 224), pretrained=False).eval()
    odd.decoder.conv2[0] = torch.nn.Conv2d(512, 256, 7, padding=3, bias=False)
    assert not plan.supports(odd)
    # CPU tensors stay on stock PyTorch whatever the dtype (no engine is built)
    with torch.no_grad():
        assert dense(torch.rand(1, 3, 64, 64)).shape == (1, 1, 64, 64)
    assert '_fd_engine' not in dense.__dict__


def test_dense_oracles_match_reference_goldens(built_lib):
    for name in ('nnconv5_stock_2x64x96', 'nnconv5_stock_1x224x224'):
        fx = np.load(os.path.join(GOLDEN, name + '.npz'))
        n, h, w = (int(v) for v in fx['shape'])
        sd = synthetic.synthetic_nnconv_state_dict(int(fx['kernel_size']), seed=int(fx['wseed']))
        x = synthetic.synthetic_input(n, h, w, seed=int(fx['xseed']))
        want = torch.from_numpy(fx['output'])
        assert rel_err(dr.torch_forward(sd, x), want) < 1e-4, name
        assert rel_err(torch.from_numpy(dr.c_forward(sd, x)), want) < 1e-4, name


def test_synthetic_dense_recipe_is_conditioned():
    """fp16 storage noise reaches the output at a few 1e-3, so the 1e-2 fp16 tolerance is meaningful."""
    sd = synthetic.synthetic_nnconv_state_dict(5, seed=1)
    x = synthetic.synthetic_input(2, 64, 96, seed=0)
    ref = dr.torch_forward(sd, x)
    assert (ref == 0).float().mean() < 0.05
    assert rel_err(dr.torch_forward(sd, x, storage=torch.float16), ref) < 5e-3
    assert rel_err(dr.torch_forward(sd, x, storage=torch.bfloat16), ref) < 5e-2
    again = synthetic.synthetic_nnconv_state_dict(5, seed=1)
    assert all(torch.equal(sd[k], again[k]) for k in sd)


def _dense_stage_list(k=5, n=1, h=64, w=96):
    import models
    m = models.MobileNet('nnconv%d' % k, (h, w), pretrained=False)
    m.load_state_dict(synthetic.synthetic_nnconv_state_dict(k, seed=2)) if k == 5 else None
    return plan.describe(m.eval())


@pytest.mark.parametrize('dtype', [torch.float16, torch.bfloat16])
def test_conv_interval_contains_storage_emulated_stages(dtype):
    """Stage by stage from the emulated forward's own rounded inputs: every element of the storage-emulated dense conv
    (fp32 arithmetic, rounded once) lies inside the CONV interval, and most are determined."""
    import torch.nn.functional as F
    descs, wts, _ = _dense_stage_list()
    rng = np.random.Generator(np.random.PCG64(11))
    for d, wt in zip(descs[14:19], wts[14:19]):
        h = 2 if d['c_in'] == 1024 else {512: 4, 256: 8, 128: 16, 64: 32}[d['c_in']]
        x = torch.from_numpy(rng.random((1, d['c_in'], h, 3 * h // 2 or 1), dtype=np.float32)).to(dtype).float()
        wq = torch.from_numpy(wt[3]).to(dtype).float().reshape(d['c_out'], d['c_in'], 5, 5)
        y = F.conv2d(x, wq, None, 1, 2) * torch.from_numpy(wt[4]).view(1, -1, 1, 1) + torch.from_numpy(wt[5]).view(1, -1, 1, 1)
        y = y.clamp_min(0).to(dtype).float().permute(0, 2, 3, 1)
        iv = sr.quantize(dr.conv(sr.exact(x.permute(0, 2, 3, 1)), wq.numpy(), wt[4], wt[5], 5, d['act']), dtype)
        det = sr.check(y, iv, dtype, str(d))
        assert det > 0.5, (d, det)
        # a swapped pair of taps is caught
        wbad = wq.clone()
        wbad[:, :, [0, 1]] = wbad[:, :, [1, 0]]
        ybad = (F.conv2d(x, wbad, None, 1, 2) * torch.from_numpy(wt[4]).view(1, -1, 1, 1) +
                torch.from_numpy(wt[5]).view(1, -1, 1, 1)).clamp_min(0).to(dtype).float().permute(0, 2, 3, 1)
        with pytest.raises(AssertionError):
            sr.check(ybad, iv, dtype, 'taps swapped')


def test_conv_interval_composition_fp64():
    """Without rounding the interval forward collapses to the fp64 forward of the same stage list (radius 0)."""
    descs, wts, _ = _dense_stage_list(n=1, h=64, w=96)
    x = synthetic.synthetic_input(1, 64, 96, seed=0)
    iv = dr.forward(descs, wts, x.double().numpy(), dtype=None)
    assert np.all(iv.r == 0)
    sd = synthetic.synthetic_nnconv_state_dict(5, seed=2)
    want = dr.torch_forward({k: v.double() if v.is_floating_point() else v for k, v in sd.items()}, x.double())
    # describe() folds BatchNorm in fp32 (plan.fold_bn), the PyTorch restatement in fp64: ~1e-6 relative apart
    assert np.abs(iv.c - want.numpy()).max() < 1e-5 * max(1.0, np.abs(want.numpy()).max())
