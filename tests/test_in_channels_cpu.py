"""MobileNet with 1 to 7 input channels (depth only, RGB-D), without a GPU.

* our ``models.MobileNet(decoder, in_channels=k)`` on the CPU against the reference's, recorded in the goldens (made by
  tests/golden/make_golden_in_channels.py; storage-emulated conditioning in DESIGN.md section 3.1);
* ``plan.describe`` hands the stem's c_in to the C-ABI, which takes 1..7 and refuses 0 (FD_ERR_INVALID) and 8
  (FD_ERR_UNSUPPORTED);
* the front route and its shared-memory budget for every c_in (``fd_debug_front_plan``);
* the interval stem for any c_in against an fp64 ``F.conv2d``, and against ``oracle.stage_ref.stem`` at 3 planes;
* the synthetic weights and inputs: 3 channels unchanged, other counts an image plus a sparse depth channel.
"""
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import in_channels_ref as icr
import test_kernel_sweep as ks
from conftest import GOLDEN, rel_err
from fastdepth_b200 import _lib
from fastdepth_b200 import plan as fplan
from fastdepth_b200 import synthetic
from oracle import stage_ref as sr

FD_ERR_INVALID, FD_ERR_UNSUPPORTED = -1, -4
SM_SMEM, CTA_RESERVED = 228 * 1024, 1024
KEYS = ('ok', 'items', 'smem_bytes', 'ctas_per_sm', 'threads', 'param_bytes', 'a_bytes', 'tile_bytes')


@pytest.fixture(scope='module')
def lib():
    return _lib.load()


def _front(lib, descs, n=64, h=224, w=224, dtype=_lib.FD_F16):
    arr = (_lib.StageDesc * len(descs))(*[_lib.StageDesc(**d) for d in descs])
    out = (ctypes.c_int * 8)()
    rc = lib.fd_debug_front_plan(arr, len(descs), dtype, n, h, w, out, 8)
    return rc, dict(zip(KEYS, out))


def _descs(c_in, decoder='nnconv5dw'):
    import models
    return fplan.describe(models.MobileNet(decoder, (224, 224), in_channels=c_in, pretrained=False))[0]


@pytest.mark.parametrize('name', list(icr.GOLDENS))
def test_module_on_cpu_matches_the_reference(name):
    fx = np.load(os.path.join(GOLDEN, name + '.npz'))
    decoder, c, n, h, w = icr.GOLDENS[name]
    assert [int(v) for v in fx['shape']] == [n, h, w] and int(fx['in_channels']) == c and str(fx['decoder']) == decoder
    m = icr.model(decoder, c, (h, w))
    sd = m.state_dict()
    assert sorted(sd) == list(fx['state_dict_keys'])
    assert [','.join(str(d) for d in sd[k].shape) for k in sorted(sd)] == list(fx['state_dict_shapes'])
    x = icr.golden_input(name)
    assert x.shape == (n, c, h, w)
    with torch.no_grad():
        y = m(x)
    assert rel_err(y, torch.from_numpy(fx['output'])) <= 1e-5


@pytest.mark.parametrize('c_in', [1, 2, 4, 7])
def test_describe_gives_the_stem_its_c_in(c_in):
    for decoder in ('nnconv5dw', 'upconv', 'nnconv5'):
        d = _descs(c_in, decoder)
        assert d[0]['kind'] == _lib.FD_STAGE_STEM and d[0]['c_in'] == c_in and d[0]['c_out'] == 32
        assert d[1]['c_in'] == 32


def test_abi_accepts_c_in_1_to_7_and_refuses_0_and_8(lib):
    base = _descs(3)
    for c_in in range(1, 8):
        d = [dict(x) for x in base]
        d[0]['c_in'] = c_in
        rc, _ = _front(lib, d)
        assert rc == 0, (c_in, lib.fd_last_error())
    for c_in, want in ((0, FD_ERR_INVALID), (-1, FD_ERR_INVALID), (8, FD_ERR_UNSUPPORTED), (16, FD_ERR_UNSUPPORTED)):
        d = [dict(x) for x in base]
        d[0]['c_in'] = c_in
        rc, _ = _front(lib, d)
        assert rc == want, (c_in, rc)
        if want == FD_ERR_UNSUPPORTED:
            assert b'1..7' in lib.fd_last_error()


def test_front_route_and_budget_per_c_in(lib):
    """c_in <= 3: the parent layout (the x box beside the stem chunk inside conv1's A region); 4: the tiles move up 2688
    bytes and two CTAs still fit on an SM; 5..7: one CTA per SM, so the stem, conv1 and conv2 stay three steps."""
    _, stock = _front(lib, _descs(3))
    assert stock['ok'] == 1 and stock['ctas_per_sm'] == 2
    for c_in in range(1, 8):
        for dtype in (_lib.FD_F16, _lib.FD_BF16):
            rc, q = _front(lib, _descs(c_in), dtype=dtype)
            assert rc == 0
            assert q['ok'] == (1 if c_in <= 4 else 0), (c_in, q)
            assert q['items'] == (64 * 7 * 7 if c_in <= 4 else 0)
            x_box = c_in * 39 * 48 * 2
            if c_in <= 3:
                assert {k: q[k] for k in KEYS[2:]} == {k: stock[k] for k in KEYS[2:]}
            else:
                over = (x_box - 12288 + 127) // 128 * 128
                assert q['a_bytes'] == stock['a_bytes'] + over and q['smem_bytes'] == stock['smem_bytes'] + over
            assert q['a_bytes'] - 28672 >= x_box                       # the box sits 28672 bytes into the A region
            fits = SM_SMEM // (q['smem_bytes'] + CTA_RESERVED)
            assert q['ctas_per_sm'] == min(fits, 2)
            assert (q['ctas_per_sm'] == 2) == (c_in <= 4)
        assert _front(lib, _descs(c_in), dtype=_lib.FD_F32)[1]['ok'] == 0
    # the other conditions of the route still apply at any c_in
    pruned = ks.enc_dec((32, 64, 136, 128, 256, 32))
    pruned[0]['c_in'] = 4
    assert _front(lib, pruned, 2, 64, 96)[1]['ok'] == 0


@pytest.mark.parametrize('c_in', range(1, 8))
@pytest.mark.parametrize('stride', [1, 2])
def test_interval_stem_matches_fp64_conv(c_in, stride):
    rng = np.random.default_rng(c_in * 10 + stride)
    x = rng.uniform(-1, 1, (2, c_in, 10, 14))
    w = rng.standard_normal((24, c_in, 3, 3))
    s, b = rng.uniform(0.5, 1.5, 24), rng.normal(0, 0.1, 24)
    want = F.conv2d(torch.from_numpy(x), torch.from_numpy(w), None, stride, 1).numpy().transpose(0, 2, 3, 1) * s + b
    iv = icr.stem(x, w.reshape(24, -1), s, b, stride, None, eps=0)
    assert iv.c.shape == want.shape
    np.testing.assert_allclose(iv.c, want, rtol=1e-12, atol=1e-12)
    assert np.all(iv.r == 0)
    iv6 = icr.stem(x, w, s, b, stride, sr.RELU6)                 # with the fp32 allowance the interval holds the centre
    assert np.all(iv6.lo <= np.clip(want, 0, 6) + 1e-12) and np.all(iv6.hi >= np.clip(want, 0, 6) - 1e-12)
    if c_in == 3:
        ref = sr.stem(x, w, s, b, stride, sr.RELU6)
        assert np.array_equal(ref.c, iv6.c) and np.array_equal(ref.r, iv6.r)


def test_synthetic_three_channels_unchanged_and_sparse_depth():
    a = synthetic.synthetic_input(2, 32, 64, seed=5)
    b = synthetic.synthetic_input(2, 32, 64, seed=5, channels=3)
    assert torch.equal(a, b)
    rng = np.random.Generator(np.random.PCG64(5))
    assert torch.equal(a, torch.from_numpy(rng.random((2, 3, 32, 64), dtype=np.float32)))
    assert all(torch.equal(synthetic.synthetic_state_dict()[k], synthetic.synthetic_state_dict(in_channels=3)[k])
               for k in synthetic.synthetic_state_dict())
    x = synthetic.synthetic_input(4, 64, 96, seed=1, channels=4)
    assert x.shape == (4, 4, 64, 96) and x.dtype == torch.float32
    assert float(x[:, :3].min()) >= 0 and float(x[:, :3].max()) < 1
    d = x[:, 3]
    frac = float((d > 0).float().mean())
    assert 0.02 < frac < 0.1                                   # mostly zeros, like sparse samples
    assert float(d[d > 0].min()) >= synthetic.SPARSE_RANGE[0] and float(d.max()) <= synthetic.SPARSE_RANGE[1]
    one = synthetic.synthetic_input(1, 32, 32, channels=1)
    assert one.shape == (1, 1, 32, 32) and float((one > 0).float().mean()) < 0.1
    sd = synthetic.synthetic_state_dict(in_channels=4)
    assert sd['conv0.0.weight'].shape == (32, 4, 3, 3)


def test_engine_checks_the_channel_count_without_a_gpu():
    """The engine refuses an input whose channel count is not the stem's, with PyTorch's wording for a channel mismatch
    (checked before anything touches a device)."""
    from fastdepth_b200.engine import SkipAddEngine
    m = icr.model('nnconv5dw', 4, (64, 96))
    eng = SkipAddEngine(m)

    class FakeCuda:                                             # only the attributes the checks read
        is_cuda = True
        shape = (2, 3, 64, 96)
        dtype = torch.float32

        def dim(self):
            return 4
    with pytest.raises(RuntimeError, match=r'expected input\[2, 3, 64, 96\] to have 4 channels, but got 3 channels'):
        eng.plan_for(FakeCuda())
