"""Helpers of the in_channels tests (MobileNet with 1 to 7 input channels: depth only, RGB-D).

* ``stem``: the fp64 interval stem of ``oracle.stage_ref`` for any number of input planes, read from the weight shape;
  at 3 planes it is the same computation, term for term;
* ``state_dict`` / ``model``: the seeded, BN-calibrated synthetic weights of ``MobileNet(decoder, in_channels=k)``;
* ``torch_forward``: that network's forward in fp32 arithmetic, optionally with the product's 16-bit storage roundings
  (used to measure the conditioning of each golden).
"""
import numpy as np
import torch
import torch.nn.functional as F

import convt_ref as cr
import dense_ref as dr
from fastdepth_b200 import synthetic
from oracle import stage_ref as sr

# golden name -> (decoder, in_channels, n, h, w)
GOLDENS = {
    'nnconv5dw_cin4_2x64x96': ('nnconv5dw', 4, 2, 64, 96),
    'nnconv5dw_cin4_1x224x224': ('nnconv5dw', 4, 1, 224, 224),
    'nnconv5dw_cin1_2x64x96': ('nnconv5dw', 1, 2, 64, 96),
    'upconv5_cin4_2x64x96': ('upconv', 4, 2, 64, 96),
}


def stem(x_nchw, w, scale, bias, stride, a, eps=sr.EPS):
    """Dense 3x3 stride-s conv (padding 1) of the exact NCHW input x over its c_in planes (c_in from ``w``: [c_out][c_in]
    [3][3] or flattened [c_out][9 c_in]), + folded BN + act; NHWC, before rounding."""
    x = np.asarray(x_nchw, np.float64).transpose(0, 2, 3, 1)
    c_in = x.shape[3]
    w = np.asarray(w, np.float64).reshape(-1, c_in, 3, 3)           # [co][ci][ky][kx]
    n, h, wd, _ = x.shape
    ho, wo = (h - 1) // stride + 1, (wd - 1) // stride + 1
    xp = np.pad(x, ((0, 0), (1, 1), (1, 1), (0, 0)))
    c = np.zeros((n, ho, wo, w.shape[0])); m = np.zeros_like(c)
    for ky in range(3):
        for kx in range(3):
            patch = xp[:, ky:ky + stride * (ho - 1) + 1:stride, kx:kx + stride * (wo - 1) + 1:stride, :]
            wk = w[:, :, ky, kx].T                                  # [ci][co]
            c += patch @ wk
            m += np.abs(patch) @ np.abs(wk)
    return sr.act(sr._affine(c, m, 0.0, scale, bias, eps), a)


def state_dict(decoder, in_channels, seed=1):
    """``models.MobileNet(decoder, in_channels=in_channels)`` schema: ``nnconv5dw`` or ``upconv``."""
    if decoder == 'nnconv5dw':
        return synthetic.to_mobilenet_keys(synthetic.synthetic_state_dict(synthetic.STOCK_WIDTHS, seed=seed,
                                                                          in_channels=in_channels))
    return synthetic.synthetic_convt_state_dict(decoder, seed=seed, in_channels=in_channels)


def model(decoder, in_channels, hw=(224, 224), seed=1):
    import models
    m = models.MobileNet(decoder, hw, in_channels=in_channels, pretrained=False)
    m.load_state_dict(state_dict(decoder, in_channels, seed))
    return m.eval()


def golden_input(name):
    decoder, c, n, h, w = GOLDENS[name]
    return synthetic.synthetic_input(n, h, w, seed=0, channels=c)


def torch_forward(sd, x, decoder, storage=None):
    """fp32 forward of ``MobileNet(decoder)`` on its state_dict (any stem c_in); ``storage``: every tensor the product
    keeps in 16 bits (x, the stem output, each depthwise and pointwise result, the head) rounded to that dtype."""
    if decoder != 'nnconv5dw':
        return cr.torch_forward(sd, x, decoder, storage=storage)

    def q(t):
        return t if storage is None else t.to(storage).float()
    sd = {k: (q(v) if v.is_floating_point() else v) for k, v in sd.items()}
    x = q(x.float())
    x = q(dr._bn(F.conv2d(x, sd['mobilenet.0.0.weight'], None, 2, 1), sd, 'mobilenet.0.1', 6.0))
    for i in range(1, 14):
        w = sd['mobilenet.%d.0.weight' % i]
        x = q(dr._bn(F.conv2d(x, w, None, dr.ENCODER_STRIDES[i], 1, 1, w.shape[0]), sd, 'mobilenet.%d.1' % i, 6.0))
        x = q(dr._bn(F.conv2d(x, sd['mobilenet.%d.3.weight' % i]), sd, 'mobilenet.%d.4' % i, 6.0))
    for j in range(1, 6):
        w = sd['decoder.conv%d.0.0.weight' % j]
        x = q(dr._bn(F.conv2d(x, w, None, 1, 2, 1, w.shape[0]), sd, 'decoder.conv%d.0.1' % j, None))
        x = q(dr._bn(F.conv2d(x, sd['decoder.conv%d.1.0.weight' % j]), sd, 'decoder.conv%d.1.1' % j, None))
        x = x.repeat_interleave(2, dim=2).repeat_interleave(2, dim=3)
    return q(dr._bn(F.conv2d(x, sd['decoder.conv6.0.weight']), sd, 'decoder.conv6.1', None))


def conditioning(name):
    """max relative error (tests/conftest.rel_err) of the storage-emulated forward against the fp32 forward, per dtype."""
    decoder, c, n, h, w = GOLDENS[name]
    sd = state_dict(decoder, c)
    x = golden_input(name)
    with torch.no_grad():
        ref = torch_forward(sd, x, decoder)
        out = {}
        for dt in (torch.float16, torch.bfloat16):
            got = torch_forward(sd, x, decoder, storage=dt).double()
            want = ref.double()
            denom = torch.maximum(want.abs(), want.abs().mean())
            out[str(dt).replace('torch.', '')] = ((got - want).abs() / denom).max().item()
    return out
