"""Test helpers for the DeConv / UpConv decoders (``models.MobileNet('deconv<k>')`` / ``('upconv')``): three references
and the phase algebra the kernels use.

* ``phase_taps``: per axis and output parity r, the (input offset d, weight tap t) pairs of a DECONV / UPCONV stage;
* ``torch_forward``: the forward restated with PyTorch primitives (F.conv_transpose2d, zero insertion + F.conv2d), optionally
  with the product's storage roundings (``storage=dtype``);
* ``c_forward``: the same composed from the plain-C oracle's fo_conv_dense on the zero-inserted input (UpConv), or on the
  zero-inserted input padded by the conv with the transposed and flipped weights (DeConv);
* ``convt`` / ``forward``: the per-stage fp64 interval reference, ``dense_ref.conv`` applied the same way.  The inserted
  zeros add nothing to the interval radius, so ``dense_ref.EPS_CONV`` stands: the longest sum is one deconv9 phase of
  stage 1, 5 x 5 taps x 1024 channels = 25 600 terms, the length of an nnconv5 stage-1 sum.
"""
import numpy as np
import torch
import torch.nn.functional as F

import dense_ref as dr
from oracle import c_oracle
from oracle import stage_ref as sr

DECONV, UPCONV = 4, 5
DECODERS = ('upconv', 'deconv3', 'deconv5', 'deconv7', 'deconv9')


# ------------------------------------------------------------------------------------------------ phase algebra
def phase_taps(kind, k, r):
    """Output pixel o = 2 Y + r (one axis) reads input Y + d with weight tap t, p = (k - 1) / 2:
    DECONV t = r + p (mod 2), d = (r + p - t) / 2; UPCONV t = r + p (mod 2), d = (r + t - p) / 2.  Sorted by d."""
    p = (k - 1) // 2
    out = []
    for t in range(k):
        if (t - r - p) % 2:
            continue
        out.append(((r + p - t) // 2 if kind == DECONV else (r + t - p) // 2, t))
    return sorted(out)


def phase_forward(kind, x, w):
    """A DECONV / UPCONV stage (no BN) as its four phase convs, NCHW, any float dtype: the algebra under test."""
    n, _, h, wd = x.shape
    k = w.shape[-1]
    wc = w.transpose(0, 1) if kind == DECONV else w                   # [c_out][c_in][k][k]
    out = x.new_zeros(n, wc.shape[0], 2 * h, 2 * wd)
    xp = F.pad(x, (2, 2, 2, 2))                                          # every offset d lies in [-2, 2]
    for ry in (0, 1):
        for rx in (0, 1):
            acc = x.new_zeros(n, wc.shape[0], h, wd)
            for dy, ty in phase_taps(kind, k, ry):
                for dx, tx in phase_taps(kind, k, rx):
                    acc += torch.einsum('nchw,oc->nohw', xp[:, :, 2 + dy:2 + dy + h, 2 + dx:2 + dx + wd], wc[:, :, ty, tx])
            out[:, :, ry::2, rx::2] = acc
    return out


# ------------------------------------------------------------------------------------------------ PyTorch primitives
def unpool(x):
    """x2 zero insertion (reference Unpool): x at even (row, column), zeros elsewhere; NCHW."""
    n, c, h, w = x.shape
    out = x.new_zeros(n, c, 2 * h, 2 * w)
    out[:, :, ::2, ::2] = x
    return out


def _children(decoder):
    return ('upconv', 1, 2) if decoder == 'upconv' else ('convt', 0, 1)


def torch_forward(sd, x, decoder, storage=None):
    """``MobileNet(decoder)`` forward on a ``synthetic_convt_state_dict``-schema state_dict, fp32 arithmetic (``storage``:
    every tensor the product keeps in 16 bits rounded to that dtype, as ``dense_ref.torch_forward``)."""
    def q(t):
        return t if storage is None else t.to(storage).float()
    sd = {k: (q(v) if v.is_floating_point() else v) for k, v in sd.items()}
    x = q(x if x.dtype == torch.float64 else x.float())
    x = q(dr._bn(F.conv2d(x, sd['mobilenet.0.0.weight'], None, 2, 1), sd, 'mobilenet.0.1', 6.0))
    for i in range(1, 14):
        w = sd['mobilenet.%d.0.weight' % i]
        x = q(dr._bn(F.conv2d(x, w, None, dr.ENCODER_STRIDES[i], 1, 1, w.shape[0]), sd, 'mobilenet.%d.1' % i, 6.0))
        x = q(dr._bn(F.conv2d(x, sd['mobilenet.%d.3.weight' % i]), sd, 'mobilenet.%d.4' % i, 6.0))
    child, ci, bi = _children(decoder)
    for j in range(1, 6):
        w = sd['decoder.%s%d.%d.weight' % (child, j, ci)]
        k = w.shape[-1]
        y = F.conv_transpose2d(x, w, None, 2, (k - 1) // 2, 1) if child == 'convt' else F.conv2d(unpool(x), w, None, 1, 2)
        x = q(dr._bn(y, sd, 'decoder.%s%d.%d' % (child, j, bi), None))
    return q(dr._bn(F.conv2d(x, sd['decoder.convf.0.weight']), sd, 'decoder.convf.1', None))


# ------------------------------------------------------------------------------------------------ C oracle composition
def _np_unpool(x):
    n, c, h, w = x.shape
    out = np.zeros((n, c, 2 * h, 2 * w), np.float32)
    out[:, :, ::2, ::2] = x
    return out


def c_forward(sd, x, decoder):
    """The same forward from the plain-C primitives.  A transposed conv is fo_conv_dense (stride 1, pad p) of the zero-
    inserted input with the weights transposed to [c_out][c_in] and flipped in both axes; the zero row and column the
    insertion leaves at the bottom / right are the output_padding."""
    g = c_oracle._np
    x = g(x)
    x = c_oracle._bn_act(c_oracle._dense(x, g(sd['mobilenet.0.0.weight']), 2, 1), sd, 'mobilenet.0.1', 2)
    for i in range(1, 14):
        x = c_oracle._bn_act(c_oracle._depthwise(x, g(sd['mobilenet.%d.0.weight' % i]), dr.ENCODER_STRIDES[i]), sd,
                             'mobilenet.%d.1' % i, 2)
        x = c_oracle._bn_act(c_oracle._pointwise(x, g(sd['mobilenet.%d.3.weight' % i])), sd, 'mobilenet.%d.4' % i, 2)
    child, ci, bi = _children(decoder)
    for j in range(1, 6):
        w = g(sd['decoder.%s%d.%d.weight' % (child, j, ci)])
        if child == 'convt':
            w = np.ascontiguousarray(w.transpose(1, 0, 2, 3)[:, :, ::-1, ::-1])
        k = w.shape[-1]
        x = c_oracle._bn_act(c_oracle._dense(_np_unpool(x), w, 1, (k - 1) // 2), sd, 'decoder.%s%d.%d' % (child, j, bi), 1)
    return c_oracle._bn_act(c_oracle._pointwise(x, g(sd['decoder.convf.0.weight'])), sd, 'decoder.convf.1', 1)


# ------------------------------------------------------------------------------------------------ interval reference
def conv_weights(kind, w, c_in, c_out, k):
    """The stage's ``pw_w`` (DECONV [c_in][c_out][k][k], UPCONV [c_out][c_in][k][k], any flattening) as the [c_out][c_in]
    [k][k] weights of the equivalent stride-1 conv of the zero-inserted input."""
    w = np.asarray(w, np.float64)
    if kind == DECONV:
        return np.ascontiguousarray(w.reshape(c_in, c_out, k, k).transpose(1, 0, 2, 3)[:, :, ::-1, ::-1])
    return w.reshape(c_out, c_in, k, k)


def convt(x, w, scale, bias, kind, k, a, eps=dr.EPS_CONV):
    """DECONV / UPCONV stage of an NHWC interval + folded BN + act, before rounding: ``dense_ref.conv`` of the zero-inserted
    interval (zeros have radius 0, so they add neither to the magnitude nor to the radius)."""
    n, h, wd, ci = x.c.shape
    up = sr.Iv(np.zeros((n, 2 * h, 2 * wd, ci)))
    up.c[:, ::2, ::2] = x.c
    up.r[:, ::2, ::2] = x.r
    return dr.conv(up, conv_weights(kind, w, ci, len(scale), k), scale, bias, k, a, eps)


def forward(descs, weights, x_nchw, dtype=None, eps=sr.EPS, eps_conv=dr.EPS_CONV, stages=None):
    """``dense_ref.forward`` with DECONV / UPCONV stages."""
    if dtype is None:
        eps = eps_conv = 0.0
    cur, outs = None, []
    for d, wt in zip(descs, weights):
        if d['kind'] in (DECONV, UPCONV):
            y = sr.quantize(convt(cur, wt[3], wt[4], wt[5], d['kind'], d['ksize'], d['act'], eps_conv), dtype)
        elif d['kind'] == sr.HEAD:
            hd = sr.quantize(sr.head(cur, wt[3], wt[4], wt[5], d['act'], eps), dtype)
            return sr.Iv(hd.c[:, None], hd.r[:, None])
        else:
            if d['kind'] == sr.STEM:
                y = sr.quantize(sr.stem(x_nchw, wt[3], wt[4], wt[5], d['stride'], d['act'], eps), dtype)
            elif d['kind'] == sr.DWPW:
                y = sr.quantize(sr.dwpw(cur, wt, d, dtype, None, eps)['out'], dtype)
            else:
                y = sr.quantize(dr.conv(cur, wt[3], wt[4], wt[5], d['ksize'], d['act'], eps_conv), dtype)
                y = sr.upsample(y) if d.get('upsample') else y
        outs.append(y)
        if stages is not None:
            stages.append(y)
        cur = y
    raise ValueError('stage list has no head')
