"""Test helpers for the dense NNConv decoder (``models.MobileNet('nnconv5')``): three independent references.

* ``torch_forward``: the forward restated with PyTorch primitives (F.conv2d, folded-from-running-stats BN, clamps,
  repeat_interleave), optionally with the product's storage roundings (``storage=dtype``);
* ``c_forward``: the same composed from the plain-C oracle primitives (``oracle/c_oracle.py``'s fo_conv_dense & co.);
* ``conv`` / ``forward``: the per-stage fp64 interval reference of ``oracle/stage_ref.py`` extended by a CONV stage
  (interval dense conv of an NHWC input, generalising ``stage_ref.stem``).

``EPS_CONV`` is the allowance for one fp32 dense-conv sum (up to k*k*c_in = 25 600 products, accumulated by wgmma or by the
SIMT kernel in any order); ``stage_ref.EPS`` stays the bound of the <= 1 024-term sums it was established on.
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import c_oracle
from oracle import stage_ref as sr

CONV = 3
EPS_CONV = 2.0 ** -18
ENCODER_STRIDES = (2, 1, 2, 1, 2, 1, 2, 1, 1, 1, 1, 1, 2, 1)


# ------------------------------------------------------------------------------------------------ PyTorch primitives
def _bn(x, sd, p, hi):
    inv = sd[p + '.weight'].double() / torch.sqrt(sd[p + '.running_var'].double() + 1e-5)
    b = sd[p + '.bias'].double() - sd[p + '.running_mean'].double() * inv
    y = x * inv.to(x.dtype).view(1, -1, 1, 1) + b.to(x.dtype).view(1, -1, 1, 1)
    return y.clamp(0.0, hi) if hi is not None else y.clamp_min(0.0)


def torch_forward(sd, x, storage=None):
    """``MobileNet('nnconv<k>')`` forward on a ``synthetic_nnconv_state_dict``-schema state_dict, fp32 arithmetic.  With
    ``storage`` (torch.float16 / bfloat16) every tensor the product keeps in 16 bits is rounded to it: the parameters, the
    input, the stem output, each depthwise and pointwise result, each dense conv result and the head output."""
    def q(t):
        return t if storage is None else t.to(storage).float()
    sd = {k: (q(v) if v.is_floating_point() else v) for k, v in sd.items()}      # what model.half() holds
    x = q(x if x.dtype == torch.float64 else x.float())
    x = q(_bn(F.conv2d(x, sd['mobilenet.0.0.weight'], None, 2, 1), sd, 'mobilenet.0.1', 6.0))
    for i in range(1, 14):
        w = sd['mobilenet.%d.0.weight' % i]
        x = q(_bn(F.conv2d(x, w, None, ENCODER_STRIDES[i], 1, 1, w.shape[0]), sd, 'mobilenet.%d.1' % i, 6.0))
        x = q(_bn(F.conv2d(x, sd['mobilenet.%d.3.weight' % i]), sd, 'mobilenet.%d.4' % i, 6.0))
    for j in range(1, 6):
        w = sd['decoder.conv%d.0.weight' % j]
        x = q(_bn(F.conv2d(x, w, None, 1, (w.shape[-1] - 1) // 2), sd, 'decoder.conv%d.1' % j, None))
        x = x.repeat_interleave(2, dim=2).repeat_interleave(2, dim=3)
    return q(_bn(F.conv2d(x, sd['decoder.conv6.0.weight']), sd, 'decoder.conv6.1', None))


# ------------------------------------------------------------------------------------------------ C oracle composition
def c_forward(sd, x):
    """The same forward from the plain-C primitives (fo_conv_dense for the stem and every decoder conv)."""
    g = c_oracle._np
    x = g(x)
    x = c_oracle._bn_act(c_oracle._dense(x, g(sd['mobilenet.0.0.weight']), 2, 1), sd, 'mobilenet.0.1', 2)
    for i in range(1, 14):
        x = c_oracle._bn_act(c_oracle._depthwise(x, g(sd['mobilenet.%d.0.weight' % i]), ENCODER_STRIDES[i]), sd,
                             'mobilenet.%d.1' % i, 2)
        x = c_oracle._bn_act(c_oracle._pointwise(x, g(sd['mobilenet.%d.3.weight' % i])), sd, 'mobilenet.%d.4' % i, 2)
    for j in range(1, 6):
        w = g(sd['decoder.conv%d.0.weight' % j])
        x = c_oracle._upsample(c_oracle._bn_act(c_oracle._dense(x, w, 1, (w.shape[-1] - 1) // 2), sd, 'decoder.conv%d.1' % j, 1))
    return c_oracle._bn_act(c_oracle._pointwise(x, g(sd['decoder.conv6.0.weight'])), sd, 'decoder.conv6.1', 1)


# ------------------------------------------------------------------------------------------------ interval reference
def conv(x, w, scale, bias, k, a, eps=EPS_CONV):
    """Dense kxk stride-1 conv (padding (k-1)/2) of an NHWC interval + folded BN + act; before rounding.
    ``w``: [c_out][c_in][k][k] (or flattened [c_out][c_in*k*k])."""
    co = len(scale)
    w = np.asarray(w, np.float64).reshape(co, -1, k, k)
    p = (k - 1) // 2
    pad = ((0, 0), (p, p), (p, p), (0, 0))
    xc, xm, xr = np.pad(x.c, pad), np.pad(x.mag(), pad), np.pad(x.r, pad)
    n, h, wd, _ = x.c.shape
    c = np.zeros((n, h, wd, co)); m = np.zeros_like(c); r = np.zeros_like(c)
    for ky in range(k):
        for kx in range(k):
            sl = (slice(None), slice(ky, ky + h), slice(kx, kx + wd))
            wk = w[:, :, ky, kx].T                                   # [ci][co]
            awk = np.abs(wk)
            c += xc[sl] @ wk
            m += xm[sl] @ awk
            r += xr[sl] @ awk
    return sr.act(sr._affine(c, m, r, scale, bias, eps), a)


def forward(descs, weights, x_nchw, dtype=None, eps=sr.EPS, eps_conv=EPS_CONV, stages=None):
    """``stage_ref.forward`` with CONV stages: the stage buffer holds the conv result, rounded, then upsampled."""
    if dtype is None:
        eps = eps_conv = 0.0
    cur = None
    outs = []
    for d, wt in zip(descs, weights):
        if d['kind'] == sr.STEM:
            y = sr.quantize(sr.stem(x_nchw, wt[3], wt[4], wt[5], d['stride'], d['act'], eps), dtype)
        elif d['kind'] == sr.DWPW:
            src = d.get('skip_src', -1)
            y = sr.quantize(sr.dwpw(cur, wt, d, dtype, outs[src] if src >= 0 else None, eps)['out'], dtype)
        elif d['kind'] == CONV:
            y = sr.quantize(conv(cur, wt[3], wt[4], wt[5], d['ksize'], d['act'], eps_conv), dtype)
            if d.get('upsample'):
                y = sr.upsample(y)
        else:
            hd = sr.quantize(sr.head(cur, wt[3], wt[4], wt[5], d['act'], eps), dtype)
            return sr.Iv(hd.c[:, None], hd.r[:, None])
        outs.append(y)
        if stages is not None:
            stages.append(y)
        cur = y
    raise ValueError('stage list has no head')
