"""ORACLE -- TEST INFRASTRUCTURE ONLY.  Per-stage fp64 reference of the C-ABI's stage list, with interval bounds.

Works on exactly what ``fd_plan_create`` / ``fd_plan_set_stage_weights`` receive: the ``fd_stage_desc`` dicts and the
per-stage weight tuples ``(dw_w, dw_scale, dw_bias, pw_w, pw_scale, pw_bias)`` with BatchNorm already folded
(``fastdepth_b200.plan.describe`` or any hand-built list).  Unlike ``fastdepth_oracle`` it is not tied to the
MobileNet names, strides or activations.

Every tensor is a midpoint-radius interval (``Iv``: fp64 centre and radius, NHWC) that contains every value a correct
kernel may hold at that point:

* a linear op (stem, depthwise, pointwise, head, skip add) maps the radius to ``|W|·r + EPS·|W|·(|c| + r)``, where
  EPS is the allowance for one fp32 sum in any order; the folded BN ``acc·scale + bias`` adds the fp32 rounding of the
  affine itself;
* an activation is applied to both ends;
* rounding to the storage dtype (fp16 / bf16: round-to-nearest-even straight from fp64) yields the interval spanned by
  the roundings of both ends -- the set of values the rounding can give.

The rounding points are the product's own (DESIGN.md section 2): the stem output, each depthwise result, each
pointwise result, the upsampled result BEFORE a skip add, the skip sum, the head output.  A stage computed from the
GPU's own input tensors therefore starts with radius 0; the only slack left is fp32 accumulation order and the rounding
flips of the intermediate depthwise result.  ``check`` then demands that every 16-bit element be one of the roundings
its interval admits, and exactly the round-to-nearest value wherever the interval contains no rounding midpoint.
"""
import numpy as np

EPS = 2.0 ** -18          # one fp32 sum of any length used here, any order (measured on the H100, DESIGN.md section 4)
U32 = 2.0 ** -24          # unit roundoff of fp32 (the BN affine's own rounding, the fp32 skip add)
RELU, RELU6 = 0, 1        # fd_act
STEM, DWPW, HEAD = 0, 1, 2

# significand bits, frexp exponent floor (subnormal spacing), largest finite value
_FMT = {'float16': (11, -13, 65504.0), 'bfloat16': (8, -125, float.fromhex('0x1.fe00000000000p+127'))}


def _dtname(dtype):
    """'float16' | 'bfloat16' | 'float32' from a torch dtype, numpy dtype or name."""
    s = str(dtype).replace('torch.', '')
    if s in ('float16', 'half'):
        return 'float16'
    if s in ('bfloat16',):
        return 'bfloat16'
    if s in ('float32', 'float'):
        return 'float32'
    raise ValueError('unsupported dtype %r' % (dtype,))


def round_rne(x, dtype):
    """Round fp64 values straight to fp16 / bf16 (round to nearest, ties to even; overflow to +-inf), returned as fp64."""
    p, emin, vmax = _FMT[_dtname(dtype)]
    x = np.asarray(x, dtype=np.float64)
    _, e = np.frexp(x)
    q = np.ldexp(1.0, np.maximum(e, emin) - p)          # spacing of the format around x
    with np.errstate(invalid='ignore', over='ignore'):
        r = np.rint(x / q) * q
        r = np.where(np.abs(r) > vmax, np.copysign(np.inf, x), r)
    return np.where(np.isfinite(x), r, x)


class Iv:
    """Midpoint-radius interval tensor (fp64)."""
    __slots__ = ('c', 'r')

    def __init__(self, c, r=None):
        self.c = np.asarray(c, dtype=np.float64)
        self.r = np.zeros_like(self.c) if r is None else np.asarray(r, dtype=np.float64)

    @property
    def lo(self):
        return self.c - self.r

    @property
    def hi(self):
        return self.c + self.r

    @staticmethod
    def span(lo, hi):
        return Iv((lo + hi) * 0.5, (hi - lo) * 0.5)

    def mag(self):
        return np.abs(self.c) + self.r


def exact(a):
    """A tensor the GPU produced (or any exactly known tensor): radius 0."""
    if hasattr(a, 'detach'):
        a = a.detach().float().cpu().numpy()
    return Iv(np.asarray(a, dtype=np.float64))


def act(iv, a):
    """ReLU / ReLU6 on both ends (``a=None``: no activation, for calibration probes)."""
    if a is None:
        return iv
    lo, hi = np.maximum(iv.lo, 0.0), np.maximum(iv.hi, 0.0)
    if a == RELU6:
        lo, hi = np.minimum(lo, 6.0), np.minimum(hi, 6.0)
    return Iv.span(lo, hi)


def quantize(iv, dtype):
    """The interval of values that rounding ``iv`` to the storage dtype can give (``None``: no rounding at all)."""
    if dtype is None:
        return iv
    if _dtname(dtype) == 'float32':
        return Iv(iv.c, iv.r + U32 * iv.mag())
    return Iv.span(round_rne(iv.lo, dtype), round_rne(iv.hi, dtype))


def _affine(c, m, r, scale, bias, eps):
    """fp32 ``acc·scale + bias`` on an accumulator with centre c, magnitude bound m (sum of |terms|) and radius r."""
    s, b = np.asarray(scale, np.float64), np.asarray(bias, np.float64)
    r = r + eps * m
    return Iv(c * s + b, np.abs(s) * r + (2 * U32 if eps else 0.0) * (np.abs(s) * (np.abs(c) + r) + np.abs(b)))


def stem(x_nchw, w, scale, bias, stride, a, eps=EPS):
    """Dense 3x3 stride-s conv (padding 1) of the exact NCHW input x, + folded BN + act; NHWC, before rounding."""
    x = np.asarray(x_nchw, np.float64).transpose(0, 2, 3, 1)
    w = np.asarray(w, np.float64).reshape(-1, 3, 3, 3)             # [co][ci][ky][kx]
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
    return act(_affine(c, m, 0.0, scale, bias, eps), a)


def depthwise(x, taps, scale, bias, k, stride, a, eps=EPS):
    """Depthwise kxk stride-s conv (padding (k-1)/2) + folded BN + act on an NHWC interval; before rounding."""
    t = np.asarray(taps, np.float64).reshape(-1, k, k)              # [c][ky][kx]
    p = (k - 1) // 2
    n, h, wd, ch = x.c.shape
    ho, wo = (h + 2 * p - k) // stride + 1, (wd + 2 * p - k) // stride + 1
    pad = ((0, 0), (p, p), (p, p), (0, 0))
    xc, xm, xr = np.pad(x.c, pad), np.pad(x.mag(), pad), np.pad(x.r, pad)
    c = np.zeros((n, ho, wo, ch)); m = np.zeros_like(c); r = np.zeros_like(c)
    for ky in range(k):
        for kx in range(k):
            sl = (slice(None), slice(ky, ky + stride * (ho - 1) + 1, stride), slice(kx, kx + stride * (wo - 1) + 1, stride))
            wk = t[:, ky, kx]
            c += xc[sl] * wk
            m += xm[sl] * np.abs(wk)
            r += xr[sl] * np.abs(wk)
    return act(_affine(c, m, r, scale, bias, eps), a)


def pointwise(x, w, scale, bias, a, eps=EPS):
    """1x1 conv [c_out][c_in] + folded BN + act on an NHWC interval; before rounding."""
    wt = np.asarray(w, np.float64).reshape(len(scale), -1).T        # [c_in][c_out]
    aw = np.abs(wt)
    return act(_affine(x.c @ wt, x.mag() @ aw, x.r @ aw, scale, bias, eps), a)


def head(x, w, scale, bias, a, eps=EPS):
    """C -> 1 pointwise + BN + act: [n,h,w] before rounding."""
    wt = np.asarray(w, np.float64).reshape(-1)
    aw = np.abs(wt)
    s, b = np.asarray(scale, np.float64).reshape(-1)[0], np.asarray(bias, np.float64).reshape(-1)[0]
    return act(_affine(x.c @ wt, x.mag() @ aw, x.r @ aw, s, b, eps), a)


def upsample(iv):
    """Nearest x2 on NHWC (or on [n,h,w] head maps)."""
    def up(t):
        return t.repeat(2, axis=1).repeat(2, axis=2)
    return Iv(up(iv.c), up(iv.r))


def add(u, skip, exact_sum=False):
    """Skip add of the ROUNDED upsampled tensor and the skip tensor, summed in fp32; before rounding."""
    c = u.c + skip.c
    return Iv(c, u.r + skip.r + (0.0 if exact_sum else U32) * (np.abs(c) + u.r + skip.r))


def concat(a, b):
    return Iv(np.concatenate([a.c, b.c], axis=-1), np.concatenate([a.r, b.r], axis=-1))


def dwpw(x, wt, desc, dtype, skip=None, eps=EPS):
    """One DWPW stage from its (interval) input.  Returns dict of pre-rounding intervals:
    'dw' (depthwise result), 'pw' (pointwise result at the conv resolution) and 'out' (what the stage buffer holds:
    the pointwise result, upsampled, plus the skip for skip_mode 0 -- ``skip`` is the skip tensor)."""
    dw_w, dw_s, dw_b, pw_w, pw_s, pw_b = wt
    k, a = desc['ksize'], desc['act']
    d = depthwise(x, dw_w, dw_s, dw_b, k, desc['stride'], a, eps)
    p = pointwise(quantize(d, dtype), pw_w, pw_s, pw_b, a, eps)
    out = p
    if desc.get('upsample'):
        out = upsample(p)
        if skip is not None and not desc.get('skip_mode', 0):
            out = add(quantize(out, dtype), skip, exact_sum=dtype is None)
    return {'dw': d, 'pw': p, 'out': out}


def forward(descs, weights, x_nchw, dtype=None, eps=EPS, stages=None):
    """Compose the whole stage list from the exact input x (NCHW).  ``dtype=None``: no rounding anywhere (pure fp64,
    eps ignored).  Returns the head output as an [n,1,h,w] interval; ``stages`` (optional list) receives each
    non-head stage's buffer content (rounded, NHWC, the stage's own channels only).  Over a whole network the
    worst-case radii of the rounding flips grow past an ulp, so kernels are checked one stage at a time."""
    if dtype is None:
        eps = 0.0
    outs = []
    cur = None
    for i, (d, wt) in enumerate(zip(descs, weights)):
        if d['kind'] == STEM:
            y = quantize(stem(x_nchw, wt[3], wt[4], wt[5], d['stride'], d['act'], eps), dtype)
            nxt = y
        elif d['kind'] == DWPW:
            src = d.get('skip_src', -1)
            skip = outs[src] if src >= 0 else None
            y = quantize(dwpw(cur, wt, d, dtype, skip, eps)['out'], dtype)
            nxt = concat(y, skip) if (skip is not None and d.get('skip_mode', 0)) else y
        else:
            hd = quantize(head(cur, wt[3], wt[4], wt[5], d['act'], eps), dtype)
            return Iv(hd.c[:, None], hd.r[:, None])
        outs.append(y)
        if stages is not None:
            stages.append(y)
        cur = nxt
    raise ValueError('stage list has no head')


def check(got, iv, dtype, what=''):
    """Assert that ``got`` (the kernel's tensor, same layout as ``iv``) is a value a correct kernel may produce.

    16-bit: every element must be a rounding of some point of its pre-rounding interval ``iv``, and exactly the
    round-to-nearest value where the interval holds no rounding midpoint.  fp32: ``|got - centre| <= radius + ulp/2``.
    Returns the fraction of elements whose result is determined (a single admissible value); for fp32 that is always
    1.0 -- the fp32 rule is the bound itself, so a floor on the determined fraction says nothing about fp32 tensors."""
    g = got.detach().float().cpu().numpy().astype(np.float64) if hasattr(got, 'detach') else np.asarray(got, np.float64)
    assert g.shape == iv.c.shape, (what, g.shape, iv.c.shape)
    name = _dtname(dtype)
    if name == 'float32':
        ulp = np.spacing(np.abs(g).astype(np.float32)).astype(np.float64)
        ok = np.abs(g - iv.c) <= iv.r + 0.5 * ulp
        det = np.ones(g.shape, bool)
        lo, hi = iv.c - iv.r, iv.c + iv.r
    else:
        lo, hi = round_rne(iv.lo, dtype), round_rne(iv.hi, dtype)
        ok = (g >= lo) & (g <= hi)                          # NaN fails both comparisons
        det = lo == hi
    if not ok.all():
        bad = np.argwhere(~ok)
        i = tuple(bad[0])
        raise AssertionError('%s: %d of %d elements outside the reference (first at %s: got %r, admissible [%r, %r], '
                             'centre %r radius %r)' % (what, len(bad), g.size, i, g[i], lo[i], hi[i], iv.c[i], iv.r[i]))
    return float(det.mean())
