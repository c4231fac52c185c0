"""Stage-by-stage check of a plan against the per-stage fp64 interval reference (oracle/stage_ref.py), computed from the
GPU's OWN input tensors.  Shared by the kernel sweep (test_kernel_sweep.py) and the production-plan check
(test_production_plans.py).

A 16-bit element must be a rounding of a value its interval admits, and exactly the round-to-nearest value wherever the
interval holds no rounding midpoint (stage_ref.check); at least half of every single-stage 16-bit tensor must be
determined that way.  A run of layers inside one chain kernel, and a last block with the head fused into it, are
compositions: they are checked for containment only, then every one of their stages is held to the full rule in a re-run
of the same plan with the chain (``chain=0``) or the fused head (``fold_head=0``) switched off.

``check_plan`` runs every forward once per pass and checks the given images in chunks, so the fp64 reference of a
64-image 224x224 batch never has to be held in host memory at once.  DWPW stages go through ``stage_ref.dwpw``; CONV
stages through ``dense_ref.conv`` (rounded, then upsampled unless the head is folded) and DECONV / UPCONV stages through
``convt_ref.convt``."""
import numpy as np
import torch

import convt_ref as cr
import dense_ref as dr
from oracle import stage_ref as sr

MIN_DETERMINED = 0.5
CHUNK = 8                  # images per CPU reference chunk
DENSE = (dr.CONV, cr.DECONV, cr.UPCONV)


def nhwc(t, pick):
    return t[pick].float().cpu().numpy().astype(np.float64)


class Checker:
    """``sr.check`` of every tensor of one pass, chunk by chunk; ``flush`` ends the pass and holds each strictly checked
    tensor, over all its checked images, to MIN_DETERMINED (``floor``: a lower floor, which the caller states together
    with the measured fractions and the reason)."""

    def __init__(self, case, dtype, floor=MIN_DETERMINED):
        self.case, self.dtype, self.floor = case, dtype, floor
        self.fracs = []          # determined fraction of every strictly checked tensor
        self.composed = {}       # what -> determined fraction of a containment-only composition (chain run, block + head)
        self.results = []        # (what, determined fraction, strict), in check order
        self.n = self.zeros = self.sixes = 0
        self._open = {}          # what -> [determined elements, elements, strict] of the pass in progress

    def __call__(self, got, iv, what, strict=True):
        self.n += got.size
        self.zeros += int((got == 0).sum())
        self.sixes += int((got == 6).sum())
        f = sr.check(got, iv, self.dtype, '%s: %s' % (self.case, what))
        acc = self._open.setdefault(what, [0, 0, strict])
        acc[0] += int(round(f * got.size))
        acc[1] += got.size

    def flush(self):
        for what, (det, size, strict) in self._open.items():
            f = det / size
            self.results.append((what, f, strict))
            if strict:
                assert f >= self.floor, \
                    '%s: %s: only %.3f of the elements are determined' % (self.case, what, f)
                self.fracs.append(f)
            else:                # its determined elements are still held to exact equality by sr.check
                self.composed[what] = f
        self._open = {}


def chain_runs(steps):
    """First stage of every chain kernel's run -> its last stage."""
    runs = {}
    for s in steps:
        if 'chain_tc' in s['kernel']:
            a, b = s['kernel'].split('{stages ')[1].rstrip('}').split('-')
            runs[int(a)] = int(b)
    return runs


def _forward(p, x, y, stream):
    p.forward(x, y, stream)
    if y.is_cuda:
        torch.cuda.synchronize()


def check_plan(p, descs, weights, dtype, x_host, x, y, images, chk, opts=None, inplace=1, stream=0, chunk=CHUNK,
               only=None, rerun_all=True):
    """Run ``p`` (a ``fastdepth_b200.plan.Plan``, or anything with its ``forward`` / ``steps`` / ``stage_tensor`` /
    ``set_option``) on x and check every stage it materialises for ``images`` (NCHW ``x_host``: x's exact values).

    Pass 1 runs with ``inplace_skip`` 0, so every skip source is kept and checked; with skip adds and ``inplace`` 1 a
    second pass rechecks the decoder blocks that add in place (and the head), against pass 1's sources.  Then, if the
    plan ran a chain kernel, a re-run with ``chain`` 0 holds the chain's layers to the strict rule, and if it fused the head
    into the last block, a re-run with ``fold_head`` 0 does the same for the fused head.  ``opts``: the options the caller
    set on the plan (``path``, ``fold_head``); ``only``: the stage indices to check (None: all, the head is index
    len(descs) - 1); ``rerun_all`` False: the re-runs check only the stages they exist for.  The plan is left with the
    caller's options.  Returns the steps of the main passes."""
    opts = dict(opts or {})
    descs = [dict({'skip_mode': 0}, **d) for d in descs]
    ns = len(descs)
    images = list(images)
    chunks = [images[k:k + chunk] for k in range(0, len(images), chunk)]
    has_add = any(d['skip_src'] >= 0 and not d['skip_mode'] for d in descs)
    is_src = {d['skip_src'] for d in descs if d['skip_src'] >= 0 and not d['skip_mode']}

    def focus(stages):
        return set(stages) if only is None else set(stages) & set(only)

    passes = [0, 1] if (has_add and inplace) else [inplace]
    ran, saved = [], {}
    for ip in passes:
        if ip and len(passes) == 2:
            # pass 1's skip sources, before pass 2 adds onto them in place
            saved = {s: p.stage_tensor(s).clone() for s in is_src}
        p.set_option('inplace_skip', ip)
        _forward(p, x, y, stream)
        steps = p.steps()
        ran.append(steps)
        for pick in chunks:
            _check_plan(p, descs, weights, dtype, x_host, y, pick, steps, chk, saved, ip, ip and len(passes) == 2, opts,
                        only)
        chk.flush()
    saved = None
    main = [s for steps in ran for s in steps]
    chain_stages = {t for a, b in chain_runs(main).items() for t in range(a, b + 1)}
    if focus(chain_stages):
        # the layers of every chain run one by one (per-block kernels), each checked from its own materialised input
        st = focus(range(ns) if rerun_all else chain_stages)
        p.set_option('chain', 0)
        p.set_option('inplace_skip', 0)
        _forward(p, x, y, stream)
        steps = p.steps()
        for pick in chunks:
            _check_plan(p, descs, weights, dtype, x_host, y, pick, steps, chk, {}, 0, False, dict(opts, chain=0), st)
        chk.flush()
        p.set_option('chain', 1)
    if any('+head' in s['kernel'] for s in main) and focus({ns - 2, ns - 1}):
        # the fused head on its own: the same plan with the head unfused materialises the last block's output (the same
        # kernel instance and accumulation order), and the fused kernel's depth map is checked against the head of it
        st = focus(range(ns) if rerun_all else {ns - 2, ns - 1})
        yf = y.clone()
        p.set_option('fold_head', 0)
        p.set_option('inplace_skip', 0)
        _forward(p, x, y, stream)
        steps = p.steps()
        for pick in chunks:
            _check_plan(p, descs, weights, dtype, x_host, y, pick, steps, chk, {}, 0, False, dict(opts, fold_head=0), st)
            last = sr.exact(nhwc(p.stage_tensor(ns - 2), pick))
            chk(nhwc(yf[:, 0], pick), sr.head(last, *weights[-1][3:], descs[-1]['act']), 'fused head')
        chk.flush()
        p.set_option('fold_head', opts.get('fold_head', 1))
        y.copy_(yf)
    p.set_option('inplace_skip', inplace)
    return ran


def _check_plan(p, descs, weights, dtype, x_host, y, pick, steps, chk, saved, ip, recheck, opts, only):
    """Check every stage the plan materialised for the images ``pick`` (``recheck``: only the decoder blocks that add in
    place, and the head; ``only``: those stage indices)."""
    ns = len(descs)
    q = None if dtype == torch.float32 else dtype
    fold = opts.get('fold_head', 1) and descs[-2]['upsample'] and descs[-2]['skip_src'] < 0
    chained = chain_runs(steps)                    # first stage of a chain run -> last stage
    head_fused = any('+head' in s['kernel'] for s in steps)
    path0 = opts.get('path', 1) == 0

    def want(i):
        return only is None or i in only

    def buf(i):
        return sr.exact(nhwc(p.stage_tensor(i), pick))

    def stage_input(i):
        if i == 0:
            return None
        d = descs[i - 1]
        t = buf(i - 1)
        if d['skip_src'] >= 0 and d['skip_mode']:
            t = sr.concat(t, buf(d['skip_src']))
        return t

    def skip_of(d):
        src = d['skip_src']
        if src < 0 or d['skip_mode']:
            return None
        return sr.exact(nhwc(saved[src], pick)) if ip else buf(src)

    i = 0
    while i < ns - 1:
        d = descs[i]
        if not want(i):
            i = chained[i] + 1 if i in chained else i + 1
            continue
        if d['kind'] == sr.STEM:
            if not recheck:
                chk(nhwc(p.stage_tensor(0), pick),
                    sr.stem(x_host[pick], weights[0][3], weights[0][4], weights[0][5], d['stride'], d['act']), 'stem')
            i += 1
            continue
        last = i == ns - 2
        if recheck and not (d['skip_src'] >= 0 and not d['skip_mode']):
            i += 1
            continue
        if d['kind'] in DENSE:
            wt = weights[i]
            if d['kind'] == dr.CONV:
                r = sr.quantize(dr.conv(stage_input(i), wt[3], wt[4], wt[5], d['ksize'], d['act']), q)
                if d['upsample'] and not (last and fold):
                    r = sr.upsample(r)
            else:
                r = sr.quantize(cr.convt(stage_input(i), wt[3], wt[4], wt[5], d['kind'], d['ksize'], d['act']), q)
            chk(nhwc(p.stage_tensor(i), pick), r, 'stage %d' % i)
            i += 1
            continue
        if i in chained:                           # a run inside one chain kernel: composition from the run's input
            j = chained[i]
            cur = stage_input(i)
            for t in range(i, j + 1):
                r = sr.dwpw(cur, weights[t], descs[t], q)['out']
                cur = sr.quantize(r, q) if t < j else r
            # containment only: over several layers the worst-case radii of the intermediate rounding flips outgrow the ulp;
            # check_plan holds every one of these layers to the full rule in the same plan without the chain kernel
            chk(nhwc(p.stage_tensor(j), pick), cur, 'chain %d-%d' % (i, j), strict=False)
            i = j + 1
            continue
        if last and head_fused:                    # block + head in one kernel: composition from the block's input
            r = sr.dwpw(stage_input(i), weights[i], dict(d, upsample=0), q)['out']
            hd = sr.head(sr.quantize(r, q), *weights[-1][3:], descs[-1]['act'])
            # a composition through a whole block: the worst-case radii of the rounding flips inside the block add up over the
            # head's dot product, so only containment is demanded here; the fused head is held to the determined-fraction rule
            # against the unfused plan in check_plan
            chk(nhwc(y[:, 0], pick), sr.upsample(hd), 'block %d + head' % i, strict=False)
            return
        dd = dict(d, upsample=0) if (last and fold) else d
        r = sr.dwpw(stage_input(i), weights[i], dd, q, skip_of(d))
        if path0:                                  # both halves on their own, from the kernel's own intermediate
            chk(nhwc(p.stage_tensor(i, which=1), pick), r['dw'], 'stage %d depthwise' % i)
            mid = sr.exact(nhwc(p.stage_tensor(i, which=1), pick))
            r = pw_from_mid(mid, weights[i], dd, q, skip_of(d))
        chk(nhwc(p.stage_tensor(i), pick), r['out'], 'stage %d' % i)
        i += 1
    if head_fused or not want(ns - 1):
        return                                     # (a fused head is checked in the first pass)
    # the head (unfused): from the last stage's buffer
    hin = stage_input(ns - 1)
    hd = sr.head(hin, *weights[-1][3:], descs[-1]['act'])
    chk(nhwc(y[:, 0], pick), sr.upsample(hd) if fold else hd, 'head')


def pw_from_mid(mid, wt, d, q, skip):
    p = sr.pointwise(mid, wt[3], wt[4], wt[5], d['act'])
    out = p
    if d['upsample']:
        out = sr.upsample(p)
        if skip is not None and not d['skip_mode']:
            out = sr.add(sr.quantize(out, q), skip)
    return {'pw': p, 'out': out}
