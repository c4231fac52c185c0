"""CPU test of the per-stage plan checker (tests/plan_check.py) on a stand-in plan: no GPU needed.

The stand-in is shaped like ``fastdepth_b200.plan.Plan``; its stage buffers are the round-to-nearest values of the
reference's own point forward, each stage computed from the previous stages' rounded buffers -- what a correct kernel
leaves wherever its result is determined.  The checker must accept it, and must reject it once a single 128-pixel x
64-channel block of one image in the middle of the batch is moved by one ulp in one stage: a fault confined to a few
work items, which a check of picked images end to end does not see."""
import numpy as np
import pytest
import torch

import plan_check as pc
from oracle import stage_ref as sr

F16 = torch.float16
R, R6 = sr.RELU, sr.RELU6
N, H, W = 12, 64, 64


def _desc(kind, c_in, c_out, k, s, act, up=0, skip=-1):
    return dict(kind=kind, c_in=c_in, c_out=c_out, ksize=k, stride=s, act=act, upsample=up, skip_src=skip, skip_mode=0)


# stem s2 -> 3x3 (64 channels at 32x32, a skip source) -> 3x3 s2 -> 3x3 -> 5x5 up + skip(1) -> 5x5 up (head folded) -> head
DESCS = [_desc(sr.STEM, 3, 16, 3, 2, R6), _desc(sr.DWPW, 16, 64, 3, 1, R6), _desc(sr.DWPW, 64, 64, 3, 2, R6),
         _desc(sr.DWPW, 64, 96, 3, 1, R6), _desc(sr.DWPW, 96, 64, 5, 1, R, 1, 1), _desc(sr.DWPW, 64, 16, 5, 1, R, 1),
         _desc(sr.HEAD, 16, 1, 1, 1, R)]


def _weights(rng):
    def rep(a):
        return sr.round_rne(a, F16).astype(np.float32)

    def affine(c):
        return rng.uniform(0.5, 1.5, c).astype(np.float32), rng.normal(0.2, 0.3, c).astype(np.float32)

    wts = []
    for d in DESCS:
        ci, co, k = d['c_in'], d['c_out'], d['ksize']
        if d['kind'] == sr.STEM:
            wts.append((None, None, None, rep(rng.normal(0, np.sqrt(2 / 27), (co, 27)))) + affine(co))
        elif d['kind'] == sr.DWPW:
            wts.append((rep(rng.normal(0, np.sqrt(2.0 / (k * k)), (ci, k * k))),) + affine(ci) +
                       (rep(rng.uniform(-1, 1, (co, ci)) * np.sqrt(3.0 / ci)),) + affine(co))
        else:
            wts.append((None, None, None, rep(np.abs(rng.normal(0, 1 / np.sqrt(ci), (1, ci)))),
                        np.ones(1, np.float32), np.ones(1, np.float32)))
    return wts


class StandInPlan:
    """``stage_tensor`` / ``steps`` / ``forward`` / ``set_option`` of a Plan whose buffers hold the reference's rounded
    point forward.  The last block's buffer is at the conv resolution and the depth map is the upsampled head, as with a
    folded head."""

    def __init__(self, descs, weights, x_host, dtype):
        fold = [dict(d, upsample=0) if i == len(descs) - 2 else d for i, d in enumerate(descs)]
        bufs, cur = [], None
        for d, wt in zip(fold, weights):
            if d['kind'] == sr.STEM:
                r = sr.stem(x_host, wt[3], wt[4], wt[5], d['stride'], d['act'], eps=0)
            elif d['kind'] == sr.DWPW:
                skip = bufs[d['skip_src']] if d['skip_src'] >= 0 else None
                r = sr.dwpw(cur, wt, d, dtype, skip, eps=0)['out']
            else:
                r = sr.head(cur, wt[3], wt[4], wt[5], d['act'], eps=0)
            cur = sr.exact(sr.round_rne(r.c, dtype))
            bufs.append(cur)
        self.bufs = [torch.from_numpy(b.c).to(dtype) for b in bufs[:-1]]
        self.depth = torch.from_numpy(sr.upsample(bufs[-1]).c[:, None]).to(dtype)
        self.options = {}
        self.forwards = 0

    def set_option(self, name, value):
        self.options[name] = int(value)

    def steps(self):
        return [dict(stage=i, kernel='block_tc<stand-in>') for i in range(len(self.bufs))] + \
            [dict(stage=len(self.bufs), kernel='head_kernel<up2x>')]

    def forward(self, x, y, stream):
        self.forwards += 1
        y.copy_(self.depth)

    def stage_tensor(self, stage, which=0):
        return self.bufs[stage]


def _check(p, x_host, images):
    chk = pc.Checker('stand-in', F16)
    y = torch.empty((N, 1, H, W), dtype=F16)
    pc.check_plan(p, DESCS, WEIGHTS, F16, x_host, torch.from_numpy(x_host).to(F16), y, images, chk)
    return chk


WEIGHTS = _weights(np.random.default_rng(5))


def test_checker_accepts_the_reference_and_catches_one_block_one_ulp_off():
    x_host = sr.round_rne(np.random.default_rng(6).uniform(0, 1, (N, 3, H, W)), F16).astype(np.float32)
    p = StandInPlan(DESCS, WEIGHTS, x_host, F16)
    chk = _check(p, x_host, range(N))
    # pass 1: stem, 5 blocks and the head; pass 2: the block that adds in place and the head
    assert [w for w, _, _ in chk.results] == ['stem'] + ['stage %d' % i for i in range(1, 6)] + ['head', 'stage 4', 'head']
    assert min(chk.fracs) >= pc.MIN_DETERMINED and p.forwards == 2 and p.options['inplace_skip'] == 1

    # one ulp up in stage 1 of image 5: pixels 0..127 of its 32x32 map, channels 0..63
    blk = p.bufs[1][5].reshape(-1, 64)[:128]
    moved = np.nextafter(blk.numpy(), np.float16(np.inf))
    assert (moved != blk.numpy()).all()
    blk.copy_(torch.from_numpy(moved))
    # the images an end-to-end check picks (first, last and a couple in between) do not contain it ...
    _check(p, x_host, [0, 3, 8, N - 1])
    # ... every image does
    with pytest.raises(AssertionError, match=r'stand-in: stage 1: \d+ of %d elements outside the reference \(first at '
                                             r'\((np\.int64\()?5\)?, ' % (8 * 32 * 32 * 64)):
        _check(p, x_host, range(N))
