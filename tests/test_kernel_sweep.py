"""Kernel sweep: seeded stage lists run through the C-ABI (fastdepth_b200.plan.Plan, no nn.Module), every stage checked
against the per-stage fp64 interval reference (oracle/stage_ref.py) computed from the GPU's OWN input tensors.

A 16-bit element must be a rounding of a value its interval admits, and exactly the round-to-nearest value wherever the
interval holds no rounding midpoint (stage_ref.check); at least half of every single-stage 16-bit tensor must be
determined that way (compositions through a chain run or a fused head: containment, see plan_check.check_plan).
The cases reach the kernel instances, activations, epilogues, cluster modes, channel tails and map edges that the two
MobileNet networks of test_gpu_parity.py never execute.  Every case names the kernels it must run, and the last test
asserts that the sweep as a whole covered every kernel variant."""
import numpy as np
import pytest
import torch

import plan_check as pc
from fastdepth_b200 import plan as fplan
from oracle import stage_ref as sr

pytestmark = pytest.mark.gpu

F16, BF16, F32 = torch.float16, torch.bfloat16, torch.float32
R, R6 = sr.RELU, sr.RELU6
SEEN = []              # (kernel name, activation of its stage, dtype) of every step every case ran
RAN = set()
WORST = {}             # case id -> lowest determined fraction of its strictly checked tensors
COMPOSED = {}          # (case id, what) -> determined fraction of a containment-only composition (chain run, block + head)


# ---------------------------------------------------------------------------------------------------------------------
# stage lists
# ---------------------------------------------------------------------------------------------------------------------
def stem(c0, stride=2, act=R6):
    return dict(kind=sr.STEM, c_in=3, c_out=c0, ksize=3, stride=stride, act=act, upsample=0, skip_src=-1, skip_mode=0)


def blk(c_out, k=3, s=1, act=R6, up=0, skip=-1, mode=0):
    return dict(kind=sr.DWPW, c_in=0, c_out=c_out, ksize=k, stride=s, act=act, upsample=up, skip_src=skip, skip_mode=mode)


def head(act=R):
    return dict(kind=sr.HEAD, c_in=0, c_out=1, ksize=1, stride=1, act=act, upsample=0, skip_src=-1, skip_mode=0)


def link(descs):
    """Fill in every c_in from its producer (c_out, or c_out + c_skip after a concatenation)."""
    ch = 3
    for d in descs:
        d['c_in'] = ch
        ch = d['c_out'] + (descs[d['skip_src']]['c_out'] if d['skip_src'] >= 0 and d['skip_mode'] else 0)
    return descs


def enc_dec(c, acts=(R6, R6, R6, R6, R6, R, R, R), head_act=R):
    """stem s2 -> 3x3 s1 -> 3x3 s2 -> 3x3 s1 -> 3x3 s2 -> 5x5 up + skip(3) -> 5x5 up + skip(1) -> 5x5 up -> head;
    c = (C0, c1, c2, c3, c4, c7): the skip adds fix c5 = c3 and c6 = c1."""
    c0, c1, c2, c3, c4, c7 = c
    a = acts
    return link([stem(c0, 2, a[0]), blk(c1, 3, 1, a[1]), blk(c2, 3, 2, a[2]), blk(c3, 3, 1, a[3]), blk(c4, 3, 2, a[4]),
                 blk(c3, 5, 1, a[5], 1, 3), blk(c1, 5, 1, a[6], 1, 1), blk(c7, 5, 1, a[7], 1), head(head_act)])


def deep(k_bottom, act=R6):
    """5 stride-2 steps to a 1x1 / 1x2 bottom map, then 5 upsampling blocks (two with skips)."""
    return link([stem(16, 2, act), blk(24, 3, 2, act), blk(40, 3, 2, act), blk(56, 3, 2, act), blk(72, 3, 2, act),
                 blk(56, k_bottom, 1, R, 1, 3), blk(40, 5, 1, R6, 1, 2), blk(24, 5, 1, R, 1), blk(16, 3, 1, R6, 1),
                 blk(8, 5, 1, R, 1), head(R)])


def chain(run, act=R, dec_act=R):
    """stem s2 -> 4 x (3x3 s2) -> the run of 3x3 s1 blocks (widths ``run``) -> 5 x (5x5 up) -> head."""
    s = [stem(16, 2, R6), blk(24, 3, 2, R6), blk(40, 3, 2, R6), blk(56, 3, 2, R6), blk(run[0], 3, 2, act)]
    s += [blk(w, 3, 1, act) for w in run[1:]]
    s += [blk(w, 5, 1, dec_act, 1) for w in (64, 40, 24, 16, 8)]
    return link(s + [head(R)])


def chain_skip_source():
    """A 3x3 s1 run at 14x14 whose middle stage is a skip source: the run ends there and chains only 2 layers."""
    return link([stem(16), blk(24, 3, 2), blk(40, 3, 2), blk(64, 3, 2), blk(96, 3, 1, R), blk(128, 3, 1, R),
                 blk(96, 3, 1, R), blk(136, 3, 2), blk(128, 5, 1, R, 1, 5), blk(40, 5, 1, R, 1), blk(24, 5, 1, R, 1),
                 blk(16, 5, 1, R, 1), blk(8, 5, 1, R, 1), head()])


def concat_net():
    return link([stem(24), blk(24, 3, 2), blk(40, 3, 2), blk(56, 5, 1, R, 1, 1, 1), blk(40, 5, 1, R, 1), blk(16, 5, 1, R, 1),
                 head()])


def stem_net(c0, stride, act, last_skip=False):
    if stride == 1:        # full-resolution stem; the last block adds it back (a last block with a skip: no head fold)
        return link([stem(c0, 1, act), blk(40, 3, 2), blk(c0, 5, 1, R, 1, 0 if last_skip else -1), head()])
    return link([stem(c0, 2, act), blk(40, 3, 1), blk(24, 5, 1, R, 1), head()])


# ---------------------------------------------------------------------------------------------------------------------
# weights: representable in the plan dtype, BN calibrated on a probe pass of the reference
# ---------------------------------------------------------------------------------------------------------------------
def _repr(a, dtype):
    a = np.asarray(a, np.float64)
    return (a if dtype == F32 else sr.round_rne(a, dtype)).astype(np.float32)


def _bn(pre, act, rng):
    """fp32 (scale, bias) that put the pre-activation of every channel at a live operating point: ~30 % exact zeros, and
    for ReLU6 a tail beyond the clamp."""
    ax = tuple(range(pre.ndim - 1))
    m, s = pre.mean(axis=ax), pre.std(axis=ax) + 1e-6
    tgt_s = rng.uniform(0.8, 1.2, m.shape) * (2.2 if act == R6 else 1.0)
    tgt_m = 0.5 * tgt_s
    scale = (tgt_s / s).astype(np.float32)
    bias = (tgt_m - m * scale.astype(np.float64)).astype(np.float32)
    return scale, bias


def make_weights(descs, dtype, x, seed):
    """Seeded weights for a stage list, calibrated stage by stage on the reference's point forward of the probe x."""
    rng = np.random.default_rng(seed)
    q = None if dtype == F32 else dtype
    weights, outs, cur = [], [], None
    for d in descs:
        if d['kind'] == sr.STEM:
            w = _repr(rng.standard_normal((d['c_out'], 3, 3, 3)) * 0.4, dtype)
            pre = sr.stem(x, w, np.ones(d['c_out']), np.zeros(d['c_out']), d['stride'], None, eps=0).c
            s, b = _bn(pre, d['act'], rng)
            wt = (None, None, None, w.reshape(d['c_out'], -1), s, b)
            y = sr.quantize(sr.stem(x, w, s, b, d['stride'], d['act'], eps=0), q)
            nxt = y
        elif d['kind'] == sr.DWPW:
            k, ci, co = d['ksize'], d['c_in'], d['c_out']
            taps = _repr(rng.standard_normal((ci, k * k)) * (1.0 / k), dtype)
            dpre = sr.depthwise(cur, taps, np.ones(ci), np.zeros(ci), k, d['stride'], None, eps=0).c
            s1, b1 = _bn(dpre, d['act'], rng)
            dq = sr.quantize(sr.depthwise(cur, taps, s1, b1, k, d['stride'], d['act'], eps=0), q)
            pw = _repr(rng.uniform(-1, 1, (co, ci)) * np.sqrt(3.0 / ci), dtype)
            ppre = dq.c @ pw.T.astype(np.float64)
            s2, b2 = _bn(ppre, d['act'], rng)
            wt = (taps, s1, b1, pw, s2, b2)
            src = d['skip_src']
            skip = outs[src] if src >= 0 else None
            y = sr.quantize(sr.dwpw(cur, wt, d, q, skip, eps=0)['out'], q)
            nxt = sr.concat(y, skip) if (skip is not None and d['skip_mode']) else y
        else:
            w = _repr(np.abs(rng.standard_normal(d['c_in'])) / np.sqrt(d['c_in']), dtype)
            pre = cur.c @ w.astype(np.float64)
            s = np.array([1.0 / (pre.std() + 1e-6)], np.float32)
            b = np.array([2.0 - pre.mean() * float(s[0])], np.float32)
            weights.append((None, None, None, w.reshape(1, -1), s, b))
            return weights
        weights.append(wt)
        outs.append(y)
        cur = sr.Iv(nxt.c)
    raise ValueError('no head')


# ---------------------------------------------------------------------------------------------------------------------
# running a case and checking it (tests/plan_check.py)
# ---------------------------------------------------------------------------------------------------------------------
def run_case(case, descs, dtype, n, h, w, must=(), must_not=(), opts=None, env=None, seed=0, pick=None, x_fn=None,
             w_fn=None, monkeypatch=None, keep=False):
    opts = dict(opts or {})
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, v)
    rng = np.random.default_rng(seed)
    x_host = _repr(rng.uniform(0.0, 1.0, (n, 3, h, w)), dtype)
    if x_fn is not None:
        x_fn(x_host)
    if pick is None:
        pick = list(range(n)) if n <= 8 else sorted({0, n - 1} | set(int(i) for i in rng.choice(n, 2, replace=False)))
    # BN calibration probe: the checked images, plus more images of the same distribution on tiny maps
    probe = x_host[pick[:2]].astype(np.float64)
    if h * w < 64 * 64:
        probe = np.concatenate([probe, _repr(rng.uniform(0.0, 1.0, (6, 3, h, w)), dtype).astype(np.float64)])
    weights = make_weights(descs, dtype, probe, seed + 1)
    if w_fn is not None:
        w_fn(weights)
    names = ['s%d' % i for i in range(len(descs))]
    p = fplan.Plan(descs, weights, names, n, h, w, dtype, 0)
    x = torch.from_numpy(x_host).to(dtype).cuda()
    y = torch.empty((n, 1, h, w), dtype=dtype, device='cuda')
    stream = torch.cuda.current_stream().cuda_stream
    inplace = opts.pop('inplace_skip', 1)
    for k, v in opts.items():
        p.set_option(k, v)
    chk = pc.Checker(case, dtype)
    # pass 1: skip sources kept (inplace_skip 0) -- every materialised stage checked; pass 2: the in-place run's decoders;
    # then the chain's layers and the fused head on their own
    ran = pc.check_plan(p, descs, weights, dtype, x_host, x, y, pick, chk, opts, inplace, stream)
    kern = ' ' + ' '.join(s['kernel'] for steps in ran for s in steps)
    for steps in ran:
        for s in steps:
            SEEN.append((s['kernel'], descs[s['stage']]['act'], dtype))
    for m in must:
        assert m in kern, (case, m, kern)
    for m in must_not:
        assert m not in kern, (case, m, kern)
    COMPOSED.update({(case, what): f for what, f in chk.composed.items()})
    # the activations are live: not mostly zeros, and ReLU6 really clamps somewhere
    assert chk.zeros < 0.5 * chk.n, (case, chk.zeros / chk.n)
    if any(d['act'] == R6 for d in descs[:-1]):
        assert chk.sixes > 0, case
    RAN.add(case)
    WORST[case] = min(chk.fracs)
    if keep:
        return p, x, y
    p.close()
    return y


# ---------------------------------------------------------------------------------------------------------------------
# the cases
# ---------------------------------------------------------------------------------------------------------------------
A1 = (R6, R6, R6, R6, R6, R, R, R)            # 3x3 blocks ReLU6, 5x5 blocks ReLU (the MobileNet pairing)
A2 = (R6, R, R, R, R, R6, R6, R6)             # ... swapped
SMALL = (8, 24, 40, 56, 72, 8)                # HALFK (c_in 8), n_cta padded to 16, fused head after c_out 8
MID = (40, 24, 40, 56, 72, 72)                # 1x8x16 instances, head_kernel<up2x> after c_out 72
WIDE = (64, 136, 200, 264, 520, 40)           # K and N tails at every 64-block, fused head after c_out 40
KNOB = (24, 136, 200, 200, 200, 64)     # cl2 / cl4 / wmc admissible blocks on small maps
B32 = ('block_tc<k3,s1,1x8x16,k32', 'block_tc<k3,s2,2x8x8', 'block_tc<k3,s1,2x8x8', 'block_tc<k5,s1,2x8x8')
B96 = ('block_tc<k3,s1,1x8x16', 'block_tc<k3,s2,1x8x16', 'block_tc<k5,s1,1x8x16')

CASES = {}
for _dt, _dn in ((F16, 'f16'), (BF16, 'bf16')):
    for _a, _an in ((A1, 'a1'), (A2, 'a2')):
        CASES['ed_small_%s_%s' % (_an, _dn)] = dict(descs=lambda a=_a: enc_dec(SMALL, a, R), dtype=_dt, n=3, h=32, w=32,
                                                     must=B32 + ('stem_tc', '+head', '+skip(red)', '+skip', '+tmast'))
        CASES['ed_mid_%s_%s' % (_an, _dn)] = dict(descs=lambda a=_a: enc_dec(MID, a, R6), dtype=_dt, n=3, h=64, w=96,
                                                   must=B96 + ('head_kernel<up2x>',))
CASES.update({
    'ed_wide_96x32_f16': dict(descs=lambda: enc_dec(WIDE, A1), dtype=F16, n=1, h=96, w=32, must=('+head',)),
    'ed_wide_288_bf16': dict(descs=lambda: enc_dec((24, 56, 72, 136, 1032, 24), A2), dtype=BF16, n=1, h=288, w=288,
                             must=('+head',)),
    'ed_small_n200_f16': dict(descs=lambda: enc_dec(SMALL, A2), dtype=F16, n=200, h=32, w=32),
    'deep_1x1_k3_f16': dict(descs=lambda: deep(3), dtype=F16, n=3, h=32, w=32),
    'deep_1x2_k5_bf16': dict(descs=lambda: deep(5, R), dtype=BF16, n=2, h=32, w=64),
    'deep_1x1_k5_f16': dict(descs=lambda: deep(5), dtype=F16, n=2, h=32, w=32),
    'chain_2x1_L2_f16': dict(descs=lambda: chain((64, 160, 160), R), dtype=F16, n=1, h=64, w=32, must=('chain_tc',)),
    'chain_3x5_L5_bf16': dict(descs=lambda: chain((72, 136, 200, 64, 160, 160), R), dtype=BF16, n=3, h=96, w=160,
                              must=('chain_tc<k3,s1,2cta>[5 layers',)),
    'chain_7x13_L8_n67_f16': dict(descs=lambda: chain((128, 96, 128, 200, 64, 40, 136, 72, 128), R6), dtype=F16, n=67,
                                  h=224, w=416, must=('chain_tc<k3,s1,2cta>[8 layers',)),
    'chain_13x2_L2_n200_bf16': dict(descs=lambda: chain((56, 24, 88), R6), dtype=BF16, n=200, h=416, w=64,
                                    must=('chain_tc',)),
    'chain_14x14_L5_f16': dict(descs=lambda: chain((64, 160, 160, 96, 512, 136), R), dtype=F16, n=1, h=448, w=448,
                               must=('chain_tc<k3,s1,2cta>[5 layers',)),
    'chain_wide_falls_back_f16': dict(descs=lambda: chain((64, 520, 96, 64), R), dtype=F16, n=2, h=64, w=64,
                                      must_not=('chain_tc',)),
    'chain_skip_source_bf16': dict(descs=chain_skip_source, dtype=BF16, n=3, h=224, w=224, must=('{stages 4-5}',)),
    'head_c64_relu6_f16': dict(descs=lambda: enc_dec((16, 24, 40, 56, 72, 64), A1, R6), dtype=F16, n=2, h=64, w=64,
                               must=('+head',)),
    'concat_tma_f16': dict(descs=concat_net, dtype=F16, n=3, h=64, w=64, must=('+tmast',)),
    'concat_path0_bf16': dict(descs=concat_net, dtype=BF16, n=3, h=64, w=64, opts=dict(path=0)),
    'concat_lsu_bf16': dict(descs=concat_net, dtype=BF16, n=3, h=64, w=64, opts=dict(tma_epilogue=0)),
    'stem_s1_lastskip_f16': dict(descs=lambda: stem_net(24, 1, R6, True), dtype=F16, n=2, h=32, w=1024,
                                 must=('stem_kernel', 'head_kernel')),
    'stem_c72_f16': dict(descs=lambda: stem_net(72, 2, R6), dtype=F16, n=2, h=32, w=1024, must=('stem_kernel',)),
    'stem_c128_relu_bf16': dict(descs=lambda: stem_net(128, 2, R), dtype=BF16, n=2, h=32, w=1024, must=('stem_kernel',)),
    'stem_c40_tc_bf16': dict(descs=lambda: stem_net(40, 2, R6), dtype=BF16, n=2, h=32, w=1024, must=('stem_tc',)),
    'knob_cl2_pdl_f16': dict(descs=lambda: enc_dec(KNOB, A1), dtype=F16, n=4, h=64, w=64, env={'FD_TC_CLUSTER': '2'},
                             opts=dict(pdl=1), must=(',cl2',)),
    'knob_cl4_sleep_bf16': dict(descs=lambda: enc_dec(KNOB, A2), dtype=BF16, n=4, h=64, w=64, env={'FD_TC_CLUSTER': '4'},
                                opts=dict(wait_sleep_ns=200), must=(',cl4',)),
    'knob_wmc2_teams2_f16': dict(descs=lambda: enc_dec(KNOB, A2), dtype=F16, n=4, h=64, w=64,
                                 env={'FD_TC_CLUSTER': '1', 'FD_TC_WMC': '2', 'FD_TC_DW_TEAMS': '2'}, must=(',wmc2', ',t2')),
    'knob_wmc4_lsu_bf16': dict(descs=lambda: enc_dec(KNOB, A1), dtype=BF16, n=4, h=64, w=64,
                               env={'FD_TC_CLUSTER': '1', 'FD_TC_WMC': '4'}, opts=dict(tma_epilogue=0), must=(',wmc4',)),
    'knob_teams1_f16': dict(descs=lambda: enc_dec(KNOB, A1), dtype=F16, n=4, h=64, w=64, env={'FD_TC_DW_TEAMS': '1'},
                            must_not=(',t2',)),
})
for _dt, _dn in ((F32, 'f32'), (F16, 'f16'), (BF16, 'bf16')):
    CASES['path0_ed_%s' % _dn] = dict(descs=lambda: enc_dec(SMALL, A2), dtype=_dt, n=3, h=32, w=32,
                                      opts=dict(path=0, fold_head=0),
                                      must=('stem_kernel', 'dw_kernel<3>', 'dw_kernel<5>', 'pw_kernel', 'head_kernel'))
    CASES['path0_chain_%s' % _dn] = dict(descs=lambda: chain((64, 160, 160), R), dtype=_dt, n=2, h=64, w=96,
                                         opts=dict(path=0), must=('head_kernel<up2x>',), must_not=('chain_tc',))


@pytest.mark.parametrize('case', list(CASES))
def test_sweep(case, built_lib, monkeypatch):
    c = dict(CASES[case])
    descs = c.pop('descs')()
    run_case(case, descs, monkeypatch=monkeypatch, seed=sum(map(ord, case)), **c)


def test_chain_does_not_carry_non_finite_values_between_images(built_lib, monkeypatch):
    """A chain cluster runs image 66 after image 0 (66 clusters for 67 images).  The last chain layer (160 -> 192) scales
    channels 160..191 by 1000, which stays finite for ordinary images; image 0 has 200x larger inputs and every layer up
    to there is a plain ReLU, so those channels overflow to +Inf for image 0 alone.  The layer writes them into the
    chain's last 64-channel K-block, where image 66's 160 -> 160 layer later reads channels 160..191 with zero taps.
    Its 64 -> 160 layer must have overwritten them first: 0 x Inf = NaN must not reach image 66."""
    descs = chain((64, 160, 160, 192), R)
    for d in descs[:5]:
        d['act'] = R                                        # nothing before the chain clamps image 0's large values

    def big_first(x):
        x[0] *= 200.0

    def hot_tail(weights):
        s, b = weights[7][4], weights[7][5]
        s[160:] *= 1000.0
        b[160:] *= 1000.0
        weights[8][0][160:] = 0.0                           # the decoder after the chain ignores those channels

    p, x, y = run_case('chain_nonfinite_leftover_f16', descs, F16, 67, 96, 96, must=('chain_tc<k3,s1,2cta>[3 layers',),
                       pick=[1, 65, 66], x_fn=big_first, w_fn=hot_tail, monkeypatch=monkeypatch, seed=7, keep=True)
    p.set_option('chain', 1)
    p.set_option('fold_head', 1)
    p.forward(x, y, torch.cuda.current_stream().cuda_stream)
    out = p.stage_tensor(7).float()                          # the chain's output (stages 5..7)
    torch.cuda.synchronize()
    assert torch.isposinf(out[0, ..., 160:]).float().mean() > 0.2     # the premise: image 0 stages +Inf there ...
    assert torch.isfinite(out[0, ..., :160]).all()                    # ... and nothing non-finite elsewhere
    assert torch.isfinite(out[1:]).all()
    p.close()


def test_stage_buffer_above_2gb(built_lib, monkeypatch):
    """N=128 at 512x512 with 40 channels at full resolution and the head unfolded: the last block's buffer is 2.7 GB, so
    its addressing must not wrap at 2^31 bytes."""
    free, _ = torch.cuda.mem_get_info()
    if free < 12 * 2 ** 30:
        pytest.skip('needs ~12 GB of free device memory')
    descs = link([stem(24), blk(40, 3, 2), blk(56, 5, 1, R, 1), blk(40, 5, 1, R, 1), head()])
    run_case('large_2gb_f16', descs, F16, 128, 512, 512, opts=dict(fold_head=0), pick=[0, 127], monkeypatch=monkeypatch,
             seed=11)


INSTANCES = {'k32': lambda k: 'k3,s1,1x8x16,k32' in k, 'k3s1': lambda k: 'k3,s1,1x8x16' in k and ',k32' not in k,
             'k3s1 2x8x8': lambda k: 'k3,s1,2x8x8' in k, 'k3s2': lambda k: 'k3,s2,1x8x16' in k,
             'k3s2 2x8x8': lambda k: 'k3,s2,2x8x8' in k, 'k5s1': lambda k: 'k5,s1,1x8x16' in k,
             'k5s1 2x8x8': lambda k: 'k5,s1,2x8x8' in k}


def test_sweep_coverage():
    """The sweep as a whole ran every fused kernel instance with both activations in both 16-bit dtypes, every cluster
    mode, every epilogue, the chain kernel with both activations and every SIMT kernel in all three dtypes."""
    if not set(CASES) <= RAN:
        pytest.skip('coverage is only meaningful after the whole sweep ran')
    seen = {(k, a, str(d)) for k, a, d in SEEN}
    missing = []
    for inst, match in INSTANCES.items():
        for a in (R, R6):
            for d in (F16, BF16):
                if not any('block_tc<' in k and match(k) and aa == a and dd == str(d) for k, aa, dd in seen):
                    missing.append((inst, a, str(d)))
    names = ' '.join(k for k, _, _ in seen)
    for m in (',cl2', ',cl4', ',wmc2', ',wmc4', ',t2', '+tmast', '+up2x', '+skip(red)', '+skip[', '+head'):
        if m not in names:
            missing.append(m)
    if not any('block_tc' in k and '+tmast' not in k and '+head' not in k for k, _, _ in seen):
        missing.append('LSU epilogue')
    for a in (R, R6):
        if not any('chain_tc' in k and aa == a for k, aa, _ in seen):
            missing.append(('chain_tc', a))
    for kn in ('stem_kernel', 'dw_kernel<3>', 'dw_kernel<5>', 'pw_kernel', 'head_kernel<up2x>'):
        for d in (F32, F16, BF16):
            if not any(k == kn and dd == str(d) for k, _, dd in seen):
                missing.append((kn, str(d)))
    for d in (F32, F16, BF16):
        if not any(k == 'head_kernel' and dd == str(d) for k, _, dd in seen):
            missing.append(('head_kernel', str(d)))
    assert any('stem_tc' in k for k, _, _ in seen)
    assert not missing, missing
    print('lowest determined fraction per case:', sorted(WORST.items(), key=lambda kv: kv[1])[:5])
    print('determined fraction of the containment-only compositions:', sorted(COMPOSED.items(), key=lambda kv: kv[1]))
