"""Host-only check of the fused block kernel's shared-memory / pipeline planner (no GPU needed): every block of
the stock and the NetAdapt-pruned network, at 224x224 b64, 480x640 b16 and tiny shapes, must get a plan that fits
the 227 KB of an H100 SM, keeps an item's register accumulator within 128 columns, uses whole 64- or 128-row weight stages and
at most the two staging tiles the kernel alternates between."""
import ctypes

import pytest

from fastdepth_b200 import _lib, synthetic

KEYS = ('ok', 'splits', 'n_cta', 'items', 'kblocks', 's_in', 's_a', 's_b', 'bn', 'nb', 'b_resident', 'n_stg',
        'smem_bytes', 'in_stage_stride', 'cs', 'dw_teams')
STRIDES = (2, 1, 2, 1, 2, 1, 2, 1, 1, 1, 1, 1, 2, 1)


def plan(ks, stride, h, w, n, cin, cout, head=0):
    lib = _lib.load()
    out = (ctypes.c_int * 16)()
    _lib.check(lib.fd_debug_block_plan(ks, stride, h, w, n, cin, cout, head, out, 16))
    return dict(zip(KEYS, out))


def blocks(widths, h, w):
    enc, dec = widths
    hh, ww = h // 2, w // 2
    for i in range(1, 14):
        hh, ww = hh // STRIDES[i], ww // STRIDES[i]
        yield ('conv%d' % i, 3, STRIDES[i], hh, ww, enc[i - 1], enc[i], 0)
    c = enc[13]
    for j, co in enumerate(dec, start=1):
        yield ('decode_conv%d' % j, 5, 1, hh, ww, c, co, 1 if j == 5 else 0)
        c, hh, ww = co, hh * 2, ww * 2


@pytest.mark.parametrize('widths', [synthetic.STOCK_WIDTHS, synthetic.PRUNED_WIDTHS], ids=['stock', 'pruned'])
@pytest.mark.parametrize('shape', [(64, 224, 224), (16, 480, 640), (2, 64, 96), (1, 32, 32), (512, 224, 224)])
def test_every_block_gets_a_valid_plan(built_lib, widths, shape):
    n, h, w = shape
    for name, ks, stride, hh, ww, cin, cout, head in blocks(widths, h, w):
        p = plan(ks, stride, hh, ww, n, cin, cout, head)
        assert p['ok'] == 1, (name, p)
        assert p['smem_bytes'] <= 227 * 1024, (name, p)
        assert p['n_cta'] % 16 == 0 and p['n_cta'] <= 128 and p['bn'] in (64, 128), (name, p)   # register accumulators, wgmma blocks
        assert p['n_cta'] * p['splits'] >= cout and (p['splits'] == 1 or p['n_cta'] % 64 == 0), (name, p)
        assert p['s_in'] >= 1 and 2 <= p['s_a'] <= (6 if p['cs'] > 1 else 4) and p['bn'] * p['nb'] >= p['n_cta'], (name, p)
        assert p['cs'] == 1 or (p['cs'] in (2, 4) and p['splits'] == p['cs'] and p['kblocks'] >= p['cs'] and not head), (name, p)
        assert p['n_stg'] == 0 if head else p['n_stg'] in (1, 2), (name, p)
        if p['b_resident']:
            assert p['splits'] == 1 and p['s_b'] == p['kblocks'] * p['nb'] <= 16


def test_stock_b64_plans_snapshot(built_lib):
    """The metric configuration: high-res blocks keep their weights resident and a deep A ring."""
    p = plan(3, 1, 112, 112, 64, 32, 64)          # conv1
    assert p['b_resident'] == 1 and p['s_a'] == 4 and p['n_stg'] == 2 and p['items'] == 6272
    p = plan(3, 1, 14, 14, 64, 512, 512)          # conv7..11
    # an item's accumulator lives in registers: at most 128 channels, so four splits of one full-width weight stage each
    assert p['splits'] == 4 and p['n_cta'] == 128 and p['bn'] == 128 and p['nb'] == 1
    p = plan(5, 1, 112, 112, 64, 64, 32, head=1)  # decode_conv5 + folded head
    assert p['n_stg'] == 0 and p['splits'] == 1 and p['dw_teams'] == 2       # one K-block, even rings: two depthwise teams
    p = plan(5, 1, 7, 7, 64, 1024, 512)           # decode_conv1: 32 tiles x 4 CTAs in one wave share the 5x5 depthwise half
    assert p['cs'] == 4 and p['splits'] == 4 and p['n_cta'] == 128 and p['dw_teams'] == 1
    p = plan(3, 1, 7, 7, 64, 1024, 1024)          # conv13: paced by its weight stream once the depthwise is shared -> no cluster
    assert p['cs'] == 1
    p = plan(5, 1, 7, 7, 512, 1024, 512)          # same block at batch 512: more than one wave -> no tile sharing
    assert p['cs'] == 1


def test_planner_invariants_on_random_blocks(built_lib):
    """Property test: ANY block the fused kernel may be asked to run gets a plan that honours the kernel's assumptions
    (the assumptions are the ones block_tc_kernel relies on without checking)."""
    from hypothesis import given, settings, strategies as st

    @settings(max_examples=400, deadline=None)
    @given(ks_stride=st.sampled_from([(3, 1), (3, 2), (5, 1)]), cin=st.integers(1, 160).map(lambda v: 8 * v),
           cout=st.integers(1, 160).map(lambda v: 8 * v), hw=st.sampled_from([(7, 7), (14, 14), (28, 28), (56, 56), (112, 112), (15, 20), (30, 40), (3, 2)]),
           n=st.sampled_from([1, 2, 3, 16, 64, 200]), head=st.booleans())
    def check(ks_stride, cin, cout, hw, n, head):
        ks, stride = ks_stride
        if head and cout > 64:
            head = False                                   # the folded head needs the whole block in one item of <= 64 channels
        p = plan(ks, stride, hw[0], hw[1], n, cin, cout, int(head))
        ctx = (ks, stride, cin, cout, hw, n, head, p)
        assert p['ok'] == 1, ctx
        assert p['smem_bytes'] <= 227 * 1024, ctx
        assert p['n_cta'] % 16 == 0 and p['n_cta'] * p['splits'] >= cout, ctx
        assert p['splits'] == 1 or p['n_cta'] % 64 == 0, ctx                       # a TMA store box must not reach into the next split
        assert p['n_cta'] <= 128 and p['bn'] in (64, 128) and p['bn'] * p['nb'] >= p['n_cta'] > p['bn'] * (p['nb'] - 1), ctx
        assert p['kblocks'] == (cin + 63) // 64 and 2 <= p['s_a'] <= (6 if p['cs'] > 1 else 4) and 1 <= p['s_in'] <= 6, ctx
        # cluster mode: one split per CTA of the cluster, every CTA owns a K-block and a non-empty split, two accumulators
        assert p['cs'] == 1 or (p['cs'] in (2, 4) and p['splits'] == p['cs'] and p['kblocks'] >= p['cs'] and
                                p['n_cta'] * (p['cs'] - 1) < cout and not head), ctx
        assert p['s_in'] >= 2 or (p['kblocks'] == 1 and p['items'] <= 132), ctx
        assert 1 <= p['s_b'] <= 16 and (not p['b_resident'] or p['s_b'] == p['kblocks'] * p['nb']), ctx
        if head:
            assert p['n_stg'] == 0 and p['splits'] == 1, ctx
        else:
            assert p['n_stg'] in (1, 2), ctx                                       # the kernel alternates between at most two tiles
        assert p['cs'] == 1 or p['items'] <= 132, ctx                              # tile-sharing clusters: one wave only
        assert p['dw_teams'] in (1, 2) and (p['dw_teams'] == 1 or (p['cs'] == 1 and p['s_in'] % 2 == 0 and p['s_a'] % 2 == 0)), ctx

    check()
