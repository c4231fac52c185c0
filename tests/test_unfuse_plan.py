"""Planning of the two-step route of a 16-bit DWPW stage (plan option ``unfuse``), without a GPU.

The pointwise half runs as a 1x1 step of conv_tc_kernel over the stage's depthwise intermediate.  A stage without an
upsample is rows of a matrix, planned as one image of rows / 16 x 16 pixels when 16 divides the rows; an upsampling stage
keeps its map because its tiles leave through the four views of the 2x map.  The automatic rule takes a stage when the
block planner would split it 8 ways or more over the output channels or run it on a tile-sharing cluster; both planners
are asked here for the stock and pruned 7x7 stages."""
import ctypes

import pytest

from fastdepth_b200 import _lib

CONV_KEYS = ('ok', 'ni', 'th', 'tw', 'bn', 'stages', 'm_tiles', 'n_splits', 'items', 'waves', 'kblocks', 'smem_bytes',
             'useful_permille', 'cost', 'stage_bytes')
BLOCK_KEYS = ('ok', 'splits', 'n_cta', 'items', 'kblocks', 's_in', 's_a', 's_b', 'bn', 'nb', 'b_resident', 'n_stg',
              'smem_bytes', 'in_stage_stride', 'cs', 'dw_teams')
SMEM_MAX = 227 * 1024


@pytest.fixture(scope='module')
def lib():
    return _lib.load()


def pw(lib, h, w, n, c_in, c_out, upsample=0, n_sms=132):
    out = (ctypes.c_int * 16)()
    assert lib.fd_debug_pw_plan(h, w, n, c_in, c_out, upsample, n_sms, out, 16) == 0
    return dict(zip(CONV_KEYS, out))


def block(lib, k, stride, h, w, n, c_in, c_out):
    out = (ctypes.c_int * 16)()
    assert lib.fd_debug_block_plan(k, stride, h, w, n, c_in, c_out, 0, out, 16) == 0
    return dict(zip(BLOCK_KEYS, out))


# (stage, batch) -> (ni, th, tw, bn, ring depth, tiles, n-splits); conv12 512->1024 and conv13 1024->1024 write a 7x7 map,
# decode_conv1 1024->512 upsamples it
STOCK = {
    ('conv12', 64): (1, 8, 16, 256, 4, 25, 4), ('conv13', 64): (1, 8, 16, 256, 4, 25, 4),
    ('decode_conv1', 64): (2, 8, 8, 128, 6, 32, 4),
    ('conv12', 32): (1, 8, 16, 128, 6, 13, 8), ('conv13', 32): (1, 8, 16, 128, 6, 13, 8),
    ('decode_conv1', 32): (2, 8, 8, 64, 8, 16, 8),
    ('conv12', 1): (1, 8, 16, 64, 8, 1, 16), ('conv13', 1): (1, 8, 16, 64, 8, 1, 16),
    ('decode_conv1', 1): (1, 8, 16, 64, 8, 1, 8),
}
SHAPES = {'conv12': (512, 1024, 0), 'conv13': (1024, 1024, 0), 'decode_conv1': (1024, 512, 1)}


@pytest.mark.parametrize('stage,n', list(STOCK))
def test_pointwise_step_of_the_stock_7x7_stages(lib, stage, n):
    c_in, c_out, up = SHAPES[stage]
    p = pw(lib, 7, 7, n, c_in, c_out, up)
    assert p['ok'] == 1
    assert (p['ni'], p['th'], p['tw'], p['bn'], p['stages'], p['m_tiles'], p['n_splits']) == STOCK[(stage, n)]
    assert p['items'] == p['m_tiles'] * p['n_splits'] and p['waves'] == 1
    assert p['kblocks'] == c_in // 64
    assert p['stage_bytes'] == 128 * 128 + p['bn'] * 128
    assert p['smem_bytes'] <= SMEM_MAX
    if not up and (n * 49) % 16 == 0:
        # rows of a matrix: 3136 rows are 24.5 tiles of 128, against 32 boxes of 2 x 8 x 8 that a 7x7 map fills to 77 %
        assert p['m_tiles'] == -(-n * 49 // 128) and p['useful_permille'] >= 940
    else:
        assert p['useful_permille'] in (765, 382)


def test_channel_tails(lib):
    # c_in mod 64 in {8, 24, 40}: the last K-block is zero-filled by the tensor map; c_out tails: the last split is clipped
    for c_in, kb in ((72, 2), (24, 1), (1000, 16)):
        assert pw(lib, 7, 7, 64, c_in, 512)['kblocks'] == kb
    for c_out in (8, 40, 72, 136, 264):
        p = pw(lib, 14, 14, 4, 128, c_out, 1)
        assert p['ok'] == 1 and p['n_splits'] == -(-c_out // p['bn'])
        assert p['bn'] // 2 < c_out or p['bn'] == 64           # no split wider than twice the need
    # 16 does not divide 3 * 5 * 5 rows: the map stays (one 1 x 8 x 16 box per image; four images of rows would be one tile)
    assert pw(lib, 5, 5, 3, 64, 64)['m_tiles'] == 3 and pw(lib, 4, 4, 8, 64, 64)['m_tiles'] == 1
    assert pw(lib, 7, 7, 64, 4, 64)['ok'] == 0


def test_rule_inputs_from_the_block_planner(lib):
    """What the automatic rule reads: output-channel splits and the cluster size of the fused plan."""
    for n in (64, 32):
        assert block(lib, 3, 2, 7, 7, n, 512, 1024)['splits'] == 8             # conv12
        assert block(lib, 3, 1, 7, 7, n, 1024, 1024)['splits'] == 8            # conv13
        assert block(lib, 5, 1, 7, 7, n, 1024, 512)['cs'] == 4                 # decode_conv1
    # stock stages that stay fused at b64: conv6 (4 splits), decode_conv2 (2 splits), and conv7 at 15x20 (b16 480x640)
    for args in ((3, 2, 14, 14, 64, 256, 512), (5, 1, 14, 14, 64, 512, 256), (3, 1, 15, 20, 16, 512, 512)):
        b = block(lib, *args)
        assert b['splits'] <= 4 and b['cs'] == 1, args
    # pruned 7x7 encoder stages split 4 ways and stay fused; its decode_conv1 (512 -> 200) is planned on a 4-CTA cluster
    assert block(lib, 3, 2, 7, 7, 64, 328, 480)['splits'] == 4 and block(lib, 3, 2, 7, 7, 64, 328, 480)['cs'] == 1
    assert block(lib, 3, 1, 7, 7, 64, 480, 512)['splits'] == 4 and block(lib, 3, 1, 7, 7, 64, 480, 512)['cs'] == 1
    assert block(lib, 5, 1, 7, 7, 64, 512, 200)['cs'] == 4
