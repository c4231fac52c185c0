"""Host-only check (no GPU) that the fused block planner sizes the per-K-block depthwise parameter block the kernel
reads: {taps, [64] fp32 scale, [64] fp32 bias} with [9][64] 16-bit taps for 3x3 blocks and, for 5x5 blocks, fp32 taps
as [5 kernel rows][32 lanes][6 pairs] (the 5x5 depthwise loop reads a lane's kernel row as three 16-byte words)."""
import pytest

from test_block_plan import plan


@pytest.mark.parametrize('ks,stride,tile_hw,taps_bytes', [(3, 1, (56, 56), 9 * 64 * 2), (3, 2, (56, 56), 9 * 64 * 2),
                                                           (3, 1, (7, 7), 9 * 64 * 2), (5, 1, (56, 56), 5 * 32 * 48),
                                                           (5, 1, (7, 7), 5 * 32 * 48)])
def test_input_stage_holds_tile_and_parameter_block(built_lib, ks, stride, tile_hw, taps_bytes):
    h, w = tile_hw
    p = plan(ks, stride, h, w, 64, 128, 64)
    ni, th, tw = (2, 8, 8) if (h <= 8 and w <= 8) else (1, 8, 16)
    tile = ni * ((th - 1) * stride + ks) * ((tw - 1) * stride + ks) * 128
    dwp = taps_bytes + 2 * 64 * 4
    assert p['ok'] == 1
    assert p['in_stage_stride'] == (tile + dwp + 127) // 128 * 128, p
