// Tile planning of the dense conv kernel (fd_conv_tc.cu), pure host C++ with no CUDA so that it can be unit-tested on a
// machine without a GPU (tests/test_conv_plan.py through fd_debug_conv_plan).
//
// An item is one tile of 128 output pixels (ni images x th rows x tw columns, one 4-D TMA box of the NHWC input per tap and
// 64-channel K-block) times bn output channels.  The planner scores every (tile shape, bn) pair with a small cost model:
//   * wave quantisation: one CTA per SM walks items; the launch takes ceil(items / SMs) item times;
//   * wasted rows: a box that hangs over the map (a 7x7 map in an 8x8 box) still costs the full 128-row MMA;
//   * per 64-channel K-block, the larger of the MMA time (128 x bn x 64 MACs at the dense 16-bit rate, 2048 MAC / clock / SM),
//     the shared-memory reads of the wgmma operands (both warpgroups read their A half and all of B) and the L2 -> SMEM
//     operand traffic (16 KB of A + bn x 128 B of B) at an ESTIMATED 40 B / clock / SM (not measured);
//   * the epilogue: the 16-bit output tile (x4 with the nearest upsample) leaves at an estimated 64 B / clock.
#pragma once

namespace fd {

constexpr int kConvMaxStages = 8;
constexpr int kConvStg = 16384;                       // one epilogue staging tile: 128 px x 64 ch x 2 B
constexpr int kConvSmemBudget = 227 * 1024 - 128;
constexpr int kConvAlignSlack = 1024;
constexpr int kConvBarrierBytes = 256;                // >= sizeof(ConvBarriers)

struct ConvPlanIn {
    int ksize, h_out, w_out, n, c_in, c_out, upsample;
    int n_sms;                 // 0 = 132 (H100 SXM)
    int force_bn;              // 0 = the cost model chooses, else 64 / 128 / 256
    int force_tile;            // -1 = the cost model chooses, else an index into kConvTiles
};
struct ConvPlanOut {
    int ok;
    int ni, th, tw, bn, stages;
    int m_tiles, n_splits, items, waves, kblocks;
    int smem_bytes, useful_permille;
    double cost;
};

// candidate tiles (images x rows x columns, 128 pixels each); small maps take several images per box
constexpr int kConvTiles[][3] = {{1, 8, 16}, {2, 8, 8}, {4, 4, 8}, {8, 4, 4}, {32, 2, 2}};
constexpr int kConvNumTiles = 5;

inline int conv_stage_bytes(int bn) { return 128 * 128 + bn * 128; }

inline ConvPlanOut plan_conv_one(const ConvPlanIn& q, int tile, int bn) {
    ConvPlanOut o{};
    const int ni = kConvTiles[tile][0], th = kConvTiles[tile][1], tw = kConvTiles[tile][2];
    const int sms = q.n_sms > 0 ? q.n_sms : 132;
    o.ni = ni; o.th = th; o.tw = tw; o.bn = bn;
    o.kblocks = (q.c_in + 63) / 64;
    o.m_tiles = ((q.n + ni - 1) / ni) * ((q.h_out + th - 1) / th) * ((q.w_out + tw - 1) / tw);
    o.n_splits = (q.c_out + bn - 1) / bn;
    o.items = o.m_tiles * o.n_splits;
    o.waves = (o.items + sms - 1) / sms;
    const int fixed = 2 * kConvStg + kConvBarrierBytes + kConvAlignSlack;
    o.stages = (kConvSmemBudget - fixed) / conv_stage_bytes(bn);
    if (o.stages > kConvMaxStages) o.stages = kConvMaxStages;
    o.smem_bytes = fixed + o.stages * conv_stage_bytes(bn);
    const double px = (double)q.n * q.h_out * q.w_out;
    o.useful_permille = (int)(1000.0 * px / ((double)o.m_tiles * 128.0));
    o.ok = o.stages >= 2 && o.smem_bytes <= kConvSmemBudget && o.kblocks > 0 && o.items > 0;
    // cost of one item in clocks (see the header comment), times the waves of the persistent launch
    const double mma = 4.0 * bn, smem_rd = (2.0 * 8192 + 2.0 * bn * 128) / 128.0, l2 = (16384.0 + 128.0 * bn) / 40.0;
    double kstep = mma;
    if (smem_rd > kstep) kstep = smem_rd;
    if (l2 > kstep) kstep = l2;
    kstep += 40.0;                                    // barrier hand-shakes per K-block
    const double steps = (double)q.ksize * q.ksize * o.kblocks;
    const double epi = 128.0 * bn * 2.0 * (q.upsample ? 4.0 : 1.0) / 64.0 + 500.0;
    o.cost = (double)o.waves * (steps * kstep + epi);
    return o;
}

inline ConvPlanOut plan_conv(const ConvPlanIn& q) {
    ConvPlanOut best{};
    best.ok = 0;
    if (q.ksize < 1 || q.h_out < 1 || q.w_out < 1 || q.n < 1 || q.c_in < 8 || q.c_out < 8) return best;
    const int bns[3] = {64, 128, 256};
    for (int t = 0; t < kConvNumTiles; ++t) {
        if (q.force_tile >= 0 && t != q.force_tile) continue;
        for (int b = 0; b < 3; ++b) {
            const int bn = bns[b];
            if (q.force_bn ? bn != q.force_bn : (b > 0 && bn / 2 >= q.c_out)) continue;   // no split wider than twice the need
            const ConvPlanOut o = plan_conv_one(q, t, bn);
            if (!o.ok) continue;
            if (!best.ok || o.cost < best.cost * 0.999) best = o;   // ties keep the earlier (larger-row, narrower) choice
        }
    }
    return best;
}

}  // namespace fd
