// Shared-memory / pipeline planning of the fused block kernel (pure host C++, no CUDA) so that it can be
// unit-tested on a machine without a GPU (tests/test_block_plan.py through fd_debug_block_plan).
#pragma once

namespace fd {

constexpr int kPlanKblk = 64;
constexpr int kPlanAStage = 128 * 128;       // one A operand stage: 128 rows x 64 x 2 B
constexpr int kPlanStg = 16384;              // one epilogue staging tile: 128 px x 64 ch x 2 B
constexpr int kPlanMaxIn = 6, kPlanMaxA = 4, kPlanMaxB = 16;
constexpr int kPlanMaxACluster = 6;          // cluster mode: the A ring is filled by several CTAs at once and wants >= cluster size stages
// An item's accumulator lives in the registers of the two consumer warpgroups (64 pixel rows each): n_cta / 2 fp32 registers per
// thread, so 128 output channels per item is the most the register file leaves room for next to the other roles.
constexpr int kPlanMaxNcta = 128;
// Bytes of the taps in a K-block's depthwise parameter block {taps, [64] fp32 scale, [64] fp32 bias}.
//   3x3: [9][64] taps in the storage dtype.
//   5x5: [5 kernel rows][32 lanes][6 fp32 pairs] -- per lane (channel pair) and kernel row the 5 tap pairs (kx = 0..4) and one
//        zero pair.  The values are rounded to the storage dtype, so the products stay exact.  The depthwise loop reads a lane's
//        kernel row with three 16-byte loads where it is used, since 25 taps held in registers do not fit beside the
//        accumulators under the kernel's register cap; the 48-byte lane stride keeps every quarter-warp's 16-byte loads on
//        distinct banks.
// (The kernel reads this too, hence the device qualifier under CUDA.)
#ifdef __CUDACC__
__host__ __device__
#endif
constexpr int dw_taps_bytes(int ksize) { return ksize == 5 ? 5 * 32 * 48 : ksize * ksize * 64 * 2; }
#ifndef FD_PLAN_SMALL_SMEM
// everything that needs 1 KB alignment sits in front of the 128-byte-granular input stages (see the kernel's carve-up): ONE alignment
// slack, and the budget is the whole 227 KB an H100 block may opt into, minus a small margin
constexpr int kPlanSmemBudget = 227 * 1024 - 128;
constexpr int kPlanAlignSlack = 1024;
#else
constexpr int kPlanSmemBudget = 224 * 1024;
constexpr int kPlanAlignSlack = 2048;
#endif

struct BlockPlanIn {
    int ksize, stride, tile;     // tile: 0 = 1 image x 8 x 16, 1 = 2 images x 8 x 8
    int c_in, c_out, n_tiles;    // n_tiles: 128-pixel tiles of the whole problem
    int head;                    // decode_conv6 folded into the epilogue
    int barrier_bytes;           // sizeof(TcBarriers)
    int max_n_cta;               // 0 = no limit; experiments: cap the output channels per item (FD_TC_MAX_NCTA)
    int n_sms;                   // SMs of the device (one CTA each); 0 = 132 (H100 SXM)
    int even_rings;              // 1: input and A rings get an even number of stages (two depthwise teams on alternate steps); 0 / 2: no constraint
    int cluster_multiwave;       // bring-up only (FD_TC_CLUSTER_MULTIWAVE=1): admit tile-sharing clusters on multi-wave launches
    int cluster;                 // 0 = the cost model may choose cluster mode, 1 = never, 2 / 4 = force that cluster size when the
                                 // block admits it (plan option "cluster", FD_TC_CLUSTER)
};
struct BlockPlanOut {
    int ok;
    int kblocks, cin_pad, splits, n_cta, cpad_all, items;
    int in_stage_bytes, dwp_bytes, in_stage_stride;
    int s_in, s_a, s_b, bn, nb, b_resident, b_stage_bytes;
    int n_stg;                   // epilogue staging tiles: 2 (one tile's TMA store overlaps filling the other), 1, or 0 (folded head)
    int dw_teams;                // 2: two depthwise teams of four warps on alternate K-block steps (needs even s_in and s_a), else 1
    int cs;                      // cluster size: 1, or 2 / 4 CTAs that share one tile -- CTA r computes the depthwise half of the
                                 // K-blocks kb % cs == r, broadcasts its operand tiles to the others through DSMEM and runs the MMAs
                                 // of output-channel split r (splits == cs)
    int smem_bytes;
};

// Shared-memory search for one choice of (splits, n_cta): ring depths / weight stage width / staging tiles, scored by what
// matters for the block at hand (stride-2 blocks stage 72 KB of input per K-block and leave little room; single-K-block
// blocks want a deep A ring so that the depthwise warps never wait for the consumers).
inline bool plan_block_smem(const BlockPlanIn& q, BlockPlanOut& p) {
    const int splits = p.splits;
    const int sms = q.n_sms > 0 ? q.n_sms : 132;
    const int fixed = q.barrier_bytes + kPlanAlignSlack + (q.head ? 3 : 2) * p.cpad_all * 4;
    const int total = kPlanSmemBudget - fixed;
    long best = -(1L << 60);
    bool found = false;
    const int bn_top = (p.n_cta + 63) / 64 * 64;                 // whole 64-column wgmma blocks (rows past c_out load as zeros)
    const int per_cta_kb = p.cs > 1 ? (p.kblocks + p.cs - 1) / p.cs : p.kblocks;      // K-blocks whose input tile THIS CTA loads
    for (int s_a = p.cs > 1 ? kPlanMaxACluster : kPlanMaxA; s_a >= 2; --s_a)
        for (int n_stg = q.head ? 0 : 2; n_stg >= (q.head ? 0 : 1); --n_stg) {
            if (q.even_rings == 1 && p.cs == 1 && (s_a & 1)) continue;
            const int avail = total - s_a * kPlanAStage - n_stg * kPlanStg;
            for (int bn = bn_top; bn >= 64; bn -= 64) {
                const int nb = (p.n_cta + bn - 1) / bn;
                const int w_all = p.kblocks * nb * bn * 128;
                const bool can_res = splits == 1 && bn == bn_top && p.kblocks * nb <= kPlanMaxB && w_all <= 64 * 1024;
                for (int res = can_res ? 1 : 0; res >= 0; --res)
                    for (int s_b = res ? p.kblocks * nb : 6; s_b >= (res ? p.kblocks * nb : 2); --s_b) {
                        if (!res && s_b > p.kblocks * nb && s_b > 2) continue;
                        const int left = avail - s_b * bn * 128;
                        if (left < 0) continue;
                        int s_in = left / p.in_stage_stride;
                        if (s_in > kPlanMaxIn) s_in = kPlanMaxIn;
                        if (q.even_rings == 1 && p.cs == 1 && s_in >= 2) s_in &= ~1;
                        if (q.even_rings && p.cs == 1 && s_in > 4) s_in &= ~1;        // beyond four stages depth buys nothing: keep the ring even
                        if (s_in < 2 && !(s_in == 1 && p.kblocks == 1 && p.items <= sms)) continue;
                        if (p.cs > 1 && s_in > per_cta_kb + 1) s_in = per_cta_kb + 1 < 2 ? 2 : per_cta_kb + 1;
                        // weight ring depth in K-blocks: below 2 the MMA of K-block k+1 waits for a weight load that can only
                        // start when the MMA of K-block k has finished
                        const int b_ahead2 = res ? 4 : (2 * s_b / nb > 4 ? 4 : 2 * s_b / nb);      // in half K-blocks, capped at 2 K-blocks
                        long score = (long)bn * 100 + (s_in > 4 ? 4 : s_in) * 2500 + s_a * (p.kblocks <= 2 ? 1500 : 400) + n_stg * 2800 +
                                     (res ? 1000 : 0) + b_ahead2 * 1800;
                        if (p.cs > 1)        // every CTA of the cluster produces operand tiles concurrently: one stage each, plus slack
                            score = (long)bn * 100 + (s_in > 3 ? 3 : s_in) * 1500 + (s_a > p.cs + 1 ? p.cs + 1 : s_a) * 4000 + n_stg * 2800 +
                                    b_ahead2 * 2500;
                        if (score > best) {
                            found = true; best = score;
                            p.s_a = s_a; p.n_stg = n_stg; p.s_in = s_in; p.s_b = s_b; p.bn = bn; p.b_resident = res;
                        }
                    }
            }
        }
    if (!found) return false;
    p.nb = (p.n_cta + p.bn - 1) / p.bn;
    p.b_stage_bytes = p.bn * 128;
    p.smem_bytes = p.s_a * kPlanAStage + p.s_b * p.b_stage_bytes + p.s_in * p.in_stage_stride + p.n_stg * kPlanStg + fixed;
    return true;
}

// two depthwise teams: asked for (even_rings 1 = wherever even rings fit, 2 = only where the plan is even anyway and the block
// has a single K-block), not on a tile-sharing cluster, and the rings really are even
inline int plan_dw_teams(const BlockPlanIn& q, const BlockPlanOut& p) {
    return (q.even_rings && p.cs == 1 && p.s_in >= 2 && !(p.s_in & 1) && !(p.s_a & 1) && (q.even_rings == 1 || p.kblocks == 1)) ? 2 : 1;
}

inline BlockPlanOut plan_block(const BlockPlanIn& q) {
    BlockPlanOut p{};
    const long sms = q.n_sms > 0 ? q.n_sms : 132;
    const int NI = q.tile ? 2 : 1, TH = 8, TW = q.tile ? 8 : 16;
    const int IH = (TH - 1) * q.stride + q.ksize, IW = (TW - 1) * q.stride + q.ksize;
    p.kblocks = (q.c_in + kPlanKblk - 1) / kPlanKblk;
    p.cin_pad = p.kblocks * kPlanKblk;
    p.in_stage_bytes = NI * IH * IW * 128;
    p.dwp_bytes = dw_taps_bytes(q.ksize) + 512;
    p.in_stage_stride = (p.in_stage_bytes + p.dwp_bytes + 127) / 128 * 128;
    // Split the output channels into items (each item recomputes the depthwise half for its 128 pixels and reloads the
    // input tile, so splitting is not free).  Candidates: n_cta <= 128 (the register accumulators), multiples of 64 when there
    // is more than one split (the epilogue moves whole [128 px][64 ch] tiles and must not touch a neighbouring split's columns).
    // Candidates are tried in the order of their modelled kernel time
    //     rounds over the SMs x (K-blocks x max(depthwise, MMA, L2 -> SM operand traffic) + epilogue of the item)
    // until one fits shared memory.  The per-K-block terms are estimates from H100 figures, not measurements:
    //   depthwise  k*k taps x 64 channels x 128 pixels on the 128 fp32 lanes of an SM, doubled for the loads, conversions
    //              and stores that issue beside the FMAs;
    //   MMA        128 x n_cta x 64 MACs at 2048 dense 16-bit MAC/clk per SM (989 TFLOP/s over 132 SMs at 1.83 GHz);
    //   L2 -> SM   the input tile and the weight stage of every active CTA at ~3000 B/clk for the whole chip (about 5.5 TB/s);
    //   epilogue   ~8 cycles per output channel of the item (registers -> staging tile -> TMA store, not overlapped with the
    //              item's MMAs), plus ~100 cycles of hand-shakes per K-block.
    const int cout_pad = (q.c_out + 15) / 16 * 16;
    struct Cand { long t; int sp, nc, cs; };
    Cand cands[12];
    int n_cands = 0;
    if (cout_pad <= 64 || q.head) {
        cands[n_cands++] = Cand{0, 1, cout_pad, 1};
    } else {
        const long dw_c = 2L * q.ksize * q.ksize * 64;
        for (int n_cta = kPlanMaxNcta; n_cta >= 64; n_cta -= 64) {
            int sp = (cout_pad + n_cta - 1) / n_cta, nc = n_cta;
            if (sp == 1) nc = cout_pad;                              // a single split needs no 64-alignment
            if (sp == 1 && cout_pad > kPlanMaxNcta) continue;
            if (sp == 1 && n_cta - 64 >= cout_pad) continue;         // same plan as the next smaller candidate
            if (q.max_n_cta > 0 && nc > q.max_n_cta && !(sp == 1 && cout_pad <= kPlanMaxNcta)) continue;
            const long items = (long)q.n_tiles * sp;
            const long rounds = (items + sms - 1) / sms;
            const long active = items < sms ? items : sms;
            const long mma_c = 4L * nc;
            const long l2_c = active * (p.in_stage_bytes + 128L * nc) / 3000;
            long kb_c = dw_c > mma_c ? dw_c : mma_c;
            if (l2_c > kb_c) kb_c = l2_c;
            const long t = rounds * (p.kblocks * (kb_c + 100) + 8L * nc);
            int at = n_cands++;
            while (at > 0 && cands[at - 1].t > t) { cands[at] = cands[at - 1]; --at; }
            cands[at] = Cand{t, sp, nc, 1};
        }
        // Cluster mode: cs CTAs share one tile.  Without it every output-channel split recomputes the whole depthwise half;
        // with it the depthwise work of a tile is divided by cs and the K loop runs at the MMA's pace, at the price of the
        // operand hand-over and the cluster's start-up.  The automatic choice is limited to the 7x7 maps with a 5x5 depthwise,
        // where the depthwise half is the largest share of a K-block; the plan option / FD_TC_CLUSTER = 2 | 4 forces it
        // wherever the block admits it (the bitwise tests do).
        for (int cs = 2; cs <= 4 && q.cluster != 1; cs *= 2) {
            if (q.cluster > 1 && q.cluster != cs) continue;
            if (q.cluster == 0 && !(q.ksize == 5 && q.tile == 1 && cs == 4)) continue;
            // one wave only (every CTA runs exactly one item): forced multi-wave launches of this mode stopped making progress
            // on the metric batch in bring-up (a timing-dependent stall between the A-ring hand-over and the item pipeline that
            // the instrumented build does not show); the single-wave case is the one the cost model wants anyway
            if ((long)q.n_tiles * cs > sms && !q.cluster_multiwave) continue;
            const int nc = ((cout_pad + cs - 1) / cs + 63) / 64 * 64;
            if (nc > kPlanMaxNcta || nc * (cs - 1) >= cout_pad || p.kblocks < cs) continue;      // every CTA owns >= 1 K-block and a non-empty split
            const long n_cl = sms / cs;
            const long rounds = ((long)q.n_tiles + n_cl - 1) / n_cl;
            const long mma_c = 4L * nc;
            const long active = (q.n_tiles < n_cl ? q.n_tiles : n_cl) * cs;
            const long l2_c = active * (p.in_stage_bytes / cs + 128L * nc) / 3000;
            long kb_c = dw_c / cs > mma_c ? dw_c / cs : mma_c;
            if (l2_c > kb_c) kb_c = l2_c;
            long t = rounds * (p.kblocks * (kb_c + 150) + 8L * nc) + 1500;               // + estimated cluster start-up and hand-over
            if (q.cluster > 1) t = -1;                                                   // forced
            int at = n_cands++;
            while (at > 0 && cands[at - 1].t > t) { cands[at] = cands[at - 1]; --at; }
            cands[at] = Cand{t, cs, nc, cs};
        }
    }
    for (int i = 0; i < n_cands; ++i) {
        p.splits = cands[i].sp; p.n_cta = cands[i].nc; p.cs = cands[i].cs;
        p.items = q.n_tiles * p.splits;
        p.cpad_all = p.n_cta * p.splits;
        if (plan_block_smem(q, p)) { p.ok = 1; p.dw_teams = plan_dw_teams(q, p); return p; }
    }
    p.ok = 0;
    return p;
}

}  // namespace fd
