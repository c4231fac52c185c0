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
//
// Transposed conv (DECONV) and unpool + conv (UPCONV) stages are four stride-1 convs at the input resolution, one per output
// parity (ry, rx): phase 2 ry + rx reads input (Y + dy, X + dx) for a box of (dy, dx) offsets with its own weight taps.  Phases
// differ in cost (9 / 6 / 6 / 4 taps for k = 5), so an item is (tile, bn split, phase group): either one phase per item or the
// two diagonal pairs {00, 11} and {01, 10}.  Items are ordered group-major, heaviest group first, and the cost model takes the
// makespan of the persistent grid's static round-robin assignment over the real per-item tap counts.
//
// The split-TF32 instance (tf32x3: an fp32 1x1, k x k or phased conv as three TF32 products per term, fd_conv_tc.cu) has an fp32
// operand format: one 128-byte row holds 32 fp32 channels, so a K-block is 32 channels, and a stage holds the A box (16 KB)
// plus two B boxes, the weights' TF32 high and low parts (2 x bn x 128 B).  Its MMA time counts three TF32 products per MAC
// at the dense TF32 rate (1024 MAC / clock / SM, half the 16-bit rate); the consumers read A with ordinary shared loads (to
// split it in registers) and every wgmma reads one of the two B boxes; the fp32 output tile is twice as many bytes.
#pragma once

namespace fd {

constexpr int kConvMaxStages = 8;
constexpr int kConvStg = 16384;                       // one epilogue staging tile: 128 px x 64 ch x 2 B
constexpr int kConvSmemBudget = 227 * 1024 - 128;
constexpr int kConvAlignSlack = 1024;
constexpr int kConvBarrierBytes = 256;                // >= sizeof(ConvBarriers)

// stage kinds of the conv kernel (the fd_stage_kind values)
constexpr int kConvKindConv = 3, kConvKindDeconv = 4, kConvKindUpconv = 5;

// one phase of a conv: taps [tap0, tap0 + ny * nx) of the repacked weights [c_out][taps][c_in], tap tap0 + iy * nx + ix reads
// input (Y + dy0 + iy, X + dx0 + ix) for conv-resolution pixel (Y, X)
struct ConvPhase { int tap0, ny, nx, dy0, dx0; };

// weight tap t (per axis, 0..k-1) of output parity r at input offset d; p = (k - 1) / 2.
//   DECONV (ConvTranspose2d(k, 2, p, 1), weights [c_in][c_out][k][k], no flip): t = r + p - 2 d
//   UPCONV (zero-insert x2, then Conv2d(k, 1, p), weights [c_out][c_in][k][k]): t = 2 d + p - r
inline int convt_tap(int kind, int k, int r, int d) {
    const int p = (k - 1) / 2;
    return kind == kConvKindDeconv ? r + p - 2 * d : 2 * d + p - r;
}

// the contiguous range [d0, d0 + n) of input offsets of parity r (the taps with t = r + p mod 2)
inline void convt_axis(int kind, int k, int r, int* d0, int* n) {
    const int p = (k - 1) / 2;
    int lo = 1 << 20, hi = -(1 << 20);
    for (int t = 0; t < k; ++t) {
        if ((t - r - p) & 1) continue;
        const int d = kind == kConvKindDeconv ? (r + p - t) / 2 : (r + t - p) / 2;
        lo = d < lo ? d : lo; hi = d > hi ? d : hi;
    }
    *d0 = lo; *n = hi - lo + 1;
}

// the phase table of a stage: CONV is one phase, the k x k square in (ky, kx) order; DECONV / UPCONV are four, phase
// 2 ry + rx, their taps stored phase-major and sorted by (dy, dx).  Returns the number of phases.
inline int conv_phases(int kind, int k, ConvPhase ph[4]) {
    const int p = (k - 1) / 2;
    if (kind == kConvKindConv) { ph[0] = ConvPhase{0, k, k, -p, -p}; return 1; }
    int tap0 = 0;
    for (int q = 0; q < 4; ++q) {
        convt_axis(kind, k, q >> 1, &ph[q].dy0, &ph[q].ny);
        convt_axis(kind, k, q & 1, &ph[q].dx0, &ph[q].nx);
        ph[q].tap0 = tap0;
        tap0 += ph[q].ny * ph[q].nx;
    }
    return 4;
}

struct ConvPlanIn {
    int ksize, h_out, w_out, n, c_in, c_out, upsample;   // h_out / w_out: the conv resolution (a DECONV's input map)
    int n_sms;                 // 0 = 132 (H100 SXM)
    int force_bn;              // 0 = the cost model chooses, else 64 / 128 / 256
    int force_tile;            // -1 = the cost model chooses, else an index into kConvTiles
    int kind;                  // kConvKind*; 0 = CONV
    int force_group;           // phases per item of a DECONV / UPCONV stage: 0 = the cost model chooses, 1 = one, 2 = pairs
    int tf32x3;                // 1: the split-TF32 instance (fp32 operands; 1x1 or k in {3, 5} CONV, DECONV, UPCONV)
};
struct ConvPlanOut {
    int ok;
    int ni, th, tw, bn, stages;
    int m_tiles, n_splits, items, waves, kblocks;
    int smem_bytes, useful_permille;
    double cost;
    int n_phases, groups;       // items = m_tiles * n_splits * groups
    ConvPhase ph[4];
    int group_ph[4][2];         // phases of group g, in order; -1 = none
};

// candidate tiles (images x rows x columns, 128 pixels each); small maps take several images per box
constexpr int kConvTiles[][3] = {{1, 8, 16}, {2, 8, 8}, {4, 4, 8}, {8, 4, 4}, {32, 2, 2}};
constexpr int kConvNumTiles = 5;

// A 1x1 conv without an upsample reads and writes rows of a matrix, M = n * h * w of them, and no box ever looks at a
// neighbour: when 16 divides M the rows are presented as ONE image of M / 16 rows x 16 columns, so that 1 x 8 x 16 tiles cover
// them with at most one partial tile (a 7x7 map in 2 x 8 x 8 boxes is 77 % used).  Returns false when the geometry stays.
inline bool conv_flat_rows(int upsample, int* n, int* h, int* w) {
    const long long m = (long long)*n * *h * *w;
    if (upsample || m % 16 || m / 128 >= (1 << 18)) return false;     // (the kernel's item decode divides numbers below 2^20)
    *n = 1; *h = (int)(m / 16); *w = 16;
    return true;
}

inline int conv_stage_bytes(int bn) { return 128 * 128 + bn * 128; }
// the split-TF32 pointwise instance: A {32 fp32 ch x 128 px} + B high + B low {32 fp32 ch x bn}
inline int conv_stage_bytes_tf32x3(int bn) { return 128 * 128 + 2 * bn * 128; }
// bn 256 is not offered: 128 accumulators plus the 32 registers of a stage's split A fragments exceed the 168 registers a
// thread of the 288-thread CTA may hold (ptxas serialises the wgmmas and spills)
constexpr int kConvTf32x3MaxBn = 128;

inline ConvPlanOut plan_conv_one(const ConvPlanIn& q, int tile, int bn, int per_item) {
    ConvPlanOut o{};
    const int kind = q.kind ? q.kind : kConvKindConv;
    o.n_phases = conv_phases(kind, q.ksize, o.ph);
    for (int g = 0; g < 4; ++g) o.group_ph[g][0] = o.group_ph[g][1] = -1;
    if (o.n_phases == 1) {
        o.groups = 1; o.group_ph[0][0] = 0;
    } else if (per_item == 2) {                     // the diagonal pairs, the heavier pair first
        const int t03 = o.ph[0].ny * o.ph[0].nx + o.ph[3].ny * o.ph[3].nx, t12 = o.ph[1].ny * o.ph[1].nx + o.ph[2].ny * o.ph[2].nx;
        o.groups = 2;
        o.group_ph[t03 >= t12 ? 0 : 1][0] = 0; o.group_ph[t03 >= t12 ? 0 : 1][1] = 3;
        o.group_ph[t03 >= t12 ? 1 : 0][0] = 1; o.group_ph[t03 >= t12 ? 1 : 0][1] = 2;
    } else {                                        // one phase per item, heaviest first (stable)
        o.groups = 4;
        int order[4] = {0, 1, 2, 3};
        for (int a = 1; a < 4; ++a)
            for (int b = a; b > 0 && o.ph[order[b]].ny * o.ph[order[b]].nx > o.ph[order[b - 1]].ny * o.ph[order[b - 1]].nx; --b) {
                const int t = order[b]; order[b] = order[b - 1]; order[b - 1] = t;
            }
        for (int g = 0; g < 4; ++g) o.group_ph[g][0] = order[g];
    }
    const int ni = kConvTiles[tile][0], th = kConvTiles[tile][1], tw = kConvTiles[tile][2];
    const int sms = q.n_sms > 0 ? q.n_sms : 132;
    o.ni = ni; o.th = th; o.tw = tw; o.bn = bn;
    const int kb_ch = q.tf32x3 ? 32 : 64;             // channels per 128-byte row
    o.kblocks = (q.c_in + kb_ch - 1) / kb_ch;
    o.m_tiles = ((q.n + ni - 1) / ni) * ((q.h_out + th - 1) / th) * ((q.w_out + tw - 1) / tw);
    o.n_splits = (q.c_out + bn - 1) / bn;
    o.items = o.m_tiles * o.n_splits * o.groups;
    o.waves = (o.items + sms - 1) / sms;
    const int fixed = 2 * kConvStg + kConvBarrierBytes + kConvAlignSlack;
    const int stage_bytes = q.tf32x3 ? conv_stage_bytes_tf32x3(bn) : conv_stage_bytes(bn);
    o.stages = (kConvSmemBudget - fixed) / stage_bytes;
    if (o.stages > kConvMaxStages) o.stages = kConvMaxStages;
    o.smem_bytes = fixed + o.stages * stage_bytes;
    const double px = (double)q.n * q.h_out * q.w_out;
    o.useful_permille = (int)(1000.0 * px / ((double)o.m_tiles * 128.0));
    o.ok = o.stages >= 2 && o.smem_bytes <= kConvSmemBudget && o.kblocks > 0 && o.items > 0;
    // cost of one item in clocks (see the header comment), times the waves of the persistent launch
    double mma = 4.0 * bn, smem_rd = (2.0 * 8192 + 2.0 * bn * 128) / 128.0, l2 = (16384.0 + 128.0 * bn) / 40.0;
    if (q.tf32x3) {                                   // 3 TF32 products of 128 x bn x 32 MACs; A by shared loads, B read by 3 wgmmas
        mma = 3.0 * 128.0 * bn * 32.0 / 1024.0;
        smem_rd = (16384.0 + 2.0 * 3.0 * bn * 128) / 128.0;
        l2 = (16384.0 + 256.0 * bn) / 40.0;
    }
    double kstep = mma;
    if (smem_rd > kstep) kstep = smem_rd;
    if (l2 > kstep) kstep = l2;
    kstep += 40.0;                                    // barrier hand-shakes per K-block
    const double epi = 128.0 * bn * (q.tf32x3 ? 4.0 : 2.0) * (q.upsample ? 4.0 : 1.0) / 64.0 + 500.0;
    // makespan of the static round-robin: CTA b of G runs items b, b + G, ...; group g holds items [g * per, (g + 1) * per)
    const int G = o.items < sms ? o.items : sms, per = o.m_tiles * o.n_splits;
    double gcost[4] = {0.0, 0.0, 0.0, 0.0};
    for (int g = 0; g < o.groups; ++g)
        for (int j = 0; j < 2; ++j) {
            const int ph = o.group_ph[g][j];
            if (ph >= 0) gcost[g] += (double)o.ph[ph].ny * o.ph[ph].nx * o.kblocks * kstep + epi;
        }
    auto fdiv = [](long long a, long long b) { return a >= 0 ? a / b : -((-a + b - 1) / b); };
    o.cost = 0.0;
    for (int b = 0; b < G && G > 0; ++b) {
        double c = 0.0;
        for (int g = 0; g < o.groups; ++g) {
            const long long s0 = (long long)g * per, s1 = s0 + per;          // items w in [s0, s1) with w % G == b
            c += gcost[g] * (double)(fdiv(s1 - 1 - b, G) - fdiv(s0 - 1 - b, G));
        }
        if (c > o.cost) o.cost = c;
    }
    return o;
}

inline ConvPlanOut plan_conv(const ConvPlanIn& q) {
    ConvPlanOut best{};
    best.ok = 0;
    const bool phased = q.kind == kConvKindDeconv || q.kind == kConvKindUpconv;
    if (q.force_group && (!phased || q.force_group > 2)) return best;
    if (phased && (q.ksize < 3 || q.ksize > 9 || !(q.ksize & 1))) return best;
    if (q.tf32x3 && !phased && q.ksize != 1 && q.ksize != 3 && q.ksize != 5) return best;
    if (q.ksize < 1 || q.h_out < 1 || q.w_out < 1 || q.n < 1 || q.c_in < 8 || q.c_out < 8) return best;
    const int bns[3] = {64, 128, 256};
    for (int t = 0; t < kConvNumTiles; ++t) {
        if (q.force_tile >= 0 && t != q.force_tile) continue;
        for (int b = 0; b < 3; ++b) {
            const int bn = bns[b];
            if (q.force_bn ? bn != q.force_bn : (b > 0 && bn / 2 >= q.c_out)) continue;   // no split wider than twice the need
            if (q.tf32x3 && bn > kConvTf32x3MaxBn) continue;
            for (int per_item = 1; per_item <= 2; ++per_item) {
                if (q.force_group ? per_item != q.force_group : (per_item == 2 && (q.kind == 0 || q.kind == kConvKindConv)))
                    continue;
                const ConvPlanOut o = plan_conv_one(q, t, bn, per_item);
                if (!o.ok) continue;
                if (!best.ok || o.cost < best.cost * 0.999) best = o;   // ties keep the earlier (larger-row, narrower) choice
            }
        }
    }
    return best;
}

}  // namespace fd
