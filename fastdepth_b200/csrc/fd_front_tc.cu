// The front of the encoder as ONE kernel: stem (3x3 s2, c_in -> C0) -> DWPW 3x3 s1 (C0 -> C1) -> DWPW 3x3 s2 (C1 -> C2),
// for c_in = 1..4 input channels (RGB: 3, depth only: 1, RGB-D: 4).
//
// The three separate steps move 379 MB at b64 224x224, and 154 MB of that is conv1 reading back the map the stem has just
// written and conv2 reading back conv1's.  Here an item is one 8x8 tile of conv2's output; the CTA computes the conv0 and
// conv1 pixels that tile needs (with their 3x3 halos) in shared memory, writes the part of each it owns to its stage buffer
// and never reads either back from HBM:
//
//   x box    c_in planes x 39 rows x 48 cols (TMA, OOB zero fill = the stem's padding), 16 bytes left of the needed columns
//   T0       19 x 19 conv0 pixels x C0: rows / cols 2..17 are this item's part of the conv0 buffer; pixels outside the map are 0
//   T1       17 x 17 conv1 pixels x C1: rows / cols 1..16 -> the conv1 buffer; pixels outside the map are 0
//   out      8 x 8 conv2 pixels x C2 -> the conv2 buffer
//
// Per item, all 256 threads (two warpgroups) go through the phases in order, separated by __syncthreads: im2col + stem
// wgmma in two chunks of 192 rows; conv1's depthwise half into the A operand; conv1's pointwise wgmma into T1; conv2's
// depthwise half; conv2's pointwise wgmma.  The depthwise halves are most of the instruction stream, so a thread computes
// a whole output row of one channel pair and widens each input word once for every output that uses it.  Two CTAs share
// an SM (front_tc_smem_bytes), so one CTA's phases overlap the other's.  The x box shares the A region with the stem chunk
// and conv2's operand but not with conv1's, so the next item's box loads from the end of conv1's GEMM through all of conv2.
// Three planes fit in conv1's A region beside the stem chunk; a fourth runs 2688 bytes past it, so at c_in = 4 the tiles
// region moves up by that much and the CTA still fits twice per SM.  Five or more planes do not fit twice (front_tc_layout).
//
// Same bits as stem_tc_kernel + block_tc_kernel (HALFK for conv1): the stem's taps sit in the same K positions and run as
// ceil(9 c_in / 16) k16 steps from a zero accumulator (two at c_in = 3); a depthwise output is one fp32 FMA per tap with ky outer and kx inner from +0 over
// 16-bit taps widened to fp32 (the zero pixels outside the map add +0 or -0 to an accumulator that starts at +0, which
// leaves it unchanged), then ffma2_abc BN and pack_act; conv1's pointwise GEMM issues K = 64 against zero channels
// 32..63 as the HALFK block kernel does; every epilogue is ffma2_abc + pack_act on the same fragment.
#include <cstdio>
#include <cstring>
#include <new>
#include <string>

#include "fd_tc_common.cuh"

namespace fd {

constexpr int FR_THREADS = 256;
constexpr int FR_C0 = 32, FR_C1 = 64, FR_C2 = 128;
constexpr int FR_T0 = 19, FR_T1 = 17, FR_T2 = 8;            // tile edges of conv0, conv1, conv2
constexpr int FR_XH = 39, FR_XW = 48;                       // x box: rows 4*oy2 - 5 .., columns 4*ox2 - 8 ..
constexpr int FR_MAX_CIN = 4;                               // planes of the x box for which two CTAs fit on an SM
constexpr int FR_A0_ROWS = 192;                             // stem A operand: two chunks of three m64 blocks (361 rows)
// shared-memory layout (offsets from the 1 KB-aligned base); SWIZZLE_128B operands first
constexpr uint32_t FR_W0 = 0, FR_W1 = FR_W0 + FR_C0 * 128, FR_W2 = FR_W1 + FR_C1 * 128;
constexpr uint32_t FR_R1 = FR_W2 + FR_C2 * 128;             // A operands: stem chunk (24 KB), conv1 (320 rows, 40 KB), conv2 (8 KB)
constexpr uint32_t FR_X = FR_R1 + 28672;                    // x box: beside the stem chunk and conv2's A, inside conv1's A
// x box bytes (11232 at c_in = 3) and how far they run past conv1's A region (rounded to 128 B; 0 for c_in <= 3)
__host__ __device__ constexpr uint32_t fr_x_bytes(int cin) { return (uint32_t)cin * FR_XH * FR_XW * 2; }
__host__ __device__ constexpr uint32_t fr_x_over(int cin) {
    return FR_X + fr_x_bytes(cin) > FR_R1 + 320 * 128 ? (FR_X + fr_x_bytes(cin) - (FR_R1 + 320 * 128) + 127) / 128 * 128 : 0;
}
__host__ __device__ constexpr uint32_t fr_r2(int cin) { return FR_R1 + 320 * 128 + fr_x_over(cin); }   // T0, then T1, then conv2's output staging
__host__ __device__ constexpr uint32_t fr_prm(int cin) { return fr_r2(cin) + 37120; }                  // after T1 (289 x 128 B)
// parameter block (global blob after the weights, copied verbatim): dw taps [9][C] 16-bit, dw scale [C] + bias [C] fp32,
// pointwise (scale, scale, bias, bias) per channel pair
constexpr uint32_t FR_P_TAP1 = 0, FR_P_SB1 = FR_P_TAP1 + 9 * FR_C0 * 2, FR_P_TAP2 = FR_P_SB1 + 2 * FR_C0 * 4;
constexpr uint32_t FR_P_SB2 = FR_P_TAP2 + 9 * FR_C1 * 2, FR_P_AFF0 = FR_P_SB2 + 2 * FR_C1 * 4;
constexpr uint32_t FR_P_AFF1 = FR_P_AFF0 + FR_C0 * 8, FR_P_AFF2 = FR_P_AFF1 + FR_C1 * 8, FR_P_BYTES = FR_P_AFF2 + FR_C2 * 8;
__host__ __device__ constexpr uint32_t fr_bar(int cin) { return fr_prm(cin) + FR_P_BYTES; }
constexpr uint32_t FR_W_BYTES = (FR_C0 + FR_C1 + FR_C2) * 128;    // weights in the blob: [224 rows][64] 16-bit, K-major

struct FrontParams {
    int n, h, w;                       // input images and their size; conv0 / conv1 are (h/2, w/2), conv2 (h/4, w/4)
    int tiles_x, tiles_y, items;       // 8x8 tiles of conv2's map
    int pitch0, pitch1, pitch2;        // elements between pixels of the three output buffers
    void* out0;
    void* out1;
    void* out2;
    const uint4* blob;                 // weights [224][64] 16-bit, then the parameter block
};

size_t front_tc_smem_bytes(int cin) { return (size_t)fr_bar(cin) + 8 + 1024; }
// CTAs of front_tc_kernel that fit on one SM with c_in input planes: 228 KB of shared memory per SM, 1 KB of it reserved
// per resident CTA, and the register file (128 registers x 256 threads) caps it at two
int front_tc_ctas_per_sm(int cin) {
    const int c = (int)((228u * 1024u) / (front_tc_smem_bytes(cin) + 1024));
    return c < 2 ? c : 2;
}
// out[0..5] for a stem of c_in planes: dynamic shared memory per CTA (with the 1 KB alignment slack), CTAs per SM, threads
// per CTA, and the bytes of the three regions: weights + parameters, A operands + x box, tiles (T0 / T1 / conv2 staging)
void front_tc_layout(int cin, int* out) {
    out[0] = (int)front_tc_smem_bytes(cin); out[1] = front_tc_ctas_per_sm(cin); out[2] = FR_THREADS;
    out[3] = (int)(FR_R1 - FR_W0 + FR_P_BYTES); out[4] = (int)(fr_r2(cin) - FR_R1); out[5] = (int)(fr_prm(cin) - fr_r2(cin));
    static_assert(FR_X + fr_x_bytes(3) <= FR_R1 + 320 * 128 && FR_X >= FR_R1 + FR_A0_ROWS * 128,
                  "three planes: x box beside the stem chunk, inside the A region");
    static_assert(fr_x_over(3) == 0 && fr_x_over(4) == 2688, "c_in <= 3 keeps the layout; c_in = 4 moves the tiles up 2688 B");
}

template <typename T, bool RELU6, int CIN>
__global__ void __launch_bounds__(FR_THREADS, 2)
front_tc_kernel(const __grid_constant__ CUtensorMap tm_x, const FrontParams p) {
    using MF = MixFma<T>;
    constexpr uint32_t FR_R2 = fr_r2(CIN), FR_PRM = fr_prm(CIN), FR_BAR = fr_bar(CIN), FR_X_BYTES = fr_x_bytes(CIN);
    constexpr int KS = (9 * CIN + 15) / 16;                  // stem k16 steps
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* smem = smem_raw + (smem_base - smem_u32(smem_raw));
    uint8_t* r1 = smem + FR_R1;
    uint8_t* r2 = smem + FR_R2;
    const uint8_t* prm = smem + FR_PRM;
    const uint32_t bar = smem_base + FR_BAR;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int wg = warp >> 2, wq = warp & 3, cq = (lane & 3) * 2;
    const int h0 = p.h >> 1, w0 = p.w >> 1, h2 = p.h >> 2, w2 = p.w >> 2;

    if (tid == 0) { mbar_init(bar, 1); fence_barrier_init(); tma_prefetch_desc(&tm_x); }
    // weights into SWIZZLE_128B K-major rows (16-byte chunk c of row r at c ^ (r & 7)), parameters verbatim
    for (int i = tid; i < (int)(FR_W_BYTES / 16); i += FR_THREADS) {
        const int r = i >> 3, c = i & 7;
        *reinterpret_cast<uint4*>(smem + r * 128 + ((c ^ (r & 7)) << 4)) = p.blob[i];
    }
    for (int i = tid; i < (int)(FR_P_BYTES / 16); i += FR_THREADS)
        reinterpret_cast<uint4*>(smem + FR_PRM)[i] = p.blob[FR_W_BYTES / 16 + i];
    fence_proxy_async();
    pdl_launch_dependents();
    pdl_wait_prior_grid();
    __syncthreads();

    auto decode = [&](int it, int& img, int& oy2, int& ox2) {
        const int t = it / p.tiles_x;
        ox2 = (it - t * p.tiles_x) * FR_T2;
        img = t / p.tiles_y;
        oy2 = (t - img * p.tiles_y) * FR_T2;
    };
    auto load_x = [&](int it) {
        int img, oy2, ox2;
        decode(it, img, oy2, ox2);
        mbar_expect_tx(bar, FR_X_BYTES);
        tma_load_4d(smem_base + FR_X, &tm_x, bar, 4 * ox2 - 8, 4 * oy2 - 5, 0, img);
    };
    if (tid == 0 && (int)blockIdx.x < p.items) load_x(blockIdx.x);

    // the depthwise taps and BN of the lane's channel pair: conv1 (pair lane & 15) and conv2 (pair lane), widened where used
    const int q1 = lane & 15;
    const float* sb1 = reinterpret_cast<const float*>(prm + FR_P_SB1);
    const float* sb2 = reinterpret_cast<const float*>(prm + FR_P_SB2);
    const float2* aff0 = reinterpret_cast<const float2*>(prm + FR_P_AFF0);
    const float2* aff1 = reinterpret_cast<const float2*>(prm + FR_P_AFF1);
    const float2* aff2 = reinterpret_cast<const float2*>(prm + FR_P_AFF2);
    const uint32_t w_lo = sw128_desc_lo(smem_base);
    const uint32_t r1_lo = sw128_desc_lo(smem_base + FR_R1);
    T* __restrict__ o0 = reinterpret_cast<T*>(p.out0);
    T* __restrict__ o1 = reinterpret_cast<T*>(p.out1);
    T* __restrict__ o2 = reinterpret_cast<T*>(p.out2);

    uint32_t ph = 0;
    for (int it = blockIdx.x; it < p.items; it += gridDim.x, ph ^= 1u) {
        int img, oy2, ox2;
        decode(it, img, oy2, ox2);
        const int y0 = 2 * oy2 - 2, x0 = 2 * ox2 - 2;     // conv0 coordinates of T0's origin
        const int y1 = 2 * oy2 - 1, x1 = 2 * ox2 - 1;     // conv1 coordinates of T1's origin
        mbar_wait(bar, ph);

        // ---- stem: im2col + wgmma + BN / ReLU6 into T0, two chunks of 192 pixels ----
        for (int ch = 0; ch < 2; ++ch) {
            if (tid < FR_A0_ROWS) {
                const int m = ch * FR_A0_ROWS + tid;
                uint32_t wd[8 * KS];                       // the KS k16 steps' K positions, two per word
                if (m < FR_T0 * FR_T0) {
                    const int ty = m / FR_T0, tx = m - ty * FR_T0;
                    // tap kx of T0 column tx is box column 2 tx + 3 + kx: the high half of word tx + 1, both halves of word tx + 2
                    const uint8_t* xs = smem + FR_X + (2 * ty * FR_XW + 2 * tx + 2) * 2;
                    constexpr int NK = 9 * CIN;
                    uint32_t hv[NK];
#pragma unroll
                    for (int r = 0; r < 3 * CIN; ++r) {
                        const int ci = r / 3, ky = r % 3;
                        const uint32_t* q = reinterpret_cast<const uint32_t*>(xs + ((ci * FR_XH + ky) * FR_XW) * 2);
                        const uint32_t v0 = q[0], v1 = q[1];
                        hv[3 * r] = v0 >> 16; hv[3 * r + 1] = v1 & 0xffffu; hv[3 * r + 2] = v1 >> 16;
                    }
#pragma unroll
                    for (int j = 0; j < 8 * KS; ++j) {
                        const uint32_t lo = (2 * j < NK) ? hv[(2 * j < NK) ? 2 * j : 0] : 0u;
                        const uint32_t hi = (2 * j + 1 < NK) ? hv[(2 * j + 1 < NK) ? 2 * j + 1 : 0] : 0u;
                        wd[j] = lo | (hi << 16);
                    }
                } else {
#pragma unroll
                    for (int j = 0; j < 8 * KS; ++j) wd[j] = 0u;
                }
                uint8_t* a_row = r1 + tid * 128;
#pragma unroll
                for (int c = 0; c < 2 * KS; ++c)
                    *reinterpret_cast<uint4*>(a_row + ((c ^ (tid & 7)) << 4)) = make_uint4(wd[4 * c], wd[4 * c + 1], wd[4 * c + 2], wd[4 * c + 3]);
            }
            fence_proxy_async();
            __syncthreads();
            for (int mb = wg; mb < 3; mb += 2) {
                float acc[16];
                wgmma_fence();
#pragma unroll
                for (int ks = 0; ks < KS; ++ks)
                    wgmma_n32<T>(acc, sw128_desc(r1_lo + (uint32_t)mb * 512u + 2u * ks), sw128_desc(w_lo + (FR_W0 >> 4) + 2u * ks),
                                 ks > 0 ? 1u : 0u);
                wgmma_commit();
                wgmma_wait0();
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int m = ch * FR_A0_ROWS + mb * 64 + wq * 16 + (lane >> 2) + 8 * h;
                    if (m >= FR_T0 * FR_T0) continue;
                    const int ty = m / FR_T0, tx = m - ty * FR_T0;
                    const bool in_map = (unsigned)(y0 + ty) < (unsigned)h0 && (unsigned)(x0 + tx) < (unsigned)w0;
                    uint8_t* row = r2 + m * 64;
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const float4 af = *reinterpret_cast<const float4*>(aff0 + i * 8 + cq);
                        const uint32_t v = in_map ? MF::template pack_act<true>(ffma2_abc(f32x2_make(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]),
                                                                                          f32x2_make(af.x, af.y), f32x2_make(af.z, af.w)))
                                                  : 0u;
                        *reinterpret_cast<uint32_t*>(row + ((i ^ ((m >> 1) & 3)) << 4) + cq * 2) = v;
                    }
                }
            }
            __syncthreads();
        }

        // ---- T0's owned 16 x 16 -> conv0; conv1's depthwise half -> A (K = 64, channels 32..63 zero) ----
        for (int i = tid; i < 16 * 16 * 4; i += FR_THREADS) {
            const int px = i >> 2, c = i & 3, ty = 2 + (px >> 4), tx = 2 + (px & 15), m = ty * FR_T0 + tx;
            const uint4 v = *reinterpret_cast<const uint4*>(r2 + m * 64 + ((c ^ ((m >> 1) & 3)) << 4));
            *reinterpret_cast<uint4*>(o0 + (((size_t)img * h0 + y0 + ty) * w0 + x0 + tx) * p.pitch0 + c * 8) = v;
        }
        // a thread takes one T1 row of one channel pair (q1 == tid & 15): every T0 word of the three input rows is loaded and
        // widened once and feeds the up to three outputs that use it.  An output still sees its taps in (ky, kx) order.
        f32x2 k1[9];
#pragma unroll
        for (int t = 0; t < 9; ++t) k1[t] = MF::widen(*reinterpret_cast<const uint32_t*>(prm + FR_P_TAP1 + (t * FR_C0 + 2 * q1) * 2));
        const f32x2 s1 = f32x2_make(sb1[2 * q1], sb1[2 * q1 + 1]), b1 = f32x2_make(sb1[FR_C0 + 2 * q1], sb1[FR_C0 + 2 * q1 + 1]);
        {
            const int uy = tid >> 4;                       // rows 0..15; row 16 below, one output per thread
            f32x2 acc[FR_T1];
#pragma unroll
            for (int o = 0; o < FR_T1; ++o) acc[o] = 0ull;
#pragma unroll
            for (int ky = 0; ky < 3; ++ky) {
                const int mrow = (uy + ky) * FR_T0;
#pragma unroll
                for (int ix = 0; ix < FR_T0; ++ix) {
                    const int mi = mrow + ix;
                    const f32x2 v = MF::widen(*reinterpret_cast<const uint32_t*>(r2 + mi * 64 + (((q1 >> 2) ^ ((mi >> 1) & 3)) << 4) + (q1 & 3) * 4));
#pragma unroll
                    for (int kx = 0; kx < 3; ++kx)
                        if (ix - kx >= 0 && ix - kx < FR_T1) ffma2(acc[ix - kx], v, k1[ky * 3 + kx]);
                }
            }
#pragma unroll
            for (int o = 0; o < FR_T1; ++o) {
                const int m = uy * FR_T1 + o;
                uint8_t* a_row = r1 + m * 128;
                *reinterpret_cast<uint32_t*>(a_row + (((q1 >> 2) ^ (m & 7)) << 4) + (q1 & 3) * 4) = MF::template pack_act<RELU6>(ffma2_abc(acc[o], s1, b1));
                *reinterpret_cast<uint32_t*>(a_row + ((((q1 >> 2) + 4) ^ (m & 7)) << 4) + (q1 & 3) * 4) = 0u;
            }
        }
        for (int u = tid; u < FR_T1 * 16; u += FR_THREADS) {      // row 16: output u >> 4 of pair q1 (== u & 15)
            const int ux = u >> 4, m = (FR_T1 - 1) * FR_T1 + ux;
            f32x2 acc = 0ull;
#pragma unroll
            for (int ky = 0; ky < 3; ++ky)
#pragma unroll
                for (int kx = 0; kx < 3; ++kx) {
                    const int mi = (FR_T1 - 1 + ky) * FR_T0 + ux + kx;
                    ffma2(acc, MF::widen(*reinterpret_cast<const uint32_t*>(r2 + mi * 64 + (((q1 >> 2) ^ ((mi >> 1) & 3)) << 4) + (q1 & 3) * 4)),
                          k1[ky * 3 + kx]);
                }
            uint8_t* a_row = r1 + m * 128;
            *reinterpret_cast<uint32_t*>(a_row + (((q1 >> 2) ^ (m & 7)) << 4) + (q1 & 3) * 4) = MF::template pack_act<RELU6>(ffma2_abc(acc, s1, b1));
            *reinterpret_cast<uint32_t*>(a_row + ((((q1 >> 2) + 4) ^ (m & 7)) << 4) + (q1 & 3) * 4) = 0u;
        }
        fence_proxy_async();
        __syncthreads();

        // ---- conv1's pointwise half: 5 m64 blocks x n64 x four k16 steps -> BN / act -> T1 (0 outside the map) ----
        for (int mb = wg; mb < 5; mb += 2) {
            float acc[32];
            wgmma_fence();
#pragma unroll
            for (int k4 = 0; k4 < 4; ++k4)
                wgmma_n64<T>(acc, sw128_desc(r1_lo + (uint32_t)mb * 512u + 2u * k4), sw128_desc(w_lo + (FR_W1 >> 4) + 2u * k4), k4 > 0 ? 1u : 0u);
            wgmma_commit();
            wgmma_wait0();
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int m = mb * 64 + wq * 16 + (lane >> 2) + 8 * h;
                if (m >= FR_T1 * FR_T1) continue;
                const int uy = m / FR_T1, ux = m - uy * FR_T1;
                const bool in_map = (unsigned)(y1 + uy) < (unsigned)h0 && (unsigned)(x1 + ux) < (unsigned)w0;
                uint8_t* row = r2 + m * 128;
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const float4 af = *reinterpret_cast<const float4*>(aff1 + i * 8 + cq);
                    const uint32_t v = in_map ? MF::template pack_act<RELU6>(ffma2_abc(f32x2_make(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]),
                                                                                      f32x2_make(af.x, af.y), f32x2_make(af.z, af.w)))
                                              : 0u;
                    *reinterpret_cast<uint32_t*>(row + ((i ^ (m & 7)) << 4) + cq * 2) = v;
                }
            }
        }
        __syncthreads();
        // conv1's A operand is consumed: the next item's x box may land beside conv2's
        if (tid == 0 && it + (int)gridDim.x < p.items) load_x(it + gridDim.x);

        // ---- T1's owned 16 x 16 -> conv1; conv2's depthwise half (stride 2) -> A ----
        for (int i = tid; i < 16 * 16 * 8; i += FR_THREADS) {
            const int px = i >> 3, c = i & 7, uy = 1 + (px >> 4), ux = 1 + (px & 15), m = uy * FR_T1 + ux;
            const uint4 v = *reinterpret_cast<const uint4*>(r2 + m * 128 + ((c ^ (m & 7)) << 4));
            *reinterpret_cast<uint4*>(o1 + (((size_t)img * h0 + y1 + uy) * w0 + x1 + ux) * p.pitch1 + c * 8) = v;
        }
        {   // a thread takes one output row of one channel pair (lane): each T1 word of the three input rows is widened once
            const int vy = tid >> 5;
            f32x2 k2[9];
#pragma unroll
            for (int t = 0; t < 9; ++t) k2[t] = MF::widen(*reinterpret_cast<const uint32_t*>(prm + FR_P_TAP2 + (t * FR_C1 + 2 * lane) * 2));
            const f32x2 s2 = f32x2_make(sb2[2 * lane], sb2[2 * lane + 1]), b2 = f32x2_make(sb2[FR_C1 + 2 * lane], sb2[FR_C1 + 2 * lane + 1]);
            f32x2 acc[FR_T2];
#pragma unroll
            for (int o = 0; o < FR_T2; ++o) acc[o] = 0ull;
#pragma unroll
            for (int ky = 0; ky < 3; ++ky) {
                const int mrow = (2 * vy + ky) * FR_T1;
#pragma unroll
                for (int ix = 0; ix < FR_T1; ++ix) {
                    const int mi = mrow + ix;
                    const f32x2 v = MF::widen(*reinterpret_cast<const uint32_t*>(r2 + mi * 128 + (((lane >> 2) ^ (mi & 7)) << 4) + (lane & 3) * 4));
#pragma unroll
                    for (int kx = 0; kx < 3; ++kx)
                        if (((ix - kx) & 1) == 0 && ix - kx >= 0 && (ix - kx) / 2 < FR_T2) ffma2(acc[(ix - kx) / 2], v, k2[ky * 3 + kx]);
                }
            }
#pragma unroll
            for (int o = 0; o < FR_T2; ++o) {
                const int m = vy * FR_T2 + o;
                *reinterpret_cast<uint32_t*>(r1 + m * 128 + (((lane >> 2) ^ (m & 7)) << 4) + (lane & 3) * 4) =
                    MF::template pack_act<RELU6>(ffma2_abc(acc[o], s2, b2));
            }
        }
        fence_proxy_async();
        __syncthreads();

        // ---- conv2's pointwise half: warpgroup wg takes output channels [64 wg, 64 wg + 64) -> staging [64 px][128 ch] ----
        {
            float acc[32];
            wgmma_fence();
#pragma unroll
            for (int k4 = 0; k4 < 4; ++k4)
                wgmma_n64<T>(acc, sw128_desc(r1_lo + 2u * k4), sw128_desc(w_lo + (FR_W2 >> 4) + (uint32_t)wg * 512u + 2u * k4), k4 > 0 ? 1u : 0u);
            wgmma_commit();
            wgmma_wait0();
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int m = wq * 16 + (lane >> 2) + 8 * h;
                uint8_t* row = r2 + m * 256;
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const int c = wg * 8 + i;                      // 16-byte chunk of the 256-byte pixel
                    const float4 af = *reinterpret_cast<const float4*>(aff2 + c * 8 + cq);
                    *reinterpret_cast<uint32_t*>(row + ((c ^ (m & 15)) << 4) + cq * 2) = MF::template pack_act<RELU6>(
                        ffma2_abc(f32x2_make(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]), f32x2_make(af.x, af.y), f32x2_make(af.z, af.w)));
                }
            }
        }
        __syncthreads();
        for (int i = tid; i < 64 * 16; i += FR_THREADS) {
            const int m = i >> 4, c = i & 15;
            const uint4 v = *reinterpret_cast<const uint4*>(r2 + m * 256 + ((c ^ (m & 15)) << 4));
            *reinterpret_cast<uint4*>(o2 + (((size_t)img * h2 + oy2 + (m >> 3)) * w2 + ox2 + (m & 7)) * p.pitch2 + c * 8) = v;
        }
        // the staging tile is read before the next item's stem epilogue overwrites it (that comes after two more barriers)
    }
}

// ----------------------------------------------------------------------------------------------
// host side
// ----------------------------------------------------------------------------------------------
struct FrontTcPlan {
    CUtensorMap tm_x;
    FrontParams p;
    dim3 grid;
    size_t smem_bytes;
    int dtype, relu6, c_in;
    TcLaunchOpts opts;
    const void* x_bound = nullptr;
    void* blob = nullptr;
    std::string name;
};

// stages 0..2 as the kernel takes them: the stem conv_bn(c_in, 32, 2) with ReLU6 and two CTAs per SM at that c_in (c_in
// 1..4), then two 3x3 DWPW blocks (stride 1, then 2) 32 -> 64 -> 128, one act for both blocks, h and w multiples of 32
// (conv2's map is whole 8x8 tiles), 16-bit.  Geometry only (no driver call), so that the host-only debug export can apply
// the same rule.
bool front_tc_shape_ok(int dtype, const StageGeom& g0, const StageGeom& g1, const StageGeom& g2) {
    if (dtype != FD_F16 && dtype != FD_BF16) return false;
    if (g0.ksize != 3 || g0.stride != 2 || g0.c_out != FR_C0 || g0.act != FD_ACT_RELU6 || g0.upsample) return false;
    if (g0.c_in < 1 || g0.c_in > FR_MAX_CIN || front_tc_ctas_per_sm(g0.c_in) < 2) return false;
    if (g0.h_in % 32 || g0.w_in % 32) return false;
    if (g1.ksize != 3 || g1.stride != 1 || g1.c_in != FR_C0 || g1.c_out != FR_C1 || g1.upsample) return false;
    if (g2.ksize != 3 || g2.stride != 2 || g2.c_in != FR_C1 || g2.c_out != FR_C2 || g2.upsample) return false;
    return g1.act == g2.act;
}

int front_tc_items(int n, int h, int w) { return n * (h / 32) * (w / 32); }

// the blob: weights [224][64] 16-bit (stem [32][64] with K = (ci, ky, kx) as the stem kernel packs it, zero past 9 c_in,
// conv1 [64][64] with K 32..63 zero, conv2 [128][64]), then the parameter block of the FR_P_* layout
template <typename T>
__global__ void pack_front_kernel(int c_in, const float* __restrict__ wk, const T* __restrict__ pw1, const T* __restrict__ pw2,
                                  const float* __restrict__ sc0, const float* __restrict__ bi0,
                                  const float* __restrict__ dw1, const float* __restrict__ dsc1, const float* __restrict__ dbi1,
                                  const float* __restrict__ sc1, const float* __restrict__ bi1,
                                  const float* __restrict__ dw2, const float* __restrict__ dsc2, const float* __restrict__ dbi2,
                                  const float* __restrict__ sc2, const float* __restrict__ bi2, uint8_t* __restrict__ blob) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    T* wt = reinterpret_cast<T*>(blob);
    if (i < (FR_C0 + FR_C1 + FR_C2) * 64) {
        const int r = i / 64, k = i % 64;
        if (r < FR_C0) wt[i] = Traits<T>::from_f(k < 9 * c_in ? wk[k * FR_C0 + r] : 0.f);
        else if (r < FR_C0 + FR_C1) wt[i] = k < FR_C0 ? pw1[(r - FR_C0) * FR_C0 + k] : Traits<T>::from_f(0.f);
        else wt[i] = pw2[(r - FR_C0 - FR_C1) * FR_C1 + k];
    }
    uint8_t* prm = blob + FR_W_BYTES;
    if (i < 9 * FR_C0) reinterpret_cast<T*>(prm + FR_P_TAP1)[i] = Traits<T>::from_f(dw1[i]);
    if (i < 9 * FR_C1) reinterpret_cast<T*>(prm + FR_P_TAP2)[i] = Traits<T>::from_f(dw2[i]);
    if (i < FR_C0) { reinterpret_cast<float*>(prm + FR_P_SB1)[i] = dsc1[i]; reinterpret_cast<float*>(prm + FR_P_SB1)[FR_C0 + i] = dbi1[i]; }
    if (i < FR_C1) { reinterpret_cast<float*>(prm + FR_P_SB2)[i] = dsc2[i]; reinterpret_cast<float*>(prm + FR_P_SB2)[FR_C1 + i] = dbi2[i]; }
    auto aff = [&](uint32_t off, const float* s, const float* b, int c) {     // (scale, scale, bias, bias) per channel pair
        float* d = reinterpret_cast<float*>(prm + off) + (c >> 1) * 4;
        d[c & 1] = s[c];
        d[2 + (c & 1)] = b[c];
    };
    if (i < FR_C0) aff(FR_P_AFF0, sc0, bi0, i);
    if (i < FR_C1) aff(FR_P_AFF1, sc1, bi1, i);
    if (i < FR_C2) aff(FR_P_AFF2, sc2, bi2, i);
}

void front_tc_destroy(FrontTcPlan* fp) {
    if (!fp) return;
    cudaFree(fp->blob);
    delete fp;
}

static int encode_front_x(FrontTcPlan* fp, const void* x) {
    PFN_encodeTiled encode = get_tensor_map_encoder();
    const CUtensorMapDataType dt = fp->dtype == FD_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
    const FrontParams& p = fp->p;
    const cuuint64_t plane = (cuuint64_t)p.w * p.h * 2;
    cuuint64_t dims[4] = {(cuuint64_t)p.w, (cuuint64_t)p.h, (cuuint64_t)fp->c_in, (cuuint64_t)p.n};
    cuuint64_t strides[3] = {(cuuint64_t)p.w * 2, plane, plane * (cuuint64_t)fp->c_in};
    cuuint32_t box[4] = {FR_XW, FR_XH, (cuuint32_t)fp->c_in, 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = encode(&fp->tm_x, dt, 4, const_cast<void*>(x), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(FD_ERR_CUDA, "cuTensorMapEncodeTiled(front input) failed: " + std::to_string((int)r));
    fp->x_bound = x;
    return FD_OK;
}

int front_tc_prepare(int dtype, const StageGeom& g0, const StageGeom& g1, const StageGeom& g2, const float* wk,
                     const float* sc0, const float* bi0, const BlockArgs& a1, const BlockArgs& a2, void* out0,
                     const TcLaunchOpts& opts, FrontTcPlan** res) {
    FrontTcPlan* fp = new (std::nothrow) FrontTcPlan();
    if (!fp) return fail(FD_ERR_CUDA, "out of host memory");
    fp->dtype = dtype; fp->relu6 = g1.act == FD_ACT_RELU6; fp->c_in = g0.c_in; fp->opts = opts;
    FrontParams& p = fp->p;
    memset(&p, 0, sizeof(p));
    p.n = g0.n; p.h = g0.h_in; p.w = g0.w_in;
    p.tiles_x = g2.w_out / FR_T2; p.tiles_y = g2.h_out / FR_T2; p.items = p.tiles_x * p.tiles_y * p.n;
    p.pitch0 = g0.out_pitch; p.pitch1 = g1.out_pitch; p.pitch2 = g2.out_pitch;
    p.out0 = out0; p.out1 = a1.out; p.out2 = a2.out;
    const size_t blob_bytes = FR_W_BYTES + FR_P_BYTES;
    if (cudaMalloc(&fp->blob, blob_bytes) != cudaSuccess) { front_tc_destroy(fp); return fail(FD_ERR_CUDA, "cudaMalloc failed"); }
    const int tot = (FR_C0 + FR_C1 + FR_C2) * 64;
    if (dtype == FD_F16)
        pack_front_kernel<__half><<<(tot + 127) / 128, 128>>>(g0.c_in, wk, (const __half*)a1.pw_w, (const __half*)a2.pw_w, sc0, bi0, a1.dw_w, a1.dw_scale,
                                                              a1.dw_bias, a1.pw_scale, a1.pw_bias, a2.dw_w, a2.dw_scale, a2.dw_bias,
                                                              a2.pw_scale, a2.pw_bias, (uint8_t*)fp->blob);
    else
        pack_front_kernel<__nv_bfloat16><<<(tot + 127) / 128, 128>>>(g0.c_in, wk, (const __nv_bfloat16*)a1.pw_w, (const __nv_bfloat16*)a2.pw_w, sc0, bi0,
                                                                     a1.dw_w, a1.dw_scale, a1.dw_bias, a1.pw_scale, a1.pw_bias, a2.dw_w,
                                                                     a2.dw_scale, a2.dw_bias, a2.pw_scale, a2.pw_bias, (uint8_t*)fp->blob);
    if (cudaGetLastError() != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) {
        front_tc_destroy(fp);
        return fail(FD_ERR_CUDA, "front parameter packing failed");
    }
    p.blob = reinterpret_cast<const uint4*>(fp->blob);
    fp->smem_bytes = front_tc_smem_bytes(g0.c_in);
    const int ctas = 2 * opts.n_sms;
    fp->grid = dim3((unsigned)(p.items < ctas ? p.items : ctas), 1, 1);
    fp->name = std::string("stem_tc+front<k3s1,k3s2,8x8>[n32,n64,n128,") + (fp->relu6 ? "relu6" : "relu") +
               (g0.c_in == 3 ? "]" : ",cin" + std::to_string(g0.c_in) + "]");
    *res = fp;
    return FD_OK;
}

size_t front_tc_param_bytes(FrontTcPlan*) { return FR_W_BYTES + FR_P_BYTES; }
const char* front_tc_name(FrontTcPlan* fp) { return fp->name.c_str(); }

template <typename T, bool R6, int CIN>
static int launch_front(FrontTcPlan* fp, cudaLaunchConfig_t& cfg) {
    static PerDeviceOnce attr_done;
    int dev = -1;
    FD_CUDA_OK(cudaGetDevice(&dev));
    if (attr_done.need(dev)) {
        FD_CUDA_OK(cudaFuncSetAttribute(front_tc_kernel<T, R6, CIN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fp->smem_bytes));
        attr_done.done(dev);
    }
    FD_CUDA_OK(cudaLaunchKernelEx(&cfg, front_tc_kernel<T, R6, CIN>, fp->tm_x, fp->p));
    return FD_OK;
}

template <typename T, bool R6>
static int launch_front_cin(FrontTcPlan* fp, cudaLaunchConfig_t& cfg) {
    switch (fp->c_in) {
        case 1: return launch_front<T, R6, 1>(fp, cfg);
        case 2: return launch_front<T, R6, 2>(fp, cfg);
        case 3: return launch_front<T, R6, 3>(fp, cfg);
        case 4: return launch_front<T, R6, 4>(fp, cfg);
        default: return fail(FD_ERR_UNSUPPORTED, "front_tc_kernel: c_in must be 1..4");
    }
}

// x may change from call to call: the input tensor map is re-encoded when it does (as stem_tc_launch)
int front_tc_launch(FrontTcPlan* fp, const void* x, cudaStream_t st) {
    if ((reinterpret_cast<uintptr_t>(x) & 15) != 0) return fail(FD_ERR_INVALID, "stem input must be 16-byte aligned");
    if (x != fp->x_bound) {
        int rc = encode_front_x(fp, x);
        if (rc) return rc;
    }
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = fp->grid; cfg.blockDim = dim3(FR_THREADS); cfg.dynamicSmemBytes = fp->smem_bytes; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = fp->opts.pdl ? 1 : 0;
    int rc;
    if (fp->dtype == FD_F16) rc = fp->relu6 ? launch_front_cin<__half, true>(fp, cfg) : launch_front_cin<__half, false>(fp, cfg);
    else rc = fp->relu6 ? launch_front_cin<__nv_bfloat16, true>(fp, cfg) : launch_front_cin<__nv_bfloat16, false>(fp, cfg);
    if (rc) return rc;
    FD_CUDA_OK(cudaGetLastError());
    return FD_OK;
}

}  // namespace fd
