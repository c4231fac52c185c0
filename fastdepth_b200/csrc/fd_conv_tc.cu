// Dense kxk stride-1 conv + folded BN + act (+ nearest x2 upsample) on wgmma: the conv() blocks of the dense NNConv decoder
// (reference models.py:52-59, 245-270) as an implicit GEMM, M = output pixels, N = output channels, K = k*k*c_in.
//
// Work item = one tile of 128 output pixels (ni images x th rows x tw columns) times bn output channels (64, 128 or 256; see
// fd_conv_plan.h for how the tile and bn are chosen).  The grid is one CTA per SM; every CTA walks items blockIdx.x,
// +gridDim.x, ...  The K loop runs over (tap, 64-channel block):
//   warp 8     TMA producer : per K step one 4-D box {64 ch, tw, th, ni} of the NHWC input, offset by (kx - p, ky - p), lands
//                             128B-swizzled: every pixel's 64 channels are one 128-byte row, which IS the K-major SW128 A operand
//                             (no im2col).  The OOB zero fill is the conv's zero padding and the channel tail.  Plus one box
//                             {64 ch, 1 tap, bn rows} of the weights [c_out][k*k][c_in] (rows past c_out and channels past c_in
//                             load as zeros)
//   warps 0-7  consumers    : two warpgroups, each owning 64 of the 128 pixel rows: one wgmma m64 n(bn) k16 per 16 channels into
//                             register accumulators, one commit group kept in flight; then BN affine + act -> 16-bit -> staging
//                             tile -> TMA tensor stores (four strided views of the output for the nearest x2 upsample)
// One mbarrier ring of operand stages (A + B) between the producer and the consumers.
//
// The same kernel runs the transposed conv (DECONV) and unpool + conv (UPCONV) stages as four stride-1 phase convs at the
// input resolution (fd_conv_plan.h): an item is then (tile, bn split, phase group); the producer's box loop and the
// consumers' K loop come from the phase's {tap0, ny, nx, dy0, dx0}, and phase 2 ry + rx is stored through output view
// tm_o[2 ry + rx] (the same four strided views as the upsample).  A CONV stage is one phase, the k x k square.
//
// conv_tc_tf32x3_kernel is an fp32 conv as split TF32 (plan option "tf32x3"): the pointwise (1x1) conv of a DWPW stage, and
// the CONV / DECONV / UPCONV stages of the dense decoders.  The same item decode, persistent item loop, phase / tap loop,
// operand ring and output views, with fp32 operands.  A K-block is 32 fp32 channels (one 128-byte row); a stage is the A box
// {32 ch, tw, th, ni} of the input at the tap's offset (the depthwise intermediate of a DWPW stage) plus two B boxes
// {32 ch, 1 tap, bn rows}, the tap's TF32 high and low weight parts (split once into [2][c_out][k*k][c_in] when the plan is
// built; a pointwise step is one phase with one tap).  The consumers split A themselves: each thread loads
// its wgmma A fragment from the swizzled tile, rounds it to a_hi = rna(a), a_lo = rna(a - a_hi), and per k8 step issues
// a_lo b_hi, a_hi b_lo, a_hi b_hi (small terms first) into one fp32 accumulator, A from registers.  The epilogue applies the
// BN affine and act in fp32 and stores [128 px][32 ch] fp32 tiles; a skip add is a TMA reduce-add (.add.f32) of that tile
// into the skip tensor (or a copy of it), so the stage output is skip + up rounded once; a phased stage stores phase q
// through view q.  It is a sibling kernel rather than an instance of conv_tc_kernel: producer, K loop and epilogue all
// differ (two B boxes, A through registers, three MMAs per step, fp32 stores or reduce-adds), and the 16-bit instances stay
// exactly as they were.
//
// A 16-bit DWPW stage that the fused block kernel would have to split many ways (plan option "unfuse", fd_api.cu) runs as two
// steps instead: dw_mid_kernel writes the depthwise half once, to the stage's intermediate, and conv_tc_kernel runs the
// pointwise half as a 1x1 CONV over it (one phase, one tap, the stage's own [c_out][c_in] weights; reduce = 1 adds the tiles
// into the skip tensor with the TMA reduce-add).  The two steps compute what block_tc_kernel computes, bit for bit: the same
// exact products in the same (ky, kx) order, the same k16 MMA sequence per accumulator, the same affine, act and rounding.
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <new>
#include <string>
#include <type_traits>

#include "fd_conv_plan.h"
#include "fd_tc_common.cuh"

namespace fd {

constexpr int CV_WARP_TMA = 8, CV_THREADS = 288;
constexpr int CV_A_BYTES = 128 * 128;

struct ConvParams {
    int n, h, w, c_in, c_out;        // conv input == conv output size (stride 1, same padding)
    int ni, th, tw;                  // tile: ni images x th rows x tw columns = 128 pixels
    int tiles_x, tiles_y, img_tiles, splits, items;
    int kblocks;
    int stages, stage_bytes;
    int upsample;                    // CONV: store the tile through all four views (nearest x2)
    int phased;                      // DECONV / UPCONV: phase q stores through view q only
    ConvPhase ph[4];
    int group_code[4];               // phases of item group g, 4 bits each, first in the low bits, ended by 0xF
    unsigned long long mg_splits, mg_tx, mg_ty, mg_img;
    const float2* affine;            // [splits * bn / 2] x (scale, scale, bias, bias) of a channel pair, zero padded
};

struct ConvBarriers {
    uint64_t full[kConvMaxStages], empty[kConvMaxStages];
};
static_assert(sizeof(ConvBarriers) <= kConvBarrierBytes, "the planner budgets the barrier block");

struct ConvCoord { int img0, oy0, ox0, n0, code; };
__device__ __forceinline__ ConvCoord conv_decode(const ConvParams& p, int w, int bn) {
    ConvCoord c;
    const uint32_t t = fdiv40((uint32_t)w, p.mg_splits);
    const int split = w - (int)t * p.splits;
    const uint32_t t2 = fdiv40(t, p.mg_tx);
    const int tx = (int)(t - t2 * (uint32_t)p.tiles_x);
    const uint32_t t3 = fdiv40(t2, p.mg_ty);
    const int ty = (int)(t2 - t3 * (uint32_t)p.tiles_y);
    const uint32_t t4 = fdiv40(t3, p.mg_img);
    c.code = p.group_code[t4];
    c.img0 = (int)(t3 - t4 * (uint32_t)p.img_tiles) * p.ni; c.oy0 = ty * p.th; c.ox0 = tx * p.tw; c.n0 = split * bn;
    return c;
}

template <typename T, int BN, bool RELU6>
__global__ void __launch_bounds__(CV_THREADS, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tm_in, const __grid_constant__ CUtensorMap tm_w,
               const __grid_constant__ CUtensorMap tm_o0, const __grid_constant__ CUtensorMap tm_o1,
               const __grid_constant__ CUtensorMap tm_o2, const __grid_constant__ CUtensorMap tm_o3,
               const __grid_constant__ ConvParams p, const int reduce) {
    using MF = MixFma<T>;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* smem = smem_raw + (smem_base - smem_u32(smem_raw));
    // carve-up: [stages x (A 16 KB | B bn x 128 B)][2 staging tiles][barriers]; every piece a multiple of 1 KB
    const uint32_t stg_off = (uint32_t)p.stages * (uint32_t)p.stage_bytes;
    const uint32_t bar_off = stg_off + 2u * (uint32_t)kConvStg;
    ConvBarriers* bars = reinterpret_cast<ConvBarriers*>(smem + bar_off);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        for (int i = 0; i < kConvMaxStages; ++i) { mbar_init(smem_u32(&bars->full[i]), 1); mbar_init(smem_u32(&bars->empty[i]), 2); }
        fence_barrier_init();
    }
    if (warp == CV_WARP_TMA && lane == 0) {
        tma_prefetch_desc(&tm_in); tma_prefetch_desc(&tm_w); tma_prefetch_desc(&tm_o0);
        if (p.upsample || p.phased) { tma_prefetch_desc(&tm_o1); tma_prefetch_desc(&tm_o2); tma_prefetch_desc(&tm_o3); }
    }
    pdl_launch_dependents();                       // the next kernel may begin its own prologue
    pdl_wait_prior_grid();                         // everything below reads what the previous kernel wrote
    __syncthreads();

    if (warp == CV_WARP_TMA) {
        // =========================== TMA producer ===========================
        if (lane == 0) {
            Ring r;
            for (int w = blockIdx.x; w < p.items; w += gridDim.x) {
                const ConvCoord c = conv_decode(p, w, BN);
                for (int code = c.code; code != 0xF; code >>= 4) {
                    const ConvPhase f = p.ph[code & 0xF];
                    for (int ky = 0; ky < f.ny; ++ky)
                        for (int kx = 0; kx < f.nx; ++kx)
                            for (int kb = 0; kb < p.kblocks; ++kb, r.next((uint32_t)p.stages)) {
                                const uint32_t st = smem_base + r.s * (uint32_t)p.stage_bytes, bar = smem_u32(&bars->full[r.s]);
                                mbar_wait(smem_u32(&bars->empty[r.s]), r.ph ^ 1u);
                                mbar_expect_tx(bar, (uint32_t)p.stage_bytes);
                                tma_load_4d(st, &tm_in, bar, kb * 64, c.ox0 + f.dx0 + kx, c.oy0 + f.dy0 + ky, c.img0);
                                tma_load_3d(st + CV_A_BYTES, &tm_w, bar, kb * 64, f.tap0 + ky * f.nx + kx, c.n0);
                            }
                }
            }
        }
    } else {
        // =========================== consumer warpgroups: wgmma + epilogue ===========================
        // warpgroup wg owns pixel rows [64 wg, 64 wg + 64) of every item; a thread holds rows r0 and r0 + 8 of every 8-column
        // group j of the accumulator (fragment layout: see the wgmma wrappers)
        const int wg = warp >> 2, wq = warp & 3;
        const int r0 = wg * 64 + wq * 16 + (lane >> 2), cq = (lane & 3) * 2;
        const bool leader = wq == 0 && lane == 0;          // releases this warpgroup's operand stages
        const bool elected = warp == 0 && lane == 0;       // issues the tensor stores
        constexpr uint32_t bar_id = 1u, bar_n = 256u;      // named barrier of the eight consumer warps
        Ring r;
        uint32_t stg_flip = 0;
        for (int w = blockIdx.x; w < p.items; w += gridDim.x) {
            const ConvCoord c = conv_decode(p, w, BN);
            for (int code = c.code; code != 0xF; code >>= 4) {        // the phases of this item's group, one after the other
                const int q = code & 0xF;
                const int ksteps = p.ph[q].ny * p.ph[q].nx * p.kblocks;
                float acc[BN / 2];
#pragma unroll
                for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
                uint32_t prev = 0;
                for (int k = 0; k < ksteps; ++k) {
                    mbar_wait(smem_u32(&bars->full[r.s]), r.ph);
                    const uint32_t st = smem_base + r.s * (uint32_t)p.stage_bytes;
                    const uint32_t a_lo = sw128_desc_lo(st + (uint32_t)wg * 8192u), b_lo = sw128_desc_lo(st + CV_A_BYTES);
                    wgmma_fence();
#pragma unroll
                    for (int k4 = 0; k4 < 4; ++k4)             // +32 B (16 channels) per K step inside the 128-byte swizzle row
                        wgmma_bn<T, BN>(acc, sw128_desc(a_lo + 2u * k4), sw128_desc(b_lo + 2u * k4), (k > 0 || k4 > 0) ? 1u : 0u);
                    wgmma_commit();
                    wgmma_wait1();                             // the previous step's MMAs are done: release its stage
                    if (k > 0 && leader) mbar_arrive(smem_u32(&bars->empty[prev]));
                    prev = r.s;
                    r.next((uint32_t)p.stages);
                }
                wgmma_wait0();
                if (leader) mbar_arrive(smem_u32(&bars->empty[prev]));

                // per block of 64 output channels: registers -> BN affine + act -> 16-bit -> shared staging tile [128 px][64 ch]
                // (16-byte chunks XOR-swizzled like a SWIZZLE_128B box) -> TMA tensor stores; image borders and the channel tail
                // are clipped by the hardware
#pragma unroll
                for (int cb = 0; cb < BN / 64; ++cb) {
                    if (c.n0 + cb * 64 >= p.c_out) break;
                    uint8_t* stg = smem + stg_off + (stg_flip & 1u) * (uint32_t)kConvStg;
                    ++stg_flip;
                    const float2* aff = p.affine + c.n0 + cb * 64;
#pragma unroll
                    for (int i = 0; i < 8; ++i) {              // 8-column group i of this block: the thread's channel pair of rows r0, r0 + 8
                        const float4 af = __ldg(reinterpret_cast<const float4*>(aff + i * 8 + cq));     // (s0, s1, b0, b1)
                        const f32x2 sc = f32x2_make(af.x, af.y), bi = f32x2_make(af.z, af.w);
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            const int rr = r0 + 8 * h;
                            const int j = cb * 8 + i;
                            *reinterpret_cast<uint32_t*>(stg + rr * 128 + ((i ^ (rr & 7)) << 4) + cq * 2) =
                                MF::template pack_act<RELU6>(ffma2_abc(f32x2_make(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]), sc, bi));
                        }
                    }
                    // before the OTHER staging buffer may be overwritten its previous store must have finished reading it
                    fence_proxy_async();
                    if (elected) bulk_wait_read0();
                    asm volatile("bar.sync %0, %1;" ::"r"(bar_id), "r"(bar_n) : "memory");
                    if (elected) {
                        const uint32_t src = smem_u32(stg);
                        const int cc = c.n0 + cb * 64;
                        if (reduce) {      // a 1x1 step with a skip: the views already hold the skip tensor (never phased)
                            tma_reduce_add_4d(&tm_o0, src, cc, c.ox0, c.oy0, c.img0);
                            if (p.upsample) {
                                tma_reduce_add_4d(&tm_o1, src, cc, c.ox0, c.oy0, c.img0);
                                tma_reduce_add_4d(&tm_o2, src, cc, c.ox0, c.oy0, c.img0);
                                tma_reduce_add_4d(&tm_o3, src, cc, c.ox0, c.oy0, c.img0);
                            }
                        } else {
                            tma_store_4d(q == 0 ? &tm_o0 : q == 1 ? &tm_o1 : q == 2 ? &tm_o2 : &tm_o3, src, cc, c.ox0, c.oy0, c.img0);
                            if (p.upsample) {
                                tma_store_4d(&tm_o1, src, cc, c.ox0, c.oy0, c.img0);
                                tma_store_4d(&tm_o2, src, cc, c.ox0, c.oy0, c.img0);
                                tma_store_4d(&tm_o3, src, cc, c.ox0, c.oy0, c.img0);
                            }
                        }
                        bulk_commit_group();
                    }
                }
            }
        }
        if (elected) bulk_wait_all();                      // all tensor stores have landed
    }
}

template <int BN, bool RELU6>
__global__ void __launch_bounds__(CV_THREADS, 1)
conv_tc_tf32x3_kernel(const __grid_constant__ CUtensorMap tm_in, const __grid_constant__ CUtensorMap tm_w,
                      const __grid_constant__ CUtensorMap tm_o0, const __grid_constant__ CUtensorMap tm_o1,
                      const __grid_constant__ CUtensorMap tm_o2, const __grid_constant__ CUtensorMap tm_o3,
                      const __grid_constant__ ConvParams p, const int reduce) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* smem = smem_raw + (smem_base - smem_u32(smem_raw));
    // carve-up: [stages x (A 16 KB | B high bn x 128 B | B low bn x 128 B)][2 staging tiles][barriers]
    const uint32_t stg_off = (uint32_t)p.stages * (uint32_t)p.stage_bytes;
    const uint32_t bar_off = stg_off + 2u * (uint32_t)kConvStg;
    ConvBarriers* bars = reinterpret_cast<ConvBarriers*>(smem + bar_off);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        // a stage is released by every consumer warp: each one reads its A fragment with its own shared loads
        for (int i = 0; i < kConvMaxStages; ++i) { mbar_init(smem_u32(&bars->full[i]), 1); mbar_init(smem_u32(&bars->empty[i]), 8); }
        fence_barrier_init();
    }
    if (warp == CV_WARP_TMA && lane == 0) {
        tma_prefetch_desc(&tm_in); tma_prefetch_desc(&tm_w); tma_prefetch_desc(&tm_o0);
        if (p.upsample || p.phased) { tma_prefetch_desc(&tm_o1); tma_prefetch_desc(&tm_o2); tma_prefetch_desc(&tm_o3); }
    }
    pdl_launch_dependents();
    pdl_wait_prior_grid();
    __syncthreads();

    if (warp == CV_WARP_TMA) {
        // =========================== TMA producer ===========================
        // per phase of the item's group, per tap (ky, kx) and 32-channel K-block: the A box at the tap's offset (the OOB zero
        // fill is the padding and the channel tail) and the tap's two B boxes; a pointwise step is one phase with one tap
        if (lane == 0) {
            Ring r;
            for (int w = blockIdx.x; w < p.items; w += gridDim.x) {
                const ConvCoord c = conv_decode(p, w, BN);
                for (int code = c.code; code != 0xF; code >>= 4) {
                    const ConvPhase f = p.ph[code & 0xF];
                    for (int ky = 0; ky < f.ny; ++ky)
                        for (int kx = 0; kx < f.nx; ++kx) {
                            const int tap = f.tap0 + ky * f.nx + kx;
                            for (int kb = 0; kb < p.kblocks; ++kb, r.next((uint32_t)p.stages)) {
                                const uint32_t st = smem_base + r.s * (uint32_t)p.stage_bytes, bar = smem_u32(&bars->full[r.s]);
                                mbar_wait(smem_u32(&bars->empty[r.s]), r.ph ^ 1u);
                                mbar_expect_tx(bar, (uint32_t)p.stage_bytes);
                                tma_load_4d(st, &tm_in, bar, kb * 32, c.ox0 + f.dx0 + kx, c.oy0 + f.dy0 + ky, c.img0);
                                tma_load_4d(st + CV_A_BYTES, &tm_w, bar, kb * 32, tap, c.n0, 0);             // high part
                                tma_load_4d(st + CV_A_BYTES + BN * 128, &tm_w, bar, kb * 32, tap, c.n0, 1);  // low part
                            }
                        }
                }
            }
        }
    } else {
        // =========================== consumer warpgroups: split + wgmma + epilogue ===========================
        const int wg = warp >> 2, wq = warp & 3;
        const int r0 = wg * 64 + wq * 16 + (lane >> 2), cq = (lane & 3) * 2, t = lane & 3;
        const uint32_t sw = (uint32_t)(lane >> 2);     // r0 & 7 == (r0 + 8) & 7: the row's 16-byte chunk swizzle
        const bool releaser = lane == 0;
        const bool elected = warp == 0 && lane == 0;
        constexpr uint32_t bar_id = 1u, bar_n = 256u;
        Ring r;
        uint32_t stg_flip = 0;
        for (int w = blockIdx.x; w < p.items; w += gridDim.x) {
            const ConvCoord c = conv_decode(p, w, BN);
            for (int code = c.code; code != 0xF; code >>= 4) {           // the phases of this item's group, one after the other
                const int q = code & 0xF;
                const int ksteps = p.ph[q].ny * p.ph[q].nx * p.kblocks;
                float acc[BN / 2];
#pragma unroll
                for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
                for (int k = 0; k < ksteps; ++k) {
                    mbar_wait(smem_u32(&bars->full[r.s]), r.ph);
                    const uint32_t st = smem_base + r.s * (uint32_t)p.stage_bytes;
                    const uint8_t* a_tile = smem + r.s * (uint32_t)p.stage_bytes;
                    // this thread's A fragments of the four k8 steps: channel 8 k4 + t (+ 4) of rows r0 and r0 + 8, split
                    uint32_t a_hi[4][4], a_lo[4][4];
#pragma unroll
                    for (int k4 = 0; k4 < 4; ++k4)
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            const int row = r0 + (e & 1) * 8, ch = 8 * k4 + t + (e >> 1) * 4;
                            const float v = *reinterpret_cast<const float*>(a_tile + row * 128 + ((((uint32_t)ch >> 2) ^ sw) << 4) + (ch & 3) * 4);
                            a_hi[k4][e] = rna_tf32(v);
                            a_lo[k4][e] = rna_tf32(v - __uint_as_float(a_hi[k4][e]));
                        }
                    const uint32_t bh = sw128_desc_lo(st + CV_A_BYTES), bl = sw128_desc_lo(st + CV_A_BYTES + BN * 128);
                    wgmma_fence();
#pragma unroll
                    for (int k4 = 0; k4 < 4; ++k4) {               // +32 B (8 fp32 channels) per k8 step inside the 128-byte row
                        wgmma_tf32_bn<BN>(acc, a_lo[k4], sw128_desc(bh + 2u * k4), (k > 0 || k4 > 0) ? 1u : 0u);
                        wgmma_tf32_bn<BN>(acc, a_hi[k4], sw128_desc(bl + 2u * k4), 1u);
                        wgmma_tf32_bn<BN>(acc, a_hi[k4], sw128_desc(bh + 2u * k4), 1u);
                    }
                    wgmma_commit();
                    // the A registers are rewritten by the next step: wait for this step's MMAs, then release the stage
                    wgmma_wait0();
                    if (releaser) mbar_arrive(smem_u32(&bars->empty[r.s]));
                    r.next((uint32_t)p.stages);
                }

                // per block of 32 output channels: registers -> BN affine + act (fp32) -> staging tile [128 px][32 ch] fp32
                // (16-byte chunks XOR-swizzled like a SWIZZLE_128B box) -> TMA tensor stores or reduce-adds
#pragma unroll
                for (int cb = 0; cb < BN / 32; ++cb) {
                    if (c.n0 + cb * 32 >= p.c_out) break;
                    uint8_t* stg = smem + stg_off + (stg_flip & 1u) * (uint32_t)kConvStg;
                    ++stg_flip;
                    const float2* aff = p.affine + c.n0 + cb * 32;
#pragma unroll
                    for (int i = 0; i < 4; ++i) {                  // 8-column group i of this block
                        const float4 af = __ldg(reinterpret_cast<const float4*>(aff + i * 8 + cq));     // (s0, s1, b0, b1)
                        const int j = cb * 4 + i, cl = i * 8 + cq;
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            const int rr = r0 + 8 * h;
                            float v0 = fmaxf(fmaf(acc[4 * j + 2 * h], af.x, af.z), 0.0f);
                            float v1 = fmaxf(fmaf(acc[4 * j + 2 * h + 1], af.y, af.w), 0.0f);
                            if (RELU6) { v0 = fminf(v0, 6.0f); v1 = fminf(v1, 6.0f); }
                            *reinterpret_cast<float2*>(stg + rr * 128 + ((((uint32_t)cl >> 2) ^ sw) << 4) + (cl & 3) * 4) = make_float2(v0, v1);
                        }
                    }
                    fence_proxy_async();
                    if (elected) bulk_wait_read0();
                    asm volatile("bar.sync %0, %1;" ::"r"(bar_id), "r"(bar_n) : "memory");
                    if (elected) {
                        const uint32_t src = smem_u32(stg);
                        const int cc = c.n0 + cb * 32;
                        // phased: phase q through view q; else view 0, or all four views of the nearest x2 map
                        const int v0 = p.phased ? q : 0, v1 = p.phased ? q + 1 : (p.upsample ? 4 : 1);
                        for (int v = v0; v < v1; ++v) {
                            const CUtensorMap* m = v == 0 ? &tm_o0 : v == 1 ? &tm_o1 : v == 2 ? &tm_o2 : &tm_o3;
                            if (reduce) tma_reduce_add_4d(m, src, cc, c.ox0, c.oy0, c.img0);
                            else tma_store_4d(m, src, cc, c.ox0, c.oy0, c.img0);
                        }
                        bulk_commit_group();
                    }
                }
            }
        }
        if (elected) bulk_wait_all();
    }
}

// The depthwise half of a 16-bit DWPW stage on its own: k x k taps (stride 1 or 2) + fp32 affine + act, one rounding to 16
// bits, NHWC in (in_pitch elements per pixel) -> dense NHWC mid.  One thread per PX neighbouring outputs of a row and 8
// channels.  It follows block_tc_kernel's depthwise warps step by step: taps rounded to the storage dtype (as pack_dwp_kernel does), inputs and
// taps widened to fp32, one fp32 FMA per tap with ky outer and kx inner, then ffma2_abc + pack_act.  The block kernel also
// adds the zero-filled taps outside the map; skipping them is the same, since an accumulator that starts at +0 never becomes
// -0 under round-to-nearest and x + 0 == x otherwise.
template <typename T, int K, bool RELU6, int PX>
__global__ void __launch_bounds__(256)
dw_mid_kernel(const T* __restrict__ in, T* __restrict__ mid, const float* __restrict__ w, const float* __restrict__ scale,
              const float* __restrict__ bias, int n, int h_in, int w_in, int h_out, int w_out, int c, int in_pitch, int stride) {
    using MF = MixFma<T>;
    const int groups = c >> 3, segs = (w_out + PX - 1) / PX;
    const long long total = (long long)n * h_out * segs * groups;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int g = (int)(idx % groups);
    long long t = idx / groups;
    const int ox0 = (int)(t % segs) * PX;
    const int oy = (int)((t / segs) % h_out);
    const int img = (int)(t / ((long long)segs * h_out));
    constexpr int PAD = (K - 1) / 2;
    auto rt = [](float v) { return Traits<T>::to_f(Traits<T>::from_f(v)); };
    f32x2 acc[PX][4];
#pragma unroll
    for (int o = 0; o < PX; ++o)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[o][j] = 0ull;
    const T* base = in + (size_t)img * h_in * w_in * in_pitch + g * 8;
    // a thread owns PX neighbouring outputs of one row: every input pixel of a kernel row is loaded and widened once and
    // feeds up to K of them; for each output the taps still arrive ky outer, kx inner (input column ascending)
    auto row = [&](auto stride_c, int ky) {
        constexpr int S = decltype(stride_c)::value;
        const int iy = oy * S - PAD + ky;
        if (iy < 0 || iy >= h_in) return;
        f32x2 wk[K][4];
#pragma unroll
        for (int kx = 0; kx < K; ++kx) {
            const float4* wp = reinterpret_cast<const float4*>(w + (size_t)(ky * K + kx) * c + g * 8);
            const float4 w0 = __ldg(wp), w1 = __ldg(wp + 1);
            wk[kx][0] = f32x2_make(rt(w0.x), rt(w0.y)); wk[kx][1] = f32x2_make(rt(w0.z), rt(w0.w));
            wk[kx][2] = f32x2_make(rt(w1.x), rt(w1.y)); wk[kx][3] = f32x2_make(rt(w1.z), rt(w1.w));
        }
#pragma unroll
        for (int j = 0; j < (PX - 1) * S + K; ++j) {
            const int ix = ox0 * S - PAD + j;
            if (ix < 0 || ix >= w_in) continue;
            const uint4 v = __ldg(reinterpret_cast<const uint4*>(base + ((size_t)iy * w_in + ix) * in_pitch));
            const f32x2 x0 = MF::widen(v.x), x1 = MF::widen(v.y), x2 = MF::widen(v.z), x3 = MF::widen(v.w);
#pragma unroll
            for (int o = 0; o < PX; ++o) {
                const int kx = j - o * S;
                if (kx < 0 || kx >= K) continue;
                ffma2(acc[o][0], x0, wk[kx][0]); ffma2(acc[o][1], x1, wk[kx][1]);
                ffma2(acc[o][2], x2, wk[kx][2]); ffma2(acc[o][3], x3, wk[kx][3]);
            }
        }
    };
#pragma unroll
    for (int ky = 0; ky < K; ++ky) {
        if (stride == 1) row(std::integral_constant<int, 1>(), ky);
        else row(std::integral_constant<int, 2>(), ky);
    }
    const float4* sp = reinterpret_cast<const float4*>(scale + g * 8);
    const float4* bp = reinterpret_cast<const float4*>(bias + g * 8);
    const float4 s0 = __ldg(sp), s1 = __ldg(sp + 1), b0 = __ldg(bp), b1 = __ldg(bp + 1);
    T* orow = mid + (((size_t)img * h_out + oy) * w_out) * c + g * 8;
#pragma unroll
    for (int o = 0; o < PX; ++o) {
        if (ox0 + o >= w_out) break;
        uint4 r;
        r.x = MF::template pack_act<RELU6>(ffma2_abc(acc[o][0], f32x2_make(s0.x, s0.y), f32x2_make(b0.x, b0.y)));
        r.y = MF::template pack_act<RELU6>(ffma2_abc(acc[o][1], f32x2_make(s0.z, s0.w), f32x2_make(b0.z, b0.w)));
        r.z = MF::template pack_act<RELU6>(ffma2_abc(acc[o][2], f32x2_make(s1.x, s1.y), f32x2_make(b1.x, b1.y)));
        r.w = MF::template pack_act<RELU6>(ffma2_abc(acc[o][3], f32x2_make(s1.z, s1.w), f32x2_make(b1.z, b1.w)));
        *reinterpret_cast<uint4*>(orow + (size_t)(ox0 + o) * c) = r;
    }
}

// ----------------------------------------------------------------------------------------------
// host side
// ----------------------------------------------------------------------------------------------
struct ConvTcPlan {
    CUtensorMap tm_in, tm_w, tm_o[4];
    ConvParams p;
    ConvPlanOut po;
    dim3 grid;
    size_t smem_bytes;
    int dtype, act;
    TcLaunchOpts opts;
    float2* affine = nullptr;
    size_t affine_bytes = 0;
    int tf32x3 = 0, reduce = 0;
    std::string name;
};

// w_hi = rna_tf32(w), w_lo = rna_tf32(w - w_hi) (w - w_hi is exact in fp32)
__global__ void split_tf32_kernel(const float* __restrict__ w, float* __restrict__ dst, int count) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < count) {
        const float v = w[i];
        const float hi = __uint_as_float(rna_tf32(v));
        dst[i] = hi;
        dst[count + i] = __uint_as_float(rna_tf32(v - hi));
    }
}

__global__ void pack_conv_affine_kernel(const float* __restrict__ scale, const float* __restrict__ bias, float2* __restrict__ dst,
                                        int c_out, int n_pad) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    // per channel PAIR (2j, 2j+1): (scale, scale, bias, bias), one 16-byte load feeds the pair (same layout as the block kernel)
    if (i < n_pad) {
        float* d = reinterpret_cast<float*>(dst) + (i >> 1) * 4;
        d[i & 1] = i < c_out ? scale[i] : 0.f;
        d[2 + (i & 1)] = i < c_out ? bias[i] : 0.f;
    }
}

bool conv_tc_supported(int dtype, const StageGeom& g, int kind) {
    if (dtype != FD_F16 && dtype != FD_BF16) return false;
    if (g.c_in % 8 || g.c_out % 8) return false;
    if (kind == kConvKindConv && ((g.ksize != 3 && g.ksize != 5) || g.stride != 1)) return false;
    return get_tensor_map_encoder() != nullptr;
}

void conv_tc_destroy(ConvTcPlan* cp) {
    if (!cp) return;
    cudaFree(cp->affine);
    delete cp;
}

ConvPlanOut conv_tc_debug_plan(int kind, int ksize, int h_out, int w_out, int n, int c_in, int c_out, int n_sms) {
    ConvPlanIn q{};
    q.ksize = ksize; q.h_out = h_out; q.w_out = w_out; q.n = n; q.c_in = c_in; q.c_out = c_out; q.n_sms = n_sms;
    q.force_tile = -1; q.kind = kind;
    return plan_conv(q);
}

// FD_CONV_TILE=<index into kConvTiles> / FD_CONV_BN=64|128|256 / FD_CONV_PHASE_GROUP=1|2 (phases per item of a DECONV / UPCONV
// stage) pin the planner's choice (tests: the result must not depend on it).  `kind` is kConvKind*; a DECONV / UPCONV stage
// passes its input map as g.h_out / g.w_out (the conv resolution) and writes the 2x map through the four phase views.
static int conv_prepare(int dtype, int kind, const StageGeom& g, const void* in, const void* w, const float* scale_dev,
                        const float* bias_dev, void* out, int reduce, const TcLaunchOpts& opts, ConvTcPlan** res) {
    PFN_encodeTiled encode = get_tensor_map_encoder();
    if (!encode) return fail(FD_ERR_CUDA, "cuTensorMapEncodeTiled is not available from this driver");
    const bool phased = kind != kConvKindConv;
    ConvPlanIn q{};
    q.ksize = g.ksize; q.h_out = g.h_out; q.w_out = g.w_out; q.n = g.n; q.c_in = g.c_in; q.c_out = g.c_out; q.upsample = g.upsample;
    q.n_sms = opts.n_sms; q.force_tile = -1; q.kind = kind;
    { const char* e = getenv("FD_CONV_TILE"); if (e && *e) q.force_tile = atoi(e); }
    { const char* e = getenv("FD_CONV_BN"); if (e && *e) q.force_bn = atoi(e); }
    { const char* e = getenv("FD_CONV_PHASE_GROUP"); if (phased && e && *e) q.force_group = atoi(e); }
    const ConvPlanOut po = plan_conv(q);
    if (!po.ok) return fail(FD_ERR_UNSUPPORTED, "dense conv stage: no tile plan fits shared memory");
    ConvTcPlan* cp = new (std::nothrow) ConvTcPlan();
    if (!cp) return fail(FD_ERR_CUDA, "out of host memory");
    cp->dtype = dtype; cp->act = g.act; cp->opts = opts; cp->po = po; cp->reduce = reduce;
    ConvParams& p = cp->p;
    memset(&p, 0, sizeof(p));
    p.n = g.n; p.h = g.h_out; p.w = g.w_out; p.c_in = g.c_in; p.c_out = g.c_out;
    p.ni = po.ni; p.th = po.th; p.tw = po.tw;
    p.tiles_x = (g.w_out + po.tw - 1) / po.tw; p.tiles_y = (g.h_out + po.th - 1) / po.th; p.img_tiles = (g.n + po.ni - 1) / po.ni;
    p.splits = po.n_splits; p.items = po.items;
    p.kblocks = po.kblocks;
    p.stages = po.stages; p.stage_bytes = conv_stage_bytes(po.bn);
    p.upsample = g.upsample; p.phased = phased ? 1 : 0;
    memcpy(p.ph, po.ph, sizeof(p.ph));
    for (int g = 0; g < 4; ++g) {
        p.group_code[g] = 0xF;
        for (int j = 1; j >= 0; --j)
            if (po.group_ph[g][j] >= 0) p.group_code[g] = (p.group_code[g] << 4) | po.group_ph[g][j];
    }
    auto magic = [](int d) { return (unsigned long long)((1ULL << 40) / (unsigned long long)d) + 1ULL; };
    p.mg_splits = magic(p.splits); p.mg_tx = magic(p.tiles_x); p.mg_ty = magic(p.tiles_y); p.mg_img = magic(p.img_tiles);
    const int n_pad = p.splits * po.bn;
    cp->affine_bytes = (size_t)n_pad * sizeof(float2);
    if (cudaMalloc(&cp->affine, cp->affine_bytes) != cudaSuccess) { conv_tc_destroy(cp); return fail(FD_ERR_CUDA, "cudaMalloc failed"); }
    pack_conv_affine_kernel<<<(n_pad + 127) / 128, 128>>>(scale_dev, bias_dev, cp->affine, g.c_out, n_pad);
    if (cudaGetLastError() != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) { conv_tc_destroy(cp); return fail(FD_ERR_CUDA, "conv affine packing failed"); }
    p.affine = cp->affine;

    const size_t es = 2;
    const CUtensorMapDataType dt = dtype == FD_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
    const int in_pitch = g.in_pitch > 0 ? g.in_pitch : g.c_in;
    {   // input: NHWC viewed as (C, W, H, N); box (64, tw, th, ni); 128B swizzle == the wgmma A layout; OOB -> 0 (padding, channel tail)
        cuuint64_t dims[4] = {(cuuint64_t)g.c_in, (cuuint64_t)g.w_in, (cuuint64_t)g.h_in, (cuuint64_t)g.n};
        cuuint64_t strides[3] = {(cuuint64_t)in_pitch * es, (cuuint64_t)g.w_in * in_pitch * es, (cuuint64_t)g.h_in * g.w_in * in_pitch * es};
        cuuint32_t box[4] = {64, (cuuint32_t)po.tw, (cuuint32_t)po.th, (cuuint32_t)po.ni};
        cuuint32_t estr[4] = {1, 1, 1, 1};
        CUresult r = encode(&cp->tm_in, dt, 4, const_cast<void*>(in), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { conv_tc_destroy(cp); return fail(FD_ERR_CUDA, "cuTensorMapEncodeTiled(conv input) failed: " + std::to_string((int)r)); }
    }
    {   // weights [c_out][k*k][c_in] (phase-major taps) viewed as (C_in, taps, C_out); box (64, 1, bn) lands as bn K-major rows
        const int taps = g.ksize * g.ksize;
        cuuint64_t dims[3] = {(cuuint64_t)g.c_in, (cuuint64_t)taps, (cuuint64_t)g.c_out};
        cuuint64_t strides[2] = {(cuuint64_t)g.c_in * es, (cuuint64_t)taps * g.c_in * es};
        cuuint32_t box[3] = {64, 1, (cuuint32_t)po.bn};
        cuuint32_t estr[3] = {1, 1, 1};
        CUresult r = encode(&cp->tm_w, dt, 3, const_cast<void*>(w), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { conv_tc_destroy(cp); return fail(FD_ERR_CUDA, "cuTensorMapEncodeTiled(conv weights) failed: " + std::to_string((int)r)); }
    }
    // output views: plain NHWC, or the four (dy, dx) phases of the 2x map (nearest upsample, or the phases of a DECONV / UPCONV)
    memset(cp->tm_o, 0, sizeof(cp->tm_o));
    {
        const bool views4 = g.upsample || phased;
        const int up = views4 ? 2 : 1;
        const cuuint64_t P = (cuuint64_t)(g.out_pitch > 0 ? g.out_pitch : g.c_out);
        const cuuint64_t W2 = (cuuint64_t)g.w_out * up, H2 = (cuuint64_t)g.h_out * up;
        for (int d = 0; d < (views4 ? 4 : 1); ++d) {
            char* base = reinterpret_cast<char*>(out) + ((size_t)(d >> 1) * W2 + (d & 1)) * P * es;
            cuuint64_t dims[4] = {(cuuint64_t)g.c_out, (cuuint64_t)g.w_out, (cuuint64_t)g.h_out, (cuuint64_t)g.n};
            cuuint64_t strides[3] = {up * P * es, up * W2 * P * es, H2 * W2 * P * es};
            cuuint32_t box[4] = {64, (cuuint32_t)po.tw, (cuuint32_t)po.th, (cuuint32_t)po.ni};
            cuuint32_t estr[4] = {1, 1, 1, 1};
            CUresult r = encode(&cp->tm_o[d], dt, 4, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            if (r != CUDA_SUCCESS) { conv_tc_destroy(cp); return fail(FD_ERR_CUDA, "cuTensorMapEncodeTiled(conv output) failed: " + std::to_string((int)r)); }
        }
    }
    cp->smem_bytes = (size_t)po.smem_bytes;
    cp->grid = dim3((unsigned)(p.items < opts.n_sms ? p.items : opts.n_sms), 1, 1);
    char buf[160];
    if (!phased)
        snprintf(buf, sizeof(buf), "conv_tc_kernel<k%d,bn%d,%s>[%dx%dx%d,n%d,st%d,%s%s]", g.ksize, po.bn, g.upsample ? "up" : "noup",
                 po.ni, po.th, po.tw, p.splits, p.stages, g.act == FD_ACT_RELU6 ? "relu6" : "relu", reduce ? ",+skip(red)" : "");
    else   // 4ph: one phase per item; 4ph2: the diagonal phase pairs
        snprintf(buf, sizeof(buf), "conv_tc_kernel<%s%d,bn%d,%s>[%dx%dx%d,n%d,st%d,%s]", kind == kConvKindDeconv ? "deconv" : "upconv",
                 g.ksize, po.bn, po.groups == 2 ? "4ph2" : "4ph", po.ni, po.th, po.tw, p.splits, p.stages,
                 g.act == FD_ACT_RELU6 ? "relu6" : "relu");
    cp->name = buf;
    *res = cp;
    return FD_OK;
}

int conv_tc_prepare(int dtype, int kind, const StageGeom& g, const void* in, const void* w, const float* scale_dev,
                    const float* bias_dev, void* out, const TcLaunchOpts& opts, ConvTcPlan** res) {
    return conv_prepare(dtype, kind, g, in, w, scale_dev, bias_dev, out, 0, opts, res);
}

bool pw_tc_supported(int dtype, const StageGeom& g) {
    if (dtype != FD_F16 && dtype != FD_BF16) return false;
    return g.c_in % 8 == 0 && g.c_out % 8 == 0 && get_tensor_map_encoder() != nullptr;
}

// the 1x1 geometry of a DWPW stage's pointwise half: the dense intermediate in, rows of a matrix where nothing is upsampled
static StageGeom pw_geom(const StageGeom& g, int out_pitch) {
    StageGeom q = g;
    q.ksize = 1; q.stride = 1;
    conv_flat_rows(q.upsample, &q.n, &q.h_out, &q.w_out);
    q.h_in = q.h_out; q.w_in = q.w_out; q.in_pitch = g.c_in; q.out_pitch = out_pitch;
    return q;
}

ConvPlanOut pw_tc_debug_plan(int h_out, int w_out, int n, int c_in, int c_out, int upsample, int n_sms) {
    ConvPlanIn q{};
    q.ksize = 1; q.h_out = h_out; q.w_out = w_out; q.n = n; q.c_in = c_in; q.c_out = c_out; q.upsample = upsample;
    q.n_sms = n_sms; q.force_tile = -1; q.kind = kConvKindConv;
    conv_flat_rows(upsample, &q.n, &q.h_out, &q.w_out);
    return plan_conv(q);
}

// The pointwise half of a 16-bit DWPW stage as a 1x1 step of conv_tc_kernel: `mid` is the stage's depthwise intermediate
// (NHWC, c_in dense), `w` its pointwise weights [c_out][c_in]; `out` / `out_pitch` what the tiles are written to (g.upsample:
// the four views of the 2x map).  reduce = 1: the tiles are reduce-added into `out`, which already holds the skip tensor.
int pw_tc_prepare(int dtype, const StageGeom& g, const void* mid, const void* w, const float* scale_dev, const float* bias_dev,
                  void* out, int out_pitch, int reduce, const TcLaunchOpts& opts, ConvTcPlan** res) {
    return conv_prepare(dtype, kConvKindConv, pw_geom(g, out_pitch), mid, w, scale_dev, bias_dev, out, reduce, opts, res);
}

template <typename T, int PX>
static int dw_mid_launch_t(const BlockArgs& a, cudaStream_t st) {
    const StageGeom& g = a.g;
    const long long total = (long long)g.n * g.h_out * ((g.w_out + PX - 1) / PX) * (g.c_in / 8);
    const unsigned blocks = (unsigned)((total + 255) / 256);
    const int in_pitch = g.in_pitch > 0 ? g.in_pitch : g.c_in;
    const bool r6 = g.act == FD_ACT_RELU6;
#define FD_DW_MID(K, R6)                                                                                                           \
    dw_mid_kernel<T, K, R6, PX><<<blocks, 256, 0, st>>>(static_cast<const T*>(a.in), static_cast<T*>(a.mid), a.dw_w, a.dw_scale,  \
                                                        a.dw_bias, g.n, g.h_in, g.w_in, g.h_out, g.w_out, g.c_in, in_pitch, g.stride)
    if (g.ksize == 3) { if (r6) FD_DW_MID(3, true); else FD_DW_MID(3, false); }
    else if (g.ksize == 5) { if (r6) FD_DW_MID(5, true); else FD_DW_MID(5, false); }
    else return fail(FD_ERR_UNSUPPORTED, "no dw_mid_kernel instance for this kernel size");
#undef FD_DW_MID
    FD_CUDA_OK(cudaGetLastError());
    return FD_OK;
}

// The depthwise half of a 16-bit DWPW stage into a.mid (see dw_mid_kernel).
int dw_mid_launch(int dtype, const BlockArgs& a, cudaStream_t st) {
    if (dtype != FD_F16 && dtype != FD_BF16) return fail(FD_ERR_UNSUPPORTED, "dw_mid_kernel is a 16-bit kernel");
    // four outputs per thread: measured against one (more gathers) and eight (too few threads in flight), DESIGN 3.6a
    return dtype == FD_F16 ? dw_mid_launch_t<__half, 4>(a, st) : dw_mid_launch_t<__nv_bfloat16, 4>(a, st);
}

bool pw_tf32x3_supported(const StageGeom& g) {
    return g.c_in % 8 == 0 && g.c_out % 8 == 0 && get_tensor_map_encoder() != nullptr;
}

// the dense stages the split-TF32 step runs: CONV k in {3, 5} stride 1, DECONV k in {3, 5, 7, 9}, UPCONV k = 5
bool conv_tc_tf32x3_supported(const StageGeom& g, int kind) {
    if (g.c_in % 8 || g.c_out % 8) return false;
    if (kind == kConvKindConv && ((g.ksize != 3 && g.ksize != 5) || g.stride != 1)) return false;
    if (kind == kConvKindDeconv && g.ksize != 3 && g.ksize != 5 && g.ksize != 7 && g.ksize != 9) return false;
    if (kind == kConvKindUpconv && g.ksize != 5) return false;
    return get_tensor_map_encoder() != nullptr;
}

ConvPlanOut pw_tf32x3_debug_plan(int h_out, int w_out, int n, int c_in, int c_out, int upsample, int n_sms) {
    ConvPlanIn q{};
    q.ksize = 1; q.h_out = h_out; q.w_out = w_out; q.n = n; q.c_in = c_in; q.c_out = c_out; q.upsample = upsample;
    q.n_sms = n_sms; q.force_tile = -1; q.kind = kConvKindConv; q.tf32x3 = 1;
    return plan_conv(q);
}

ConvPlanOut conv_tc_tf32x3_debug_plan(int kind, int ksize, int h_out, int w_out, int n, int c_in, int c_out, int upsample,
                                      int n_sms) {
    ConvPlanIn q{};
    q.ksize = ksize; q.h_out = h_out; q.w_out = w_out; q.n = n; q.c_in = c_in; q.c_out = c_out; q.upsample = upsample;
    q.n_sms = n_sms; q.force_tile = -1; q.kind = kind; q.tf32x3 = 1;
    return plan_conv(q);
}

// One split-TF32 step.  kind / ksize: a 1x1 CONV (the pointwise half of a DWPW stage), a k x k CONV, or a DECONV / UPCONV
// as four phase convs at the input resolution.  `in` is NHWC fp32 of in_w x in_h pixels with in_pitch elements per pixel;
// `w_split` the fp32 weights [c_out][k*k][c_in] (phase-major taps) split into [2][c_out][k*k][c_in] (TF32 high, then
// low part, by tf32_split_weights; the caller owns it and may share it between steps); `out` / `out_pitch` what the tiles are written to (g.upsample: the four views of the 2x map; phased: phase q
// through view q).  reduce = 1: the tiles are reduce-added into `out`, which already holds the skip tensor.
// FD_CONV_TILE / FD_CONV_BN / FD_CONV_PHASE_GROUP pin the planner's choice as for conv_tc_prepare.
static int tf32x3_prepare(int kind, int ksize, const StageGeom& g, const void* in, int in_w, int in_h, int in_pitch,
                          const float* w_split, const float* scale_dev, const float* bias_dev, void* out, int out_pitch,
                          int reduce, const TcLaunchOpts& opts, ConvTcPlan** res) {
    PFN_encodeTiled encode = get_tensor_map_encoder();
    if (!encode) return fail(FD_ERR_CUDA, "cuTensorMapEncodeTiled is not available from this driver");
    const bool phased = kind != kConvKindConv;
    const bool pw = ksize == 1;
    ConvPlanIn q{};
    q.ksize = ksize; q.h_out = g.h_out; q.w_out = g.w_out; q.n = g.n; q.c_in = g.c_in; q.c_out = g.c_out; q.upsample = g.upsample;
    q.n_sms = opts.n_sms; q.force_tile = -1; q.kind = kind; q.tf32x3 = 1;
    { const char* e = getenv("FD_CONV_TILE"); if (e && *e) q.force_tile = atoi(e); }
    { const char* e = getenv("FD_CONV_BN"); if (e && *e) q.force_bn = atoi(e); }
    { const char* e = getenv("FD_CONV_PHASE_GROUP"); if (phased && e && *e) q.force_group = atoi(e); }
    const ConvPlanOut po = plan_conv(q);
    if (!po.ok) return fail(FD_ERR_UNSUPPORTED, "tf32x3 conv step: no tile plan fits shared memory");
    ConvTcPlan* cp = new (std::nothrow) ConvTcPlan();
    if (!cp) return fail(FD_ERR_CUDA, "out of host memory");
    cp->dtype = FD_F32; cp->act = g.act; cp->opts = opts; cp->po = po; cp->tf32x3 = 1; cp->reduce = reduce;
    ConvParams& p = cp->p;
    memset(&p, 0, sizeof(p));
    p.n = g.n; p.h = g.h_out; p.w = g.w_out; p.c_in = g.c_in; p.c_out = g.c_out;
    p.ni = po.ni; p.th = po.th; p.tw = po.tw;
    p.tiles_x = (g.w_out + po.tw - 1) / po.tw; p.tiles_y = (g.h_out + po.th - 1) / po.th; p.img_tiles = (g.n + po.ni - 1) / po.ni;
    p.splits = po.n_splits; p.items = po.items;
    p.kblocks = po.kblocks;
    p.stages = po.stages; p.stage_bytes = conv_stage_bytes_tf32x3(po.bn);
    p.upsample = g.upsample; p.phased = phased ? 1 : 0;
    memcpy(p.ph, po.ph, sizeof(p.ph));
    for (int i = 0; i < 4; ++i) {
        p.group_code[i] = 0xF;
        for (int j = 1; j >= 0; --j)
            if (po.group_ph[i][j] >= 0) p.group_code[i] = (p.group_code[i] << 4) | po.group_ph[i][j];
    }
    auto magic = [](int d) { return (unsigned long long)((1ULL << 40) / (unsigned long long)d) + 1ULL; };
    p.mg_splits = magic(p.splits); p.mg_tx = magic(p.tiles_x); p.mg_ty = magic(p.tiles_y); p.mg_img = magic(p.img_tiles);
    const int n_pad = p.splits * po.bn;
    const int taps = ksize * ksize;
    const size_t wcount = (size_t)g.c_out * taps * g.c_in;
    cp->affine_bytes = (size_t)n_pad * sizeof(float2);
    if (cudaMalloc(&cp->affine, cp->affine_bytes) != cudaSuccess) { conv_tc_destroy(cp); return fail(FD_ERR_CUDA, "cudaMalloc failed"); }
    pack_conv_affine_kernel<<<(n_pad + 127) / 128, 128>>>(scale_dev, bias_dev, cp->affine, g.c_out, n_pad);
    if (cudaGetLastError() != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) { conv_tc_destroy(cp); return fail(FD_ERR_CUDA, "tf32x3 affine packing failed"); }
    p.affine = cp->affine;

    const size_t es = 4;
    const CUtensorMapDataType dt = CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
    {   // input: NHWC (C, W, H, N), box (32, tw, th, ni); OOB -> 0 (the conv's zero padding and the channel tail of the last K-block)
        cuuint64_t dims[4] = {(cuuint64_t)g.c_in, (cuuint64_t)in_w, (cuuint64_t)in_h, (cuuint64_t)g.n};
        cuuint64_t strides[3] = {(cuuint64_t)in_pitch * es, (cuuint64_t)in_w * in_pitch * es, (cuuint64_t)in_h * in_w * in_pitch * es};
        cuuint32_t box[4] = {32, (cuuint32_t)po.tw, (cuuint32_t)po.th, (cuuint32_t)po.ni};
        cuuint32_t estr[4] = {1, 1, 1, 1};
        CUresult r = encode(&cp->tm_in, dt, 4, const_cast<void*>(in), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { conv_tc_destroy(cp); return fail(FD_ERR_CUDA, "cuTensorMapEncodeTiled(tf32x3 input) failed: " + std::to_string((int)r)); }
    }
    {   // split weights [2][c_out][k*k][c_in] viewed as (C_in, taps, C_out, part); box (32, 1, bn, 1) lands as bn K-major rows
        cuuint64_t dims[4] = {(cuuint64_t)g.c_in, (cuuint64_t)taps, (cuuint64_t)g.c_out, 2};
        cuuint64_t strides[3] = {(cuuint64_t)g.c_in * es, (cuuint64_t)taps * g.c_in * es, (cuuint64_t)wcount * es};
        cuuint32_t box[4] = {32, 1, (cuuint32_t)po.bn, 1};
        cuuint32_t estr[4] = {1, 1, 1, 1};
        CUresult r = encode(&cp->tm_w, dt, 4, const_cast<float*>(w_split), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { conv_tc_destroy(cp); return fail(FD_ERR_CUDA, "cuTensorMapEncodeTiled(tf32x3 weights) failed: " + std::to_string((int)r)); }
    }
    memset(cp->tm_o, 0, sizeof(cp->tm_o));
    {   // plain NHWC, or the four (dy, dx) views of the 2x map (nearest upsample, or the phases of a DECONV / UPCONV)
        const bool views4 = g.upsample || phased;
        const int up = views4 ? 2 : 1;
        const cuuint64_t P = (cuuint64_t)out_pitch;
        const cuuint64_t W2 = (cuuint64_t)g.w_out * up, H2 = (cuuint64_t)g.h_out * up;
        for (int d = 0; d < (views4 ? 4 : 1); ++d) {
            char* base = reinterpret_cast<char*>(out) + ((size_t)(d >> 1) * W2 + (d & 1)) * P * es;
            cuuint64_t dims[4] = {(cuuint64_t)g.c_out, (cuuint64_t)g.w_out, (cuuint64_t)g.h_out, (cuuint64_t)g.n};
            cuuint64_t strides[3] = {up * P * es, up * W2 * P * es, H2 * W2 * P * es};
            cuuint32_t box[4] = {32, (cuuint32_t)po.tw, (cuuint32_t)po.th, (cuuint32_t)po.ni};
            cuuint32_t estr[4] = {1, 1, 1, 1};
            CUresult r = encode(&cp->tm_o[d], dt, 4, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            if (r != CUDA_SUCCESS) { conv_tc_destroy(cp); return fail(FD_ERR_CUDA, "cuTensorMapEncodeTiled(tf32x3 output) failed: " + std::to_string((int)r)); }
        }
    }
    cp->smem_bytes = (size_t)po.smem_bytes;
    cp->grid = dim3((unsigned)(p.items < opts.n_sms ? p.items : opts.n_sms), 1, 1);
    char buf[160];
    const char* act = g.act == FD_ACT_RELU6 ? "relu6" : "relu";
    if (pw)
        snprintf(buf, sizeof(buf), "conv_tc_kernel<pw,tf32x3,bn%d,%s>[%dx%dx%d,n%d,st%d,%s%s]", po.bn, g.upsample ? "up" : "noup",
                 po.ni, po.th, po.tw, p.splits, p.stages, act, reduce ? ",+skip(red)" : "");
    else if (!phased)
        snprintf(buf, sizeof(buf), "conv_tc_kernel<k%d,tf32x3,bn%d,%s>[%dx%dx%d,n%d,st%d,%s]", ksize, po.bn,
                 g.upsample ? "up" : "noup", po.ni, po.th, po.tw, p.splits, p.stages, act);
    else
        snprintf(buf, sizeof(buf), "conv_tc_kernel<%s%d,tf32x3,bn%d,%s>[%dx%dx%d,n%d,st%d,%s]",
                 kind == kConvKindDeconv ? "deconv" : "upconv", ksize, po.bn, po.groups == 2 ? "4ph2" : "4ph", po.ni, po.th, po.tw,
                 p.splits, p.stages, act);
    cp->name = buf;
    *res = cp;
    return FD_OK;
}

// The split-TF32 pointwise step of an fp32 DWPW stage: `mid` is the stage's depthwise intermediate (NHWC fp32, c_in dense),
// `w_split` its split pointwise weights [2][c_out][c_in].
int pw_tf32x3_prepare(const StageGeom& g, const void* mid, const float* w_split, const float* scale_dev, const float* bias_dev,
                      void* out, int out_pitch, int reduce, const TcLaunchOpts& opts, ConvTcPlan** res) {
    return tf32x3_prepare(kConvKindConv, 1, g, mid, g.w_out, g.h_out, g.c_in, w_split, scale_dev, bias_dev, out, out_pitch, reduce,
                          opts, res);
}

// The split-TF32 step of a dense fp32 CONV / DECONV / UPCONV stage (arguments as for conv_tc_prepare; `w_split` is the
// repacked fp32 [c_out][k*k][c_in] split into [2][c_out][k*k][c_in]).
int conv_tc_tf32x3_prepare(int kind, const StageGeom& g, const void* in, const float* w_split, const float* scale_dev,
                           const float* bias_dev, void* out, const TcLaunchOpts& opts, ConvTcPlan** res) {
    return tf32x3_prepare(kind, g.ksize, g, in, g.w_in, g.h_in, g.in_pitch > 0 ? g.in_pitch : g.c_in, w_split, scale_dev, bias_dev, out,
                          g.out_pitch > 0 ? g.out_pitch : g.c_out, 0, opts, res);
}

// Split `count` fp32 weights into dst[2][count]: the TF32 high parts, then the low parts.  Synchronous.
int tf32_split_weights(const float* w, size_t count, float* dst) {
    if (count > (size_t)INT32_MAX) return fail(FD_ERR_UNSUPPORTED, "tf32x3: weights too large");
    split_tf32_kernel<<<(unsigned)((count + 255) / 256), 256>>>(w, dst, (int)count);
    if (cudaGetLastError() != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) return fail(FD_ERR_CUDA, "tf32x3 weight split failed");
    return FD_OK;
}

size_t conv_tc_param_bytes(ConvTcPlan* cp) { return cp->affine_bytes; }

const char* conv_tc_name(ConvTcPlan* cp) { return cp->name.c_str(); }

template <typename T, int BN, bool RELU6>
static int conv_launch_inst(ConvTcPlan* cp, cudaStream_t st) {
    auto kern = conv_tc_kernel<T, BN, RELU6>;
    static PerDeviceOnce attr_set;             // the opt-in is per device (and per kernel instance)
    int dev = -1;
    FD_CUDA_OK(cudaGetDevice(&dev));
    if (attr_set.need(dev)) {
        FD_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        attr_set.done(dev);
    }
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = cp->grid; cfg.blockDim = dim3(CV_THREADS); cfg.dynamicSmemBytes = cp->smem_bytes; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = cp->opts.pdl ? 1 : 0;
    FD_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, cp->tm_in, cp->tm_w, cp->tm_o[0], cp->tm_o[1], cp->tm_o[2], cp->tm_o[3], cp->p,
                                  cp->reduce));
    FD_CUDA_OK(cudaGetLastError());
    return FD_OK;
}

template <typename T>
static int conv_launch_t(ConvTcPlan* cp, cudaStream_t st) {
    const bool r6 = cp->act == FD_ACT_RELU6;
    switch (cp->po.bn) {
        case 64: return r6 ? conv_launch_inst<T, 64, true>(cp, st) : conv_launch_inst<T, 64, false>(cp, st);
        case 128: return r6 ? conv_launch_inst<T, 128, true>(cp, st) : conv_launch_inst<T, 128, false>(cp, st);
        case 256: return r6 ? conv_launch_inst<T, 256, true>(cp, st) : conv_launch_inst<T, 256, false>(cp, st);
        default: return fail(FD_ERR_UNSUPPORTED, "no conv_tc_kernel instance for this bn");
    }
}

template <int BN, bool RELU6>
static int tf32x3_launch_inst(ConvTcPlan* cp, cudaStream_t st) {
    auto kern = conv_tc_tf32x3_kernel<BN, RELU6>;
    static PerDeviceOnce attr_set;
    int dev = -1;
    FD_CUDA_OK(cudaGetDevice(&dev));
    if (attr_set.need(dev)) {
        FD_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        attr_set.done(dev);
    }
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = cp->grid; cfg.blockDim = dim3(CV_THREADS); cfg.dynamicSmemBytes = cp->smem_bytes; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = cp->opts.pdl ? 1 : 0;
    FD_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, cp->tm_in, cp->tm_w, cp->tm_o[0], cp->tm_o[1], cp->tm_o[2], cp->tm_o[3], cp->p,
                                  cp->reduce));
    FD_CUDA_OK(cudaGetLastError());
    return FD_OK;
}

static int tf32x3_launch(ConvTcPlan* cp, cudaStream_t st) {
    const bool r6 = cp->act == FD_ACT_RELU6;
    switch (cp->po.bn) {
        case 64: return r6 ? tf32x3_launch_inst<64, true>(cp, st) : tf32x3_launch_inst<64, false>(cp, st);
        case 128: return r6 ? tf32x3_launch_inst<128, true>(cp, st) : tf32x3_launch_inst<128, false>(cp, st);
        default: return fail(FD_ERR_UNSUPPORTED, "no conv_tc_tf32x3_kernel instance for this bn");
    }
}

int conv_tc_launch(ConvTcPlan* cp, cudaStream_t st) {
    if (cp->tf32x3) return tf32x3_launch(cp, st);
    return cp->dtype == FD_F16 ? conv_launch_t<__half>(cp, st) : conv_launch_t<__nv_bfloat16>(cp, st);
}

}  // namespace fd
