// Chain kernel: a run of consecutive 3x3 stride-1 conv_dw blocks on a small feature map (conv7..conv11 of MobileNet at 14x14,
// reference imagenet/mobilenet.py:47-51 applied by models.py:710-712) executed as ONE kernel by thread-block clusters of two
// CTAs, one image per cluster, with every intermediate activation resident in shared memory -- no HBM round trip, no launch,
// no pipeline fill/drain between the layers.
//
//   * The CTA pair splits the image by ROWS (CTA 0: rows [0, rows0), CTA 1: the rest): each CTA keeps its rows plus one halo row
//     above and below for all channels, as <= 8 K-blocks of [9 rows][15 px][64 ch] (pixel pitch 15: column 14 is a zero column
//     that serves as the right padding of its row and the left padding of the next one), 128 B per pixel, 16-byte chunks
//     XOR-swizzled with the pixel slot index -- the SWIZZLE_128B pattern TMA writes and wgmma reads.
//   * Depthwise (16 warps, lane = channel pair, 2 columns x 7 rows per warp): reads a K-block's pixels,
//     and -- after the eight warps working on that K-block have all finished reading -- writes the 128 result rows IN PLACE over
//     the block in the K-major SWIZZLE_128B operand layout.  The block is then the A operand of that K-block; there is no
//     separate A ring (the shared memory holds 136 KB of activations + a 64 KB weight ring).
//   * Pointwise (the same 16 warps = four warpgroups): each CTA runs wgmma on its own 128 pixel slots with whole weight tiles
//     [128 output channels][64 K] streamed by its own TMA.  The output channels go in passes of 128: warpgroup (rh, ch) owns
//     rows [64 rh, 64 rh + 64) and columns [64 ch, 64 ch + 64) of the pass, accumulates over every K-block in registers
//     (wgmma.m64n64k16), applies BN + act and keeps the 16-bit result in registers -- the activation blocks are still the
//     A operand of the later passes.  After the last pass all results go into the NEXT layer's activation blocks in shared
//     memory; the boundary row also goes into the peer CTA's halo row (st.shared::cluster), then one remote mbarrier arrive
//     tells the peer its halo is complete.  The last layer stores to global memory instead.
//
// Layer boundaries therefore cost a named barrier + one DSMEM hand-shake instead of a kernel boundary; weights for the next
// K-blocks / layer stream through the 4-deep ring while the epilogue runs.
#include <cuda.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <string>
#include <vector>

#include "fd_tc_common.cuh"

namespace fd {

constexpr int CH_WORKERS = 16;                       // warps 0..15: depthwise + epilogue
constexpr int CH_WARP_TMA = 16;
constexpr int CH_THREADS = 17 * 32;
constexpr int CH_MAX_PASS = 4;                       // output channels per layer <= CH_MAX_PASS x 128
constexpr int CH_MAX_LAYERS = 8, CH_MAX_KB = 8;
constexpr int CH_PITCH = 15, CH_ROWS = 9;            // pixel slots: slot(r, c) = r * 15 + c, r in [0, 9), c in [0, 15)
constexpr int CH_BLK = 136 * 128;                    // 135 slots + 1 spare zero slot; 17 x 1024 B keeps every block 1 KB aligned
constexpr int CH_IN_BYTES = CH_ROWS * CH_PITCH * 128;   // bytes one TMA box of the first layer's input lands
constexpr int CH_SB = 4, CH_B_STAGE = 128 * 128;     // weight ring: 4 x [128 rows][64 K] 16-bit
constexpr int CH_SD = 4, CH_DWP = 9 * 128 + 512;     // depthwise parameter ring: {[9][64] taps, [64] fp32 scale, [64] fp32 bias}
constexpr int CH_AFF_BYTES = 512 * 8;                // pointwise BN affine of one layer: (scale, scale, bias, bias) per channel pair
constexpr int CH_OFF_ACT = 1024;
constexpr int CH_OFF_B = CH_OFF_ACT + CH_MAX_KB * CH_BLK;
constexpr int CH_OFF_DWP = CH_OFF_B + CH_SB * CH_B_STAGE;
constexpr int CH_OFF_AFF = CH_OFF_DWP + CH_SD * CH_DWP;
constexpr int CH_OFF_BAR = CH_OFF_AFF + 2 * CH_AFF_BYTES;

struct ChainBarriers {
    uint64_t in_full[CH_MAX_KB];        // layer-0 input block landed (TMA tx), once per image
    uint64_t a_full[CH_MAX_KB];         // the 8 depthwise warps of the K-block's group have written its operand tile, once per layer
    uint64_t b_full[CH_SB];             // weight tile landed (tx)
    uint64_t b_empty[CH_SB];            // all four warpgroups are done reading the stage
    uint64_t dwp_full[CH_SD], dwp_empty[CH_SD];
    uint64_t aff_full[2], aff_empty[2];
    uint64_t mma_done;                  // one remote arrival: the peer's warpgroups have finished reading their operand tiles, so
                                        // its halo rows (which the in-place tiles cover) may be overwritten
    uint64_t halo_full;                 // one remote arrival (cluster-scope release): the peer has written my halo row of the next layer
    uint64_t act_free;                  // the last layer's output has left the activation blocks (TMA stores have read them)
};
constexpr int CH_SMEM_BYTES = CH_OFF_BAR + (int)sizeof(ChainBarriers) + 1024;     // + alignment slack

struct ChainLayer {
    int c_in, c_out;
    int kblocks;           // ceil(c_in / 64)
    int np;                // passes of 128 output channels: ceil(n_pad / 128)
    int n_pad;             // c_out rounded up to 64 (accumulator columns in use; every written K-block is whole)
    int aff_bytes;         // n_pad * 8
    const void* dwp;       // [kblocks] x CH_DWP bytes
    const float2* affine;  // [n_pad]: (scale, scale, bias, bias) per channel PAIR (see pack_affine_kernel)
};

struct ChainParams {
    int n_img, h, w, rows0;            // CTA 0 owns image rows [0, rows0), CTA 1 rows [rows0, h)
    int n_layers;
    int out_pitch;                     // elements between pixels of the output tensor
    int sleep_ns;
    int n_zero[2];
    void* out;
    ChainLayer L[CH_MAX_LAYERS];
    unsigned long long* trace;         // debug timeline (fd_plan_trace_stage) or nullptr: [12 rows][256] SM clocks of the leader CTA of cluster 0
    unsigned char zero_slots[2][48];   // per cluster rank: pixel slots that must read as zero for the next layer (padding column,
                                       // image-border halo row); re-zeroed after every layer because the in-place operand tile
                                       // has overwritten slots 0..127
};

struct ChainMaps {
    CUtensorMap in;                    // first layer's input, NHWC as (C, W, H, N), box (64, 15, 9, 1), SWIZZLE_128B, OOB -> 0
    CUtensorMap w[CH_MAX_LAYERS];      // pointwise weights [c_out][c_in] as (K, N), box (64, 128), SWIZZLE_128B
    CUtensorMap out[2];                // last layer's output, NHWC as (C, W, H, N), per cluster rank: box (64, 15, rows of that rank, 1),
                                       // SWIZZLE_128B; column 14 and channels >= c_out are clipped by the hardware
};

__device__ __forceinline__ void st_cluster_u32(uint32_t cluster_addr, uint32_t v) {
    asm volatile("st.shared::cluster.b32 [%0], %1;" ::"r"(cluster_addr), "r"(v) : "memory");
}

#define CH_TRACE(row, idx)                                                                                \
    do {                                                                                                  \
        if (p.trace != nullptr && blockIdx.x == 0 && (idx) < 256) p.trace[(row) * 256 + (idx)] = clock64(); \
    } while (0)

// ----------------------------------------------------------------------------------------------------------
template <typename T, bool RELU6>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(CH_THREADS, 1)
chain_tc_kernel(const __grid_constant__ ChainMaps maps, const __grid_constant__ ChainParams p) {
    using MF = MixFma<T>;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* smem = smem_raw + (smem_base - smem_u32(smem_raw));
    ChainBarriers* bars = reinterpret_cast<ChainBarriers*>(smem + CH_OFF_BAR);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t rank = cluster_ctarank();
    const int cluster_id = blockIdx.x >> 1, n_clusters = gridDim.x >> 1;
    const int rows_local = rank == 0 ? p.rows0 : p.h - p.rows0;
    const int row_first = rank == 0 ? 0 : p.rows0;              // image row of local row 0

    if (threadIdx.x == 0) {
        for (int i = 0; i < CH_MAX_KB; ++i) { mbar_init(smem_u32(&bars->in_full[i]), 1); mbar_init(smem_u32(&bars->a_full[i]), CH_WORKERS / 2); }
        for (int i = 0; i < CH_SB; ++i) { mbar_init(smem_u32(&bars->b_full[i]), 1); mbar_init(smem_u32(&bars->b_empty[i]), CH_WORKERS / 4); }
        for (int i = 0; i < CH_SD; ++i) { mbar_init(smem_u32(&bars->dwp_full[i]), 1); mbar_init(smem_u32(&bars->dwp_empty[i]), CH_WORKERS / 2); }
        for (int i = 0; i < 2; ++i) { mbar_init(smem_u32(&bars->aff_full[i]), 1); mbar_init(smem_u32(&bars->aff_empty[i]), CH_WORKERS); }
        mbar_init(smem_u32(&bars->mma_done), 1);
        mbar_init(smem_u32(&bars->halo_full), 1);
        mbar_init(smem_u32(&bars->act_free), 1);
        fence_barrier_init();
    }
    // every activation slot starts as finite zeros (padding, channels a narrower layer never writes)
    for (int i = threadIdx.x; i < (CH_OFF_B) / 16; i += CH_THREADS) reinterpret_cast<uint4*>(smem)[i] = make_uint4(0u, 0u, 0u, 0u);
    fence_proxy_async();
    if (warp == CH_WARP_TMA && lane == 0) {
        tma_prefetch_desc(&maps.in);
        tma_prefetch_desc(&maps.out[rank]);
        for (int l = 0; l < p.n_layers; ++l) tma_prefetch_desc(&maps.w[l]);
    }
    pdl_launch_dependents();
    pdl_wait_prior_grid();                         // everything below reads what the previous kernel wrote
    cluster_sync_all();                            // barriers initialised + smem zeroed in BOTH CTAs before any remote access

    if (warp == CH_WARP_TMA) {
        // =========================== producers (single threads) ===========================
        if (lane == 0) {
            // pointwise weights: [128 output channels][64 K] tiles in the order the passes consume them, all layers, all images
            uint32_t seq = 0;
            for (int img = cluster_id; img < p.n_img; img += n_clusters)
                for (int l = 0; l < p.n_layers; ++l) {
                    const ChainLayer& L = p.L[l];
                    for (int ps = 0; ps < L.np; ++ps)
                        for (int kb = 0; kb < L.kblocks; ++kb, ++seq) {
                            const uint32_t s = seq & (CH_SB - 1), ph = (seq / CH_SB) & 1u;
                            mbar_wait_sleep(smem_u32(&bars->b_empty[s]), ph ^ 1u, (uint32_t)p.sleep_ns);
                            if (kb == 0 && ps == 0 && img == cluster_id) CH_TRACE(10, l);
                            mbar_expect_tx(smem_u32(&bars->b_full[s]), (uint32_t)CH_B_STAGE);
                            tma_load_2d(smem_base + CH_OFF_B + s * CH_B_STAGE, &maps.w[l], smem_u32(&bars->b_full[s]), kb * 64, ps * 128);
                        }
                }
        } else if (lane == 1) {
            // depthwise parameter blocks (ring) and the per-layer pointwise BN affine (double buffer)
            uint32_t dseq = 0, lseq = 0;
            for (int img = cluster_id; img < p.n_img; img += n_clusters)
                for (int l = 0; l < p.n_layers; ++l, ++lseq) {
                    const ChainLayer& L = p.L[l];
                    {
                        const uint32_t s = lseq & 1u, ph = (lseq >> 1) & 1u;
                        mbar_wait_sleep(smem_u32(&bars->aff_empty[s]), ph ^ 1u, (uint32_t)p.sleep_ns);
                        mbar_expect_tx(smem_u32(&bars->aff_full[s]), (uint32_t)L.aff_bytes);
                        bulk_load(smem_base + CH_OFF_AFF + s * CH_AFF_BYTES, L.affine, (uint32_t)L.aff_bytes, smem_u32(&bars->aff_full[s]));
                    }
                    for (int kb = 0; kb < L.kblocks; ++kb, ++dseq) {
                        const uint32_t s = dseq & (CH_SD - 1), ph = (dseq / CH_SD) & 1u;
                        mbar_wait_sleep(smem_u32(&bars->dwp_empty[s]), ph ^ 1u, (uint32_t)p.sleep_ns);
                        mbar_expect_tx(smem_u32(&bars->dwp_full[s]), (uint32_t)CH_DWP);
                        bulk_load(smem_base + CH_OFF_DWP + s * CH_DWP, reinterpret_cast<const uint8_t*>(L.dwp) + (size_t)kb * CH_DWP,
                                  (uint32_t)CH_DWP, smem_u32(&bars->dwp_full[s]));
                    }
                }
        } else if (lane == 2) {
            // the first layer's input: one box per K-block, rows row_first - 1 .. + 7 (OOB rows / column 14 arrive as zeros)
            uint32_t it = 0;
            for (int img = cluster_id; img < p.n_img; img += n_clusters, ++it) {
                // the activation blocks are free once the previous image's output tiles have been read out of them
                if (it > 0) mbar_wait_sleep(smem_u32(&bars->act_free), (it - 1u) & 1u, (uint32_t)p.sleep_ns);
                for (int kb = 0; kb < p.L[0].kblocks; ++kb) {
                    mbar_expect_tx(smem_u32(&bars->in_full[kb]), (uint32_t)CH_IN_BYTES);
                    tma_load_4d(smem_base + CH_OFF_ACT + kb * CH_BLK, &maps.in, smem_u32(&bars->in_full[kb]), kb * 64, 0, row_first - 1, img);
                }
            }
        }
    } else {
        // =========================== workers: depthwise, then epilogue, per layer ===========================
        const int grp = warp >> 3, wi = warp & 7;
        // Depthwise mapping: a CTA owns at most 7 rows x 14 columns, so warp wi < 7 computes the two columns 2 wi, 2 wi + 1 of
        // all seven rows (14 outputs from a 9 x 4 input patch; every computed pixel can be a real one) and the eighth warp of the
        // group only takes part in the hand-shakes.  (A 4x4-blocks-of-an-8x16-tile mapping would spend 23 % of its FMAs on
        // slots that are never pixels.)
        const bool dw_active = wi < 7;
        const int tx0 = 2 * (dw_active ? wi : 0);
        const int s0 = tx0 - 1;                                             // slot of the patch's top-left pixel (-1: the spare zero slot)
        // lane = channel pair; 16-byte chunk (lane >> 2) lives at chunk position (lane >> 2) ^ (slot & 7): one byte offset per
        // residue of the slot index modulo 8, rotated so that a compile-time slot offset k selects rd_off[k & 7]
        uint32_t rd_off[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) rd_off[j] = ((((uint32_t)lane >> 2) ^ ((uint32_t)(s0 + j) & 7u)) << 4) + (((uint32_t)lane & 3u) << 2);
        uint32_t wr_off[2];                                                 // operand row m = ty * 16 + tx: m & 7 == (tx0 + ox) & 7
#pragma unroll
        for (int ox = 0; ox < 2; ++ox) wr_off[ox] = ((((uint32_t)lane >> 2) ^ ((uint32_t)(tx0 + ox) & 7u)) << 4) + (((uint32_t)lane & 3u) << 2);
        // zero list: thread t < n_zero * 8 re-zeroes 16-byte chunk (t & 7) of slot zero_slots[t >> 3] in every K-block
        const int nzc = p.n_zero[rank] * 8;
        const uint32_t z_off = (int)threadIdx.x < nzc ? (uint32_t)p.zero_slots[rank][threadIdx.x >> 3] * 128u + ((uint32_t)threadIdx.x & 7u) * 16u : 0u;
        // pointwise role: warpgroup (rh, ch) = operand rows [64 rh, +64) x pass columns [64 ch, +64); a thread holds rows
        // m and m + 8 (m = 64 rh + 16 (warp % 4) + lane / 4) and the channel pair cp of every 8-column group
        const int rh = (warp >> 2) & 1, ch = warp >> 3, cp = (lane & 3) * 2;
        const bool wg_leader = (warp & 3) == 0 && lane == 0;
        int e_slot[2], e_halo_slot[2], e_last_slot[2];
        bool e_valid[2], e_halo[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int m = rh * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h, e_ty = m >> 4, e_tx = m & 15;
            e_valid[h] = e_ty < rows_local && e_tx < p.w;
            e_slot[h] = (e_ty + 1) * CH_PITCH + e_tx;                       // where this pixel lives in the next layer's input blocks
            e_last_slot[h] = e_ty * CH_PITCH + e_tx;                        // the last layer's staging slot
            // boundary rows also go to the peer: CTA 0's last row is CTA 1's top halo (its buffer row 0), CTA 1's first row is
            // CTA 0's bottom halo (buffer row rows0 + 1)
            e_halo[h] = e_valid[h] && (rank == 0 ? e_ty == rows_local - 1 : e_ty == 0);
            e_halo_slot[h] = (rank == 0 ? 0 : (p.rows0 + 1) * CH_PITCH) + e_tx;
        }
        const uint32_t peer_act = mapa_u32(smem_base + CH_OFF_ACT, rank ^ 1u);
        const uint32_t peer_halo_full = mapa_u32(smem_u32(&bars->halo_full), rank ^ 1u);
        const uint32_t peer_mma_done = mapa_u32(smem_u32(&bars->mma_done), rank ^ 1u);
        uint32_t dseq_base = 0, lseq = 0, halo_seq = 0, it = 0, bseq = 0, a_par = 0;
        for (int img = cluster_id; img < p.n_img; img += n_clusters, ++it) {
            for (int l = 0; l < p.n_layers; ++l, ++lseq) {
                const ChainLayer& L = p.L[l];
                const bool last = l == p.n_layers - 1;
                const bool tr0 = it == 0 && warp == 0 && lane == 0, tr8 = it == 0 && warp == 8 && lane == 0;
                if (tr0) CH_TRACE(0, l);
                // ---------------- depthwise: K-blocks grp, grp + 2, ... ----------------
                for (int kb = grp; kb < L.kblocks; kb += 2) {
                    uint8_t* blk = smem + CH_OFF_ACT + kb * CH_BLK;
                    if (l == 0) mbar_wait_sleep(smem_u32(&bars->in_full[kb]), it & 1u, (uint32_t)p.sleep_ns);
                    const uint32_t dseq = dseq_base + (uint32_t)kb, ds = dseq & (CH_SD - 1), dph = (dseq / CH_SD) & 1u;
                    mbar_wait(smem_u32(&bars->dwp_full[ds]), dph);
                    const uint8_t* prm = smem + CH_OFF_DWP + ds * CH_DWP;
                    const f32x2 sc = *reinterpret_cast<const f32x2*>(prm + 9 * 128 + lane * 8);
                    const f32x2 bi = *reinterpret_cast<const f32x2*>(prm + 9 * 128 + 256 + lane * 8);
                    const uint8_t* in0 = blk + s0 * 128;
                    uint32_t o[7][2];
                    if (dw_active) {
                        f32x2 acc[7][2];
#pragma unroll
                        for (int a = 0; a < 7; ++a) acc[a][0] = acc[a][1] = 0ull;
                        f32x2 wq[3][3];
#pragma unroll
                        for (int iy = 0; iy < 9; ++iy) {
                            if (iy < 3) {
#pragma unroll
                                for (int kx = 0; kx < 3; ++kx) wq[iy][kx] = MF::widen(*reinterpret_cast<const uint32_t*>(prm + (iy * 3 + kx) * 128 + lane * 4));
                            }
                            f32x2 row[4];
#pragma unroll
                            for (int ix = 0; ix < 4; ++ix) {
                                const int k = iy * CH_PITCH + ix;
                                row[ix] = MF::widen(*reinterpret_cast<const uint32_t*>(in0 + k * 128 + rd_off[k & 7]));
                            }
#pragma unroll
                            for (int oy = 0; oy < 7; ++oy) {
                                const int ky = iy - oy;
                                if (ky < 0 || ky >= 3) continue;
#pragma unroll
                                for (int ox = 0; ox < 2; ++ox)
#pragma unroll
                                    for (int kx = 0; kx < 3; ++kx) ffma2(acc[oy][ox], row[ox + kx], wq[ky][kx]);
                            }
                        }
#pragma unroll
                        for (int oy = 0; oy < 7; ++oy)
#pragma unroll
                            for (int ox = 0; ox < 2; ++ox) o[oy][ox] = MF::template pack_act<RELU6>(ffma2_abc(acc[oy][ox], sc, bi));
                    }
                    __syncwarp();
                    if (tr0 && kb == 0) CH_TRACE(1, l);
                    if (lane == 0) mbar_arrive(smem_u32(&bars->dwp_empty[ds]));
                    // all eight warps of this K-block have read their pixels: the block may now be overwritten by the operand tile
                    asm volatile("bar.sync %0, %1;" ::"r"(1 + grp), "r"(256) : "memory");
                    if (dw_active) {
#pragma unroll
                        for (int oy = 0; oy < 7; ++oy)
#pragma unroll
                            for (int ox = 0; ox < 2; ++ox)
                                *reinterpret_cast<uint32_t*>(blk + (oy * 16 + tx0 + ox) * 128 + wr_off[ox]) = o[oy][ox];
                    }
                    fence_proxy_async();                       // generic-proxy writes -> visible to the tensor cores (async proxy)
                    __syncwarp();
                    if (lane == 0) mbar_arrive(smem_u32(&bars->a_full[kb]));
                }
                dseq_base += (uint32_t)L.kblocks;
                if (tr0) CH_TRACE(2, l);
                if (tr8) CH_TRACE(9, l);

                // ---------------- pointwise: passes of 128 output channels over every K-block ----------------
                const uint32_t as = lseq & 1u;
                mbar_wait(smem_u32(&bars->aff_full[as]), (lseq >> 1) & 1u);
                const float2* aff = reinterpret_cast<const float2*>(smem + CH_OFF_AFF + as * CH_AFF_BYTES);
                uint32_t pk[CH_MAX_PASS][16];                              // [pass][8 h + i]: 16-bit results, channel pair of group i
#pragma unroll
                for (int ps = 0; ps < CH_MAX_PASS; ++ps) {
                    if (ps >= L.np) break;
                    const int col0 = ps * 128 + ch * 64;                  // first output channel of this warpgroup's block
                    const bool act = col0 < L.n_pad;
                    float acc[32];
#pragma unroll
                    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
                    for (int kb = 0; kb < L.kblocks; ++kb, ++bseq) {
                        const uint32_t s = bseq & (CH_SB - 1), ph = (bseq / CH_SB) & 1u;
                        mbar_wait(smem_u32(&bars->a_full[kb]), (a_par >> kb) & 1u);   // (a no-op after the first pass)
                        mbar_wait(smem_u32(&bars->b_full[s]), ph);
                        if (tr0 && kb == 0 && ps == 0) CH_TRACE(7, l);
                        if (act) {
                            const uint32_t a_lo = sw128_desc_lo(smem_base + CH_OFF_ACT + (uint32_t)kb * CH_BLK + (uint32_t)rh * 8192u);
                            const uint32_t b_lo = sw128_desc_lo(smem_base + CH_OFF_B + s * CH_B_STAGE + (uint32_t)ch * 8192u);
                            wgmma_fence();
#pragma unroll
                            for (int k4 = 0; k4 < 4; ++k4)                // +32 B (16 elements) per K step
                                wgmma_n64<T>(acc, sw128_desc(a_lo + 2u * k4), sw128_desc(b_lo + 2u * k4), (kb > 0 || k4 > 0) ? 1u : 0u);
                            wgmma_commit();
                            wgmma_wait0();
                        }
                        if (wg_leader) mbar_arrive(smem_u32(&bars->b_empty[s]));
                    }
#pragma unroll
                    for (int i = 0; i < 8; ++i) {
                        const int c = col0 + i * 8 + cp;
                        const bool ok = act && col0 + i * 8 < L.n_pad;
                        const float4 af = ok ? *reinterpret_cast<const float4*>(aff + c) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                        for (int h = 0; h < 2; ++h)
                            pk[ps][8 * h + i] = MF::template pack_act<RELU6>(ffma2_abc(f32x2_make(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]),
                                                                                        f32x2_make(af.x, af.y), f32x2_make(af.z, af.w)));
                    }
                }
                for (int kb = 0; kb < L.kblocks; ++kb) a_par ^= 1u << kb;
                if (tr0) CH_TRACE(8, l);
                // every warpgroup has finished reading the operand tiles: the activation blocks may be overwritten
                asm volatile("bar.sync %0, %1;" ::"r"(3), "r"(CH_WORKERS * 32) : "memory");
                if (!last) {                      // ... and so has the peer, before this CTA writes into the peer's halo rows
                    if (threadIdx.x == 0) mbar_arrive_cluster(peer_mma_done);
                    mbar_wait_cluster(smem_u32(&bars->mma_done), halo_seq & 1u, 0u);
                }
                if (tr0) CH_TRACE(3, l);
                // the last layer's tile is staged in the (now dead) activation blocks from slot 0 on -- a 1 KB-aligned TMA source --
                // and leaves through tensor stores; every other layer writes the next layer's input rows 1.. and the peer's halo
#pragma unroll
                for (int ps = 0; ps < CH_MAX_PASS; ++ps) {
                    if (ps >= L.np) break;
                    const int col0 = ps * 128 + ch * 64;
                    if (col0 >= L.n_pad) continue;
                    const uint32_t boff = (uint32_t)(col0 >> 6) * CH_BLK;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int w_slot = last ? e_last_slot[h] : e_slot[h];
#pragma unroll
                        for (int i = 0; i < 8; ++i) {
                            if (col0 + i * 8 >= L.n_pad) break;
                            if (e_valid[h])
                                *reinterpret_cast<uint32_t*>(smem + CH_OFF_ACT + boff + w_slot * 128 + (((uint32_t)i ^ ((uint32_t)w_slot & 7u)) << 4) + cp * 2) =
                                    pk[ps][8 * h + i];
                            if (e_halo[h] && !last)
                                st_cluster_u32(peer_act + boff + (uint32_t)e_halo_slot[h] * 128u + (((uint32_t)i ^ ((uint32_t)e_halo_slot[h] & 7u)) << 4) + cp * 2,
                                               pk[ps][8 * h + i]);
                        }
                    }
                }
                if (tr0) CH_TRACE(4, l);
                if (!last) {
                    // padding slots the in-place operand tiles have overwritten: zero again for the next layer's depthwise
                    if ((int)threadIdx.x < nzc) {
                        const int kbn = p.L[l + 1].kblocks;
                        for (int kb = 0; kb < kbn; ++kb)
                            *reinterpret_cast<uint4*>(smem + CH_OFF_ACT + kb * CH_BLK + z_off) = make_uint4(0u, 0u, 0u, 0u);
                    }
                }
                fence_proxy_async();        // these generic-proxy writes precede async-proxy accesses (MMA reads, the next image's TMA)
                __syncwarp();
                if (lane == 0) mbar_arrive(smem_u32(&bars->aff_empty[as]));
                // every local worker has left the epilogue (activations written, halo row stored into the peer) ...
                asm volatile("bar.sync %0, %1;" ::"r"(3), "r"(CH_WORKERS * 32) : "memory");
                // ... so ONE cluster-scope release (MEMBAR.GPU class, ~500 cycles) publishes all sixteen warps' halo stores: the
                // barrier orders them before this thread, and a release is cumulative
                if (!last && threadIdx.x == 0) mbar_arrive_cluster(peer_halo_full);
                if (tr0) CH_TRACE(5, l);
                // ... and the peer has delivered my halo row
                if (!last) { mbar_wait_cluster(smem_u32(&bars->halo_full), halo_seq & 1u, 0u); ++halo_seq; }
                if (last && threadIdx.x == 0) {
                    // every worker's staging writes are complete (barrier above) and fenced towards the async proxy
                    for (int kb = 0; kb < (L.c_out + 63) / 64; ++kb)
                        tma_store_4d(&maps.out[rank], smem_base + CH_OFF_ACT + kb * CH_BLK, kb * 64, 0, row_first, img);
                    bulk_commit_group();
                    bulk_wait_read0();                                    // the blocks may be refilled with the next image
                    mbar_arrive(smem_u32(&bars->act_free));
                }
                if (tr0) CH_TRACE(6, l);
            }
        }
        if (threadIdx.x == 0) bulk_wait_all();     // the output tiles have landed in global memory
    }

    __syncwarp();
    cluster_sync_all();                            // nobody exits while the peer may still touch this CTA
}

// ----------------------------------------------------------------------------------------------------------
// host side
// ----------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void chain_pack_dwp_kernel(const float* __restrict__ w, const float* __restrict__ scale, const float* __restrict__ bias,
                                      uint8_t* __restrict__ dst, int c_in, int kblocks) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= kblocks * 64) return;
    const int kb = i / 64, cl = i % 64, c = kb * 64 + cl;
    uint8_t* blk = dst + (size_t)kb * CH_DWP;
    T* wt = reinterpret_cast<T*>(blk);
    for (int t = 0; t < 9; ++t) wt[t * 64 + cl] = Traits<T>::from_f(c < c_in ? w[t * c_in + c] : 0.f);
    reinterpret_cast<float*>(blk + 9 * 128)[cl] = c < c_in ? scale[c] : 0.f;
    reinterpret_cast<float*>(blk + 9 * 128 + 256)[cl] = c < c_in ? bias[c] : 0.f;
}
__global__ void chain_pack_affine_kernel(const float* __restrict__ scale, const float* __restrict__ bias, float2* __restrict__ dst,
                                         int n_src, int n_dst) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_dst) {                                   // per channel PAIR (2j, 2j+1): (scale, scale, bias, bias)
        const int pair = i >> 1, odd = i & 1;
        float* d = reinterpret_cast<float*>(dst) + pair * 4;
        d[odd] = i < n_src ? scale[i] : 0.f;
        d[2 + odd] = i < n_src ? bias[i] : 0.f;
    }
}

struct ChainTcPlan {
    ChainMaps maps;
    ChainParams p;
    dim3 grid;
    int dtype, relu6;
    TcLaunchOpts opts;
    std::vector<void*> owned;
    size_t owned_bytes = 0;
    std::string name;
};

// a run of blocks the chain kernel can execute: 3x3 stride 1, no upsample / skip, same activation, small map, <= 512 channels
bool chain_tc_supported(int dtype, const StageGeom* g, int n_layers) {
    if (dtype != FD_F16 && dtype != FD_BF16) return false;
    if (n_layers < 2 || n_layers > CH_MAX_LAYERS) return false;
    if (get_tensor_map_encoder() == nullptr) return false;
    for (int i = 0; i < n_layers; ++i) {
        const StageGeom& s = g[i];
        if (s.ksize != 3 || s.stride != 1 || s.upsample) return false;
        if (s.c_in % 8 || s.c_out % 8 || s.c_in > 512 || s.c_out > 512) return false;
        if (s.h_out != g[0].h_out || s.w_out != g[0].w_out || s.h_in != s.h_out || s.w_in != s.w_out) return false;
        if (s.act != g[0].act) return false;
        if (i > 0 && s.c_in != g[i - 1].c_out) return false;
        if (i > 0 && s.in_pitch > 0 && s.in_pitch != s.c_in) return false;        // intermediates never exist in memory
    }
    const int h = g[0].h_out, w = g[0].w_out;
    return h >= 2 && h <= 14 && w >= 1 && w <= 14;        // two row halves of <= 7 rows; pitch-15 slots need a zero column
}

void chain_tc_destroy(ChainTcPlan* cp) {
    if (!cp) return;
    for (void* q : cp->owned) cudaFree(q);
    delete cp;
}
const char* chain_tc_name(ChainTcPlan* cp) { return cp->name.c_str(); }
size_t chain_tc_param_bytes(ChainTcPlan* cp) { return cp->owned_bytes; }

int chain_tc_prepare(int dtype, const BlockArgs* layers, int n_layers, const TcLaunchOpts& opts, ChainTcPlan** out) {
    PFN_encodeTiled encode = get_tensor_map_encoder();
    if (!encode) return fail(FD_ERR_CUDA, "cuTensorMapEncodeTiled is not available from this driver");
    ChainTcPlan* cp = new (std::nothrow) ChainTcPlan();
    if (!cp) return fail(FD_ERR_CUDA, "out of host memory");
    cp->dtype = dtype; cp->opts = opts; cp->relu6 = layers[0].g.act == FD_ACT_RELU6;
    ChainParams& p = cp->p;
    memset(&p, 0, sizeof(p));
    memset(&cp->maps, 0, sizeof(cp->maps));
    const StageGeom& g0 = layers[0].g;
    p.n_img = g0.n; p.h = g0.h_out; p.w = g0.w_out; p.rows0 = (p.h + 1) / 2; p.n_layers = n_layers;
    p.sleep_ns = opts.sleep_ns;
    const StageGeom& gl = layers[n_layers - 1].g;
    p.out = layers[n_layers - 1].out;
    p.out_pitch = gl.out_pitch > 0 ? gl.out_pitch : gl.c_out;
    for (int r = 0; r < 2; ++r) {
        const int rows_local = r == 0 ? p.rows0 : p.h - p.rows0;
        int nz = 0;
        auto add = [&](int slot) {
            for (int i = 0; i < nz; ++i) if (p.zero_slots[r][i] == slot) return;
            p.zero_slots[r][nz++] = (unsigned char)slot;
        };
        for (int rr = 0; rr <= rows_local + 1; ++rr) { add(rr * CH_PITCH + p.w); add(rr * CH_PITCH + CH_PITCH - 1); }
        const int border = r == 0 ? 0 : rows_local + 1;          // the halo row that lies outside the image
        for (int c = 0; c < p.w; ++c) add(border * CH_PITCH + c);
        p.n_zero[r] = nz;
    }
    const size_t es = 2;
    const CUtensorMapDataType dt = dtype == FD_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
    int rc = FD_OK;
    for (int l = 0; l < n_layers && rc == FD_OK; ++l) {
        const StageGeom& g = layers[l].g;
        ChainLayer& L = p.L[l];
        L.c_in = g.c_in; L.c_out = g.c_out;
        L.kblocks = (g.c_in + 63) / 64;
        // whole 64-channel blocks: the epilogue then writes every channel of the next layer's last K-block (zeros past c_out), so
        // its depthwise never reads shared memory this launch did not write (0 x a leftover Inf would be NaN).  The wgmma is n64
        // either way, so the padding costs no MMA work.
        L.n_pad = (g.c_out + 63) / 64 * 64;
        L.np = (L.n_pad + 127) / 128;
        L.aff_bytes = L.n_pad * 8;
        void* dwp = nullptr; float2* aff = nullptr;
        if (cudaMalloc(&dwp, (size_t)L.kblocks * CH_DWP) != cudaSuccess || cudaMalloc(&aff, (size_t)L.n_pad * sizeof(float2)) != cudaSuccess) {
            cudaFree(dwp); rc = fail(FD_ERR_CUDA, "cudaMalloc failed"); break;
        }
        cp->owned.push_back(dwp); cp->owned.push_back(aff);
        cp->owned_bytes += (size_t)L.kblocks * CH_DWP + (size_t)L.n_pad * sizeof(float2);
        const int tot = L.kblocks * 64;
        if (dtype == FD_F16) chain_pack_dwp_kernel<__half><<<(tot + 127) / 128, 128>>>(layers[l].dw_w, layers[l].dw_scale, layers[l].dw_bias, (uint8_t*)dwp, g.c_in, L.kblocks);
        else chain_pack_dwp_kernel<__nv_bfloat16><<<(tot + 127) / 128, 128>>>(layers[l].dw_w, layers[l].dw_scale, layers[l].dw_bias, (uint8_t*)dwp, g.c_in, L.kblocks);
        chain_pack_affine_kernel<<<(L.n_pad + 127) / 128, 128>>>(layers[l].pw_scale, layers[l].pw_bias, aff, g.c_out, L.n_pad);
        if (cudaGetLastError() != cudaSuccess) { rc = fail(FD_ERR_CUDA, "chain parameter packing launch failed"); break; }
        L.dwp = dwp; L.affine = aff;
        cuuint64_t dims[2] = {(cuuint64_t)g.c_in, (cuuint64_t)g.c_out};
        cuuint64_t strides[1] = {(cuuint64_t)g.c_in * es};
        cuuint32_t box[2] = {64, 128};
        cuuint32_t estr[2] = {1, 1};
        CUresult r = encode(&cp->maps.w[l], dt, 2, const_cast<void*>(layers[l].pw_w), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) rc = fail(FD_ERR_CUDA, "cuTensorMapEncodeTiled(chain weights) failed: " + std::to_string((int)r));
    }
    if (rc == FD_OK && cudaDeviceSynchronize() != cudaSuccess) rc = fail(FD_ERR_CUDA, "chain parameter packing failed");
    if (rc == FD_OK) {
        const int in_pitch = g0.in_pitch > 0 ? g0.in_pitch : g0.c_in;
        cuuint64_t dims[4] = {(cuuint64_t)g0.c_in, (cuuint64_t)g0.w_in, (cuuint64_t)g0.h_in, (cuuint64_t)g0.n};
        cuuint64_t strides[3] = {(cuuint64_t)in_pitch * es, (cuuint64_t)g0.w_in * in_pitch * es, (cuuint64_t)g0.h_in * g0.w_in * in_pitch * es};
        cuuint32_t box[4] = {64, (cuuint32_t)CH_PITCH, (cuuint32_t)CH_ROWS, 1};
        cuuint32_t estr[4] = {1, 1, 1, 1};
        CUresult r = encode(&cp->maps.in, dt, 4, const_cast<void*>(layers[0].in), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) rc = fail(FD_ERR_CUDA, "cuTensorMapEncodeTiled(chain input) failed: " + std::to_string((int)r));
    }
    for (int r = 0; r < 2 && rc == FD_OK; ++r) {
        const int rows_r = r == 0 ? p.rows0 : p.h - p.rows0;
        const cuuint64_t P = (cuuint64_t)p.out_pitch;
        cuuint64_t dims[4] = {(cuuint64_t)gl.c_out, (cuuint64_t)gl.w_out, (cuuint64_t)gl.h_out, (cuuint64_t)gl.n};
        cuuint64_t strides[3] = {P * es, (cuuint64_t)gl.w_out * P * es, (cuuint64_t)gl.h_out * gl.w_out * P * es};
        cuuint32_t box[4] = {64, (cuuint32_t)CH_PITCH, (cuuint32_t)rows_r, 1};
        cuuint32_t estr[4] = {1, 1, 1, 1};
        CUresult cr = encode(&cp->maps.out[r], dt, 4, p.out, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                             CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (cr != CUDA_SUCCESS) rc = fail(FD_ERR_CUDA, "cuTensorMapEncodeTiled(chain output) failed: " + std::to_string((int)cr));
    }
    if (rc != FD_OK) { chain_tc_destroy(cp); return rc; }
    const int clusters = std::min(p.n_img, std::max(1, opts.n_sms / 2));
    cp->grid = dim3((unsigned)(2 * clusters), 1, 1);
    char buf[160];
    snprintf(buf, sizeof(buf), "chain_tc<k3,s1,2cta>[%d layers,%dx%d,c%d..%d,kb%d,smem%dK]", n_layers, p.h, p.w, p.L[0].c_in, p.L[n_layers - 1].c_out,
             p.L[0].kblocks, CH_SMEM_BYTES / 1024);
    cp->name = buf;
    *out = cp;
    return FD_OK;
}

template <typename T, bool RELU6>
static int chain_launch_inst(ChainTcPlan* cp, cudaStream_t st) {
    auto kern = chain_tc_kernel<T, RELU6>;
    static PerDeviceOnce attr_set;
    int dev = -1;
    FD_CUDA_OK(cudaGetDevice(&dev));
    if (attr_set.need(dev)) {
        FD_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, CH_SMEM_BYTES));
        attr_set.done(dev);
    }
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = cp->grid; cfg.blockDim = dim3(CH_THREADS); cfg.dynamicSmemBytes = CH_SMEM_BYTES; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = cp->opts.pdl ? 1 : 0;
    FD_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, cp->maps, cp->p));
    FD_CUDA_OK(cudaGetLastError());
    return FD_OK;
}

int chain_tc_launch(ChainTcPlan* cp, cudaStream_t st);
// debug: run once with the timeline enabled; out_host[12 * 256] SM clocks of the leader CTA of cluster 0 (0 = slot unused)
int chain_tc_trace(ChainTcPlan* cp, cudaStream_t st, unsigned long long* out_host, int* rows, int* cols) {
    unsigned long long* dev = nullptr;
    const size_t bytes = 12 * 256 * sizeof(unsigned long long);
    FD_CUDA_OK(cudaMalloc(&dev, bytes));
    FD_CUDA_OK(cudaMemsetAsync(dev, 0, bytes, st));
    cp->p.trace = dev;
    int rc = chain_tc_launch(cp, st);
    cp->p.trace = nullptr;
    if (rc == FD_OK && cudaStreamSynchronize(st) != cudaSuccess) rc = fail(FD_ERR_CUDA, "chain trace run failed");
    if (rc == FD_OK) cudaMemcpy(out_host, dev, bytes, cudaMemcpyDeviceToHost);
    cudaFree(dev);
    *rows = 12; *cols = 256;
    return rc;
}

int chain_tc_launch(ChainTcPlan* cp, cudaStream_t st) {
    if (cp->dtype == FD_F16) return cp->relu6 ? chain_launch_inst<__half, true>(cp, st) : chain_launch_inst<__half, false>(cp, st);
    return cp->relu6 ? chain_launch_inst<__nv_bfloat16, true>(cp, st) : chain_launch_inst<__nv_bfloat16, false>(cp, st);
}

}  // namespace fd
