// Fused depthwise -> pointwise block kernel for sm_90a (wgmma + TMA + mbarrier rings), persistent and
// warp-specialised.
//
// One kernel per conv_dw / decode_conv block (reference imagenet/mobilenet.py:29-38, models.py:61-75,
// 683-697) including, for decoder blocks, the nearest-x2 upsample and the skip add of models.py:723-729
// in the epilogue, and optionally decode_conv6 (models.py:698,731) folded below the last upsample.
//
// Work item = one tile of 128 output pixels (NI images x TH x TW) times n_cta (<= 128) output channels.  The grid is
// one CTA per SM; every CTA walks items blockIdx.x, +gridDim.x, ... and the roles run concurrently on different
// items / K-blocks:
//   warp 16     TMA producer : per 64-channel K-block, one 4-D box load of the input halo tile
//                              [NI][IH][IW][64ch] (OOB zero fill == conv zero padding) and the [bn x 64]
//                              slices of the pointwise weights (128B-swizzled, K-major); when the whole weight
//                              matrix fits it is loaded once and stays resident
//   warps 8-15  depthwise    : lane = channel pair, 4x4 output pixels per warp, exact 16-bit products accumulated in fp32 ->
//                              BN affine -> act folded into the 16-bit conversion -> written straight into the
//                              128B-swizzled K-major A operand tile in shared memory (never touches HBM)
//   warps 0-7   consumers    : two warpgroups, each owning 64 of the tile's 128 pixel rows: wgmma m64n64k16 (fp32
//                              accumulators in registers) over the K-blocks, then BN affine + act -> 16-bit -> staging
//                              tile -> TMA tensor stores (x4 strided views for the nearest-x2 upsample, reduce-add into
//                              the skip tensor; or the folded 1-channel head)
// mbarrier rings: input stages (TMA -> dw), A stages (dw -> wgmma), B stages (TMA -> wgmma).
#include <cuda.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <string>

#include "fd_block_plan.h"
#include "fd_tc_common.cuh"

namespace fd {

constexpr int TC_DW_WARPS = 8;
constexpr int TC_EPI_WARPS = 8;                              // two consumer warpgroups (wgmma + epilogue)
// consumers on warps 0..7 (warpgroups 0 and 1), depthwise on 8..15; TcParams::epi_high swaps the two groups (both stay
// warpgroup-aligned, as wgmma requires)
constexpr int TC_WARP_EPI0 = 0, TC_WARP_DW0 = TC_EPI_WARPS;
constexpr int TC_WARP_TMA = TC_DW_WARPS + TC_EPI_WARPS;      // 16
constexpr int TC_THREADS = (TC_WARP_TMA + 1) * 32;           // 544
constexpr int TC_WARP_BCAST = TC_WARP_TMA + 1;               // 17: cluster mode only -- hands finished operand tiles to the peer CTAs
constexpr int TC_THREADS_CL = (TC_WARP_BCAST + 1) * 32;      // 576
constexpr int TC_NCH = 2;                                    // 64-column accumulator blocks per item (n_cta <= 128)
constexpr int TC_KBLK = 64;                     // channels per K-block (one 128-byte swizzle row)
constexpr int TC_A_STAGE_BYTES = 128 * 128;     // 128 rows x 64 x 2 B
constexpr int TC_MAX_IN = 6, TC_MAX_A = 6, TC_MAX_B = 16;
static_assert(TC_MAX_A >= kPlanMaxACluster && TC_MAX_A >= kPlanMaxA && TC_MAX_IN >= kPlanMaxIn && TC_MAX_B >= kPlanMaxB, "barrier arrays cover the planner's ring depths");
constexpr int TC_TRACE_N = 256;

struct TcParams {
    int n, h_in, w_in, h_out, w_out, c_in, c_out;
    int tiles_x, tiles_y;
    int items, splits;    // work items = spatial tiles x output-channel splits
    int kblocks;          // ceil(c_in / 64)
    int cin_pad;          // kblocks * 64
    int n_cta;            // output channels per item (multiple of 16)
    int bn;               // B sub-block width: 64 or 128 rows of the weight matrix per stage (rows past c_out load as zeros)
    int nb;               // sub-blocks per K-block = ceil(n_cta / bn)
    int s_in, s_a, s_b;   // pipeline depths
    int b_resident;       // 1: all kblocks*nb weight blocks are loaded once and kept (s_b == kblocks*nb)
    int in_stage_bytes, b_stage_bytes;
    int act, upsample;
    int head;             // 1: fold the C->1 head (writes head_out instead of out)
    int head_act;
    float head_scale, head_bias;
    const void* skip;
    void* out;
    void* head_out;
    int in_stage_stride;  // in_stage_bytes + dw parameter block, rounded to 128
    int dwp_bytes;        // bytes of one K-block's depthwise parameter block
    int cpad_all;         // n_cta * splits: padded length of the pointwise BN vectors
    int n_stg;            // epilogue staging tiles (16 KB each): with two, one tile's TMA store overlaps filling the other
    int out_pitch, skip_pitch;   // elements between pixels of the output / skip tensors (>= c_out: channel slice of a concat buffer)
    int sleep_ns;         // > 0: latency-tolerant waits (TMA producer: stage free) back off with nanosleep between probes
                          //      instead of re-issuing try_wait (those probes take issue slots from the depthwise warps)
    int mma_sleep_ns;     // same for the consumers' waits for an operand stage
    int dw_sleep_ns;      // same for the depthwise warps' wait for an input stage
    int epi_tma;          // 1: staging tiles leave through TMA tensor stores (4 strided views for nearest-x2 upsampling)
    int epi_red;          // 1: ... as element-wise ADD into the skip tensor, which then IS the block's output (in place)
    unsigned long long mg_splits, mg_tx, mg_ty;   // 2^40 / d reciprocals for the item -> tile decode
    const void* dwp;      // [kblocks] x { taps (see dw_taps_bytes), [64] fp32 scale, [64] fp32 bias }
    const float2* pw_affine;  // [cpad_all / 2] x (scale, scale, bias, bias) of a channel pair
    const float* head_w;  // [cpad_all]
    int dw_teams;         // 2: the depthwise warps form two teams of four that take alternate K-block steps, two 4x4 blocks per warp
                          // (needs even s_in and s_a); 1: eight warps in lock-step, one block each
    int epi_high;         // 1: the consumers run on warps 8..15 and the depthwise on 0..7 (default: the other way round)
    int wmc;              // weight-multicast cluster size (1, 2, 4): the wmc CTAs of a cluster take wmc consecutive tiles with the SAME
                          // output-channel split and each loads 1/wmc of every weight block, TMA-multicast into all of them
    int cs;               // cluster size (1, 2, 4): the cs CTAs of a cluster work on the SAME tile (splits == cs); CTA r computes the
                          // depthwise half of the K-blocks kb % cs == r only and broadcasts each finished operand tile into the A
                          // ring of every CTA of the cluster (bulk copies over DSMEM), then runs the MMAs of output-channel split r
    unsigned long long* trace;   // debug timeline (fd_plan_trace_stage) or nullptr: [12 rows][TC_TRACE_N] SM clocks of CTA 0
};

// shared-memory bookkeeping block (after the operand stages)
struct TcBarriers {
    uint64_t in_full[TC_MAX_IN], in_empty[TC_MAX_IN];
    uint64_t a_full[TC_MAX_A], a_empty[TC_MAX_A];
    uint64_t b_full[TC_MAX_B], b_empty[TC_MAX_B];
    uint64_t aff_full;    // the pointwise BN affine has landed in shared memory (one bulk copy issued in the prologue)
    uint64_t dw_done[4];  // cluster mode: the depthwise warps have finished (and proxy-fenced) an operand tile -> broadcast thread
};

struct ItemCoord { int img0, oy0, ox0, n0; };
__device__ __forceinline__ ItemCoord decode_item(const TcParams& p, int w, int NI, int TH, int TW) {
    ItemCoord c;
    uint32_t t = fdiv40((uint32_t)w, p.mg_splits);
    const int split = w - (int)t * p.splits;
    uint32_t t2 = fdiv40(t, p.mg_tx);
    const int tile_x = (int)(t - t2 * (uint32_t)p.tiles_x);
    uint32_t t3 = fdiv40(t2, p.mg_ty);
    const int tile_y = (int)(t2 - t3 * (uint32_t)p.tiles_y);
    c.img0 = (int)t3 * NI; c.oy0 = tile_y * TH; c.ox0 = tile_x * TW; c.n0 = split * p.n_cta;
    return c;
}

// ----------------------------------------------------------------------------------------------
// the kernel
// ----------------------------------------------------------------------------------------------
// debug timeline: row r, slot i <- SM clock (only CTA 0, only when p.trace != nullptr)
#define TC_TRACE(row, idx)                                                                       \
    do {                                                                                         \
        if (p.trace != nullptr && blockIdx.x == 0 && (idx) < TC_TRACE_N) p.trace[(row) * TC_TRACE_N + (idx)] = clock64(); \
    } while (0)

// HALFK: the block has at most 32 input channels (conv1): the 16 channel pairs fill half a warp, so the two half-warps split the
// warp's 4x4 pixel block into its upper and lower two rows instead of computing 32 zero channels each.
// CLM: cluster mode.  1 = the CTAs of a cluster share one TILE and split its depthwise half and its output channels (TcParams::cs);
// 2 = the CTAs of a cluster work on DIFFERENT tiles with the SAME output-channel split and share the weight stream: every CTA loads
// 1/wmc of each weight block and TMA-multicasts it to all (TcParams::wmc).
template <typename T, int KS, int STRIDE, int NI, int TH, int TW, bool RELU6, bool HALFK = false, int CLM = 0>
__global__ void __launch_bounds__(CLM == 1 ? TC_THREADS_CL : TC_THREADS, 1)
block_tc_kernel(const __grid_constant__ CUtensorMap tm_in, const __grid_constant__ CUtensorMap tm_w,
                const __grid_constant__ CUtensorMap tm_o0, const __grid_constant__ CUtensorMap tm_o1,
                const __grid_constant__ CUtensorMap tm_o2, const __grid_constant__ CUtensorMap tm_o3, const TcParams p) {
    static_assert(NI * TH * TW == 128, "tile must hold 128 pixels");
    static_assert(NI * (TH / 4) * (TW / 4) == TC_DW_WARPS, "one 4x4 pixel block per depthwise warp");
    constexpr int PAD = (KS - 1) / 2;
    constexpr int IH = (TH - 1) * STRIDE + KS, IW = (TW - 1) * STRIDE + KS;     // input box
    constexpr int IBH = 3 * STRIDE + KS, IBW = 3 * STRIDE + KS;                   // per-warp input block
    using MF = MixFma<T>;

    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* smem = smem_raw + (smem_base - smem_u32(smem_raw));
    // carve-up: [A stages][B stages][epilogue staging][input stages (+ dw parameter block each)][pw BN vectors][barriers].  A stages and
    // staging tiles are 16 KB, B stages multiples of 2 KB: everything that needs 1 KB alignment (SWIZZLE_128B atoms) sits in front of the
    // 128-byte-granular input stages, so the aligned base is the only alignment slack the plan has to budget
    const uint32_t a_off = 0;
    const uint32_t b_off = a_off + p.s_a * TC_A_STAGE_BYTES;
    const uint32_t stg_off = b_off + p.s_b * p.b_stage_bytes;                          // epilogue staging: [128 px][64 ch] 16-bit, SW128 atoms
    const uint32_t in_off = stg_off + (uint32_t)p.n_stg * 16384u;
    const uint32_t pw_off = in_off + p.s_in * p.in_stage_stride;
    const uint32_t bar_off = pw_off + (p.head ? 3u : 2u) * (uint32_t)p.cpad_all * 4u;     // (head: 16-bit weights use half of their slot)
    TcBarriers* bars = reinterpret_cast<TcBarriers*>(smem + bar_off);
    float2* s_pw_affine = reinterpret_cast<float2*>(smem + pw_off);           // (scale, scale, bias, bias) per output-channel pair
    uint32_t* s_head_w2 = reinterpret_cast<uint32_t*>(s_pw_affine + p.cpad_all);   // head weights of a channel pair, 16-bit x 2

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // role id of the sixteen worker warps: normally epilogue = warps 0..7, depthwise = 8..15; with TcParams::epi_high the two
    // groups trade places (the warp schedulers favour one end of the id range, see TcParams::epi_high)
    const int rwarp = (p.epi_high && warp < TC_DW_WARPS + TC_EPI_WARPS) ? (warp ^ 8) : warp;
    constexpr bool CL = CLM == 1, CW = CLM == 2;
    constexpr bool kHint = CLM != 1;                                   // barrier waits with a suspend-time hint (see mbar_wait_nohint)
    static_assert(!(HALFK && CLM != 0), "the half-K block has one K-block and resident weights: nothing to share");
    const uint32_t cs = CL ? (uint32_t)p.cs : 1u;                      // tile-sharing cluster: size and this CTA's rank in it
    const uint32_t crank = (CL || CW) ? cluster_ctarank() : 0u;
    // Item walk.  Normally CTA b takes items b, b + grid, ...; in weight-multicast mode the UNIT is a cluster-item = wmc
    // consecutive tiles x one output-channel split (every CTA of the cluster then streams the same weights in the same order):
    // cluster c takes units c, c + n_clusters, ... and rank r of it the unit's tile r.
    const uint32_t wmc = CW ? (uint32_t)p.wmc : 1u;
    const int u_first = CW ? (int)(blockIdx.x / wmc) : (int)blockIdx.x;
    const int u_stride = CW ? (int)(gridDim.x / wmc) : (int)gridDim.x;
    const int u_count = CW ? p.items / (int)wmc : p.items;             // tiles % wmc == 0 (checked by the host)
    auto item_of = [&](int u) -> int {
        if (!CW) return u;
        const int g = (int)fdiv40((uint32_t)u, p.mg_splits), sp = u - g * p.splits;
        return (g * (int)wmc + (int)crank) * p.splits + sp;
    };

    if (threadIdx.x == 0) {
        const uint32_t dw_arrivals = (uint32_t)(TC_DW_WARPS / ((CL || p.dw_teams != 2) ? 1 : 2));     // warps that work on one K-block step
        for (int i = 0; i < TC_MAX_IN; ++i) { mbar_init(smem_u32(&bars->in_full[i]), 1); mbar_init(smem_u32(&bars->in_empty[i]), dw_arrivals); }
        // cluster mode: an A stage is full after ONE arrival (the owner's broadcast thread, or this CTA's own expect_tx for a
        // tile that arrives by bulk copy) and free again when both consumer warpgroups of all cs CTAs are done reading it
        for (int i = 0; i < TC_MAX_A; ++i) { mbar_init(smem_u32(&bars->a_full[i]), CL ? 1u : dw_arrivals); mbar_init(smem_u32(&bars->a_empty[i]), 2u * cs); }
        for (int i = 0; i < 4; ++i) mbar_init(smem_u32(&bars->dw_done[i]), TC_DW_WARPS);
        for (int i = 0; i < TC_MAX_B; ++i) { mbar_init(smem_u32(&bars->b_full[i]), 1); mbar_init(smem_u32(&bars->b_empty[i]), 2u * wmc); }   // multicast: freed by all
        mbar_init(smem_u32(&bars->aff_full), 1);
        fence_barrier_init();
        // the pointwise BN affine (constant data, independent of the previous kernel) comes in as ONE asynchronous bulk copy that the
        // epilogue warps wait for before their first tile, instead of a strided copy loop of all threads on the start-up path
        mbar_expect_tx(smem_u32(&bars->aff_full), (uint32_t)p.cpad_all * 8u);
        bulk_load(smem_base + pw_off, p.pw_affine, (uint32_t)p.cpad_all * 8u, smem_u32(&bars->aff_full));
    }
#ifdef FD_TC_WATCHDOG_MAP
    if (blockIdx.x == 0 && threadIdx.x == 0)
        printf("WATCHDOG map (cs %d wmc %d items %d kb %d s_in %d s_a %d s_b %d): in_full %u in_empty %u a_full %u a_empty %u b_full %u b_empty %u acc_full %u acc_empty %u dw_done %u\n",
               p.cs, p.wmc, p.items, p.kblocks, p.s_in, p.s_a, p.s_b, smem_u32(&bars->in_full[0]), smem_u32(&bars->in_empty[0]), smem_u32(&bars->a_full[0]),
               smem_u32(&bars->a_empty[0]), smem_u32(&bars->b_full[0]), smem_u32(&bars->b_empty[0]), smem_u32(&bars->acc_full[0]), smem_u32(&bars->acc_empty[0]),
               smem_u32(&bars->dw_done[0]));
#endif
    if (warp == TC_WARP_TMA && lane == 0) {
        tma_prefetch_desc(&tm_in);
        tma_prefetch_desc(&tm_w);
        if (p.epi_tma) { tma_prefetch_desc(&tm_o0); if (p.upsample) { tma_prefetch_desc(&tm_o1); tma_prefetch_desc(&tm_o2); tma_prefetch_desc(&tm_o3); } }
    }
    if (p.head)                                                            // head weights of a channel pair, 16-bit x 2 (cpad_all is even)
        for (int i = 2 * threadIdx.x; i < p.cpad_all; i += 2 * (int)blockDim.x) s_head_w2[i >> 1] = MF::pack(p.head_w[i], p.head_w[i + 1]);
    if constexpr (HALFK) {
        // channels 32..63 of every A row are never written by the depthwise warps: zero the stages once (their products meet
        // the zero-filled K rows of the weights, but 0 x NaN from uninitialised shared memory would still poison the sum)
        for (int i = threadIdx.x; i < p.s_a * (TC_A_STAGE_BYTES / 16); i += (int)blockDim.x)
            reinterpret_cast<uint4*>(smem + a_off)[i] = make_uint4(0u, 0u, 0u, 0u);
        fence_proxy_async();
    }
    pdl_launch_dependents();                       // the next kernel may begin its own prologue
    pdl_wait_prior_grid();                         // everything below reads what the previous kernel wrote
    if constexpr (CLM != 0) cluster_sync_all();    // every CTA's barriers exist before a peer may signal or copy into them
    else __syncthreads();

    if (warp == TC_WARP_TMA) {
        // =========================== TMA producer ===========================
        // two independent single-thread loops in one warp: lane 0 streams input tiles (+ depthwise parameter blocks),
        // lane 1 streams pointwise-weight blocks, so a full weight ring never holds back the input prefetch
        if (lane == 0) {
            Ring rin;
            int tr = 0;
            for (int u = u_first; u < u_count; u += u_stride) {
                const int w = item_of(u);
                const ItemCoord c = decode_item(p, w, NI, TH, TW);
                for (int kb = CL ? (int)crank : 0; kb < p.kblocks; kb += (int)cs, rin.next((uint32_t)p.s_in)) {     // cluster mode: my K-blocks only
                    const uint32_t s = rin.s, ph = rin.ph;
                    mbar_wait_sleep_sel<kHint>(smem_u32(&bars->in_empty[s]), ph ^ 1u, (uint32_t)p.sleep_ns >> 2);
                    mbar_expect_tx(smem_u32(&bars->in_full[s]), (uint32_t)(p.in_stage_bytes + p.dwp_bytes));
                    tma_load_4d(smem_base + in_off + s * p.in_stage_stride, &tm_in, smem_u32(&bars->in_full[s]), kb * TC_KBLK,
                                c.ox0 * STRIDE - PAD, c.oy0 * STRIDE - PAD, c.img0);
                    bulk_load(smem_base + in_off + s * p.in_stage_stride + p.in_stage_bytes,
                              reinterpret_cast<const uint8_t*>(p.dwp) + (size_t)kb * p.dwp_bytes, (uint32_t)p.dwp_bytes,
                              smem_u32(&bars->in_full[s]));
                    TC_TRACE(0, tr); ++tr;
                }
            }
        } else if (lane == 1) {
            Ring rb;
            bool first = true;
            const uint16_t w_mask = (uint16_t)((1u << wmc) - 1u);
            const uint32_t slice_rows = (uint32_t)p.bn / wmc, slice_bytes = slice_rows * 128u;   // this CTA's share of a weight block
            for (int u = u_first; u < u_count; u += u_stride, first = false) {
                if (p.b_resident && !first) break;
                const int w = item_of(u);
                const int n0 = (w - (int)fdiv40((uint32_t)w, p.mg_splits) * p.splits) * p.n_cta;
                for (int kb = 0; kb < p.kblocks; ++kb)
                    for (int nbi = 0; nbi < p.nb; ++nbi) {
                        uint32_t sb;
                        if (p.b_resident) {
                            sb = (uint32_t)(kb * p.nb + nbi);
                        } else {
                            sb = rb.s;
                            mbar_wait_sleep_sel<kHint>(smem_u32(&bars->b_empty[sb]), rb.ph ^ 1u, (uint32_t)p.sleep_ns >> 2);
                            rb.next((uint32_t)p.s_b);
                        }
                        mbar_expect_tx(smem_u32(&bars->b_full[sb]), (uint32_t)p.b_stage_bytes);
                        if constexpr (CW)      // rows [crank * bn / wmc, ...) of the block, delivered to the same stage of every CTA
                            tma_load_2d_multicast(smem_base + b_off + sb * p.b_stage_bytes + crank * slice_bytes, &tm_w,
                                                  smem_u32(&bars->b_full[sb]), kb * TC_KBLK, n0 + nbi * p.bn + (int)(crank * slice_rows), w_mask);
                        else
                            tma_load_2d(smem_base + b_off + sb * p.b_stage_bytes, &tm_w, smem_u32(&bars->b_full[sb]), kb * TC_KBLK,
                                        n0 + nbi * p.bn);
                    }
            }
        }
    } else if (CL && warp == TC_WARP_BCAST) {
        // =========================== cluster mode: broadcast thread ===========================
        // An operand tile the local depthwise warps have finished goes to the same A stage of every other CTA of the cluster as
        // one 16 KB bulk copy each (async proxy at both ends, completion bytes on the receiver's a_full).  A warp of its own: a
        // lane of the TMA warp parked in a barrier wait does not reliably let its sibling lanes run.
        if (lane == 0) {
            Ring ra;
            uint32_t o = 0;
            for (int u = u_first; u < u_count; u += u_stride)
                for (int kb = 0; kb < p.kblocks; ++kb, ra.next((uint32_t)p.s_a)) {
                    if ((uint32_t)kb % cs != crank) continue;
                    mbar_wait_sel<kHint>(smem_u32(&bars->dw_done[o & 3u]), (o >> 2) & 1u);
                    ++o;
                    const uint32_t slot = smem_base + a_off + ra.s * TC_A_STAGE_BYTES, bar = smem_u32(&bars->a_full[ra.s]);
                    mbar_arrive(bar);                                            // the local MMA stream reads it in place
                    for (uint32_t peer = 0; peer < cs; ++peer)
                        if (peer != crank) bulk_copy_to_peer(mapa_u32(slot, peer), slot, (uint32_t)TC_A_STAGE_BYTES, mapa_u32(bar, peer));
                }
        }
    } else if (rwarp >= TC_WARP_DW0 && rwarp < TC_WARP_DW0 + TC_DW_WARPS) {
        // =========================== depthwise workers ===========================
        // The tile's eight 4x4-pixel blocks are computed either by eight warps in lock-step on the same K-block step (one block
        // each), or -- TcParams::dw_teams == 2 -- by two TEAMS of four warps that take alternate steps, two blocks per warp: a
        // step's hand-shakes (two barrier waits, proxy fence, two arrives: ~300-500 cycles in which a warp issues nothing) are
        // paid once per two blocks, and while one team is in them the other team's warps on the same schedulers are in their FMA
        // stream.  Ring depths are even in that mode, so a team always meets the same stages and its parity tracking stays exact.
        constexpr int BPR = TW / 4, BPI = (TH / 4) * BPR;
        const int dwi = rwarp - TC_WARP_DW0;
        const int teams = CL ? 1 : p.dw_teams;
        const int team = teams == 2 ? dwi >> 2 : 0, member = teams == 2 ? dwi & 3 : dwi, nblk = teams;
        Ring rin, ra;
        int tr = 0;
        uint32_t own = 0;                                  // steps this CTA computes (cluster mode: the K-blocks it owns), both teams
        const bool tracer = dwi == 0 && lane == 0;
        for (int u = u_first; u < u_count; u += u_stride) {
            for (int kb = 0; kb < p.kblocks; ++kb, ra.next((uint32_t)p.s_a)) {
                if (CL && (uint32_t)kb % cs != crank) {
                    // A peer computes this K-block; its tile arrives by bulk copy.  The stage's release is still awaited, in order:
                    // a parity wait only tells "one phase further", and this CTA's next own use of a stage may lie several uses
                    // ahead (the uses in between belong to peers) -- skipping them would let the parity alias.  Free of charge:
                    // uses are released in K-block order, so an earlier one never completes later than the one needed next.
                    mbar_wait_sel<kHint>(smem_u32(&bars->a_empty[ra.s]), ra.ph ^ 1u);
                    continue;
                }
                const uint32_t s = rin.s, ph = rin.ph, sa = ra.s, pha = ra.ph;
                rin.next((uint32_t)p.s_in);
                if (teams == 2 && (int)(own & 1u) != team) { ++own; continue; }      // the other team's step
                mbar_wait_sleep_sel<kHint>(smem_u32(&bars->in_full[s]), ph, (uint32_t)p.dw_sleep_ns);
                if (tracer) TC_TRACE(1, tr);
                const uint8_t* stage = smem + in_off + s * p.in_stage_stride;
                // this K-block's depthwise taps + folded BN for the lane's channel pair (landed with the tile)
                const uint8_t* prm = stage + p.in_stage_bytes;
                constexpr int TAPS = dw_taps_bytes(KS);
                const f32x2 sc = *reinterpret_cast<const f32x2*>(prm + TAPS + lane * 8);        // (scale, scale) of the pair
                const f32x2 bi = *reinterpret_cast<const f32x2*>(prm + TAPS + 256 + lane * 8);  // (bias, bias)
                // the A stage is normally free long before (deep ring): take it now so that every output row can be
                // published the moment its last input row has been consumed -- the stores then drain during the math and
                // the proxy fence at the end (a MEMBAR.ALL.CTA, ~36 cycles per store still in flight) finds few pending
                mbar_wait_sel<kHint>(smem_u32(&bars->a_empty[sa]), pha ^ 1u);
                uint8_t* a_s = smem + a_off + sa * TC_A_STAGE_BYTES;
#pragma unroll 1
                for (int blk = 0; blk < nblk; ++blk) {
                const int bidx = member * nblk + blk;                      // 4x4-pixel block of the tile
                const int ni = bidx / BPI, rem = bidx % BPI, br = rem / BPR, bc = rem % BPR;
                const uint8_t* in_s = stage + (uint32_t)((ni * IH + br * 4 * STRIDE) * IW + bc * 4 * STRIDE) * 128u + lane * 4u;
                if constexpr (HALFK) {
                    static_assert(KS == 3 && STRIDE == 1, "half-K depthwise exists for the 3x3 stride-1 block only");
                    const int hl = lane & 15, hh = lane >> 4;       // channel pair, row half of the 4x4 block
                    const uint8_t* in_h = in_s - lane * 4 + hl * 4 + (hh * 2 * IW) * 128;
                    const f32x2 sc2 = *reinterpret_cast<const f32x2*>(prm + TAPS + hl * 8);
                    const f32x2 bi2 = *reinterpret_cast<const f32x2*>(prm + TAPS + 256 + hl * 8);
                    f32x2 acc[2][4];
#pragma unroll
                    for (int a = 0; a < 2; ++a)
#pragma unroll
                        for (int b = 0; b < 4; ++b) acc[a][b] = 0ull;
                    f32x2 wq[KS][KS];
#pragma unroll
                    for (int iy = 0; iy < 1 + KS; ++iy) {           // 2 output rows need 2 - 1 + KS input rows
                        if (iy < KS) {
#pragma unroll
                            for (int kx = 0; kx < KS; ++kx)
                                wq[iy][kx] = MF::widen(*reinterpret_cast<const uint32_t*>(prm + (iy * KS + kx) * 128 + hl * 4));
                        }
                        f32x2 row[IBW];
#pragma unroll
                        for (int ix = 0; ix < IBW; ++ix) row[ix] = MF::widen(*reinterpret_cast<const uint32_t*>(in_h + (iy * IW + ix) * 128));
#pragma unroll
                        for (int oy = 0; oy < 2; ++oy) {
                            const int ky = iy - oy;
                            if (ky < 0 || ky >= KS) continue;
#pragma unroll
                            for (int ox = 0; ox < 4; ++ox)
#pragma unroll
                                for (int kx = 0; kx < KS; ++kx) ffma2(acc[oy][ox], row[ox + kx], wq[ky][kx]);
                            if (ky == KS - 1) {
#pragma unroll
                                for (int ox = 0; ox < 4; ++ox) {
                                    const int m = (ni * TH + br * 4 + hh * 2 + oy) * TW + bc * 4 + ox;
                                    *reinterpret_cast<uint32_t*>(a_s + m * 128 + (((hl >> 2) ^ (m & 7)) << 4) + ((hl & 3) << 2)) =
                                        MF::template pack_act<RELU6>(ffma2_abc(acc[oy][ox], sc2, bi2));
                                }
                            }
                        }
                    }
                } else {
                    // Every 16-bit input word (the lane's channel pair) is widened to an fp32 pair once per row, then one fp32 FMA
                    // per channel and pixel-tap.  A 16-bit x 16-bit product is exact in fp32, so this is the mixed-precision
                    // result.  3x3: the 9 taps are widened once per step and stay in registers.  5x5: the taps are fp32 in the
                    // parameter block and each (input row, output row) pair reads the lane's kernel row ky with three 16-byte
                    // loads; holding all 25 would not fit beside the 32 accumulators and the row.
                    f32x2 acc[4][4];
#pragma unroll
                    for (int a = 0; a < 4; ++a)
#pragma unroll
                        for (int b = 0; b < 4; ++b) acc[a][b] = 0ull;
                    constexpr bool kTapsInRegs = KS == 3;
                    f32x2 wq[kTapsInRegs ? KS : 1][KS];
#pragma unroll
                    for (int iy = 0; iy < IBH; ++iy) {
                        if constexpr (kTapsInRegs) {
                            if (iy < KS) {                                // a kernel row is widened when its first input row arrives
#pragma unroll
                                for (int kx = 0; kx < KS; ++kx)
                                    wq[iy][kx] = MF::widen(*reinterpret_cast<const uint32_t*>(prm + (iy * KS + kx) * 128 + lane * 4));
                            }
                        }
                        f32x2 row[IBW];
#pragma unroll
                        for (int ix = 0; ix < IBW; ++ix) row[ix] = MF::widen(*reinterpret_cast<const uint32_t*>(in_s + (iy * IW + ix) * 128));
#pragma unroll
                        for (int oy = 0; oy < 4; ++oy) {
                            const int ky = iy - oy * STRIDE;
                            if (ky < 0 || ky >= KS) continue;
                            f32x2 wk[KS];
                            if constexpr (kTapsInRegs) {
#pragma unroll
                                for (int kx = 0; kx < KS; ++kx) wk[kx] = wq[ky][kx];
                            } else {                                      // [5 rows][32 lanes][6 pairs], see dw_taps_bytes
                                const uint8_t* tr = prm + (ky * 32 + lane) * 48;
                                const uint4 t01 = lds_u4_here(tr), t23 = lds_u4_here(tr + 16), t4 = lds_u4_here(tr + 32);
                                wk[0] = ((f32x2)t01.y << 32) | t01.x; wk[1] = ((f32x2)t01.w << 32) | t01.z;
                                wk[2] = ((f32x2)t23.y << 32) | t23.x; wk[3] = ((f32x2)t23.w << 32) | t23.z;
                                wk[4] = ((f32x2)t4.y << 32) | t4.x;
                            }
#pragma unroll
                            for (int ox = 0; ox < 4; ++ox)
#pragma unroll
                                for (int kx = 0; kx < KS; ++kx) ffma2(acc[oy][ox], row[ox * STRIDE + kx], wk[kx]);
                            if (ky == KS - 1) {                           // output row oy is complete: BN, act, pack, publish
#pragma unroll
                                for (int ox = 0; ox < 4; ++ox) {
                                    const int m = (ni * TH + br * 4 + oy) * TW + bc * 4 + ox;
                                    *reinterpret_cast<uint32_t*>(a_s + m * 128 + (((lane >> 2) ^ (m & 7)) << 4) + ((lane & 3) << 2)) =
                                        MF::template pack_act<RELU6>(ffma2_abc(acc[oy][ox], sc, bi));
                                }
                            }
                        }
                    }
                }
                }   // blk
                if (tracer) TC_TRACE(2, tr);
                // the input stage can be refilled as soon as every warp has read it
                __syncwarp();
                if (lane == 0) mbar_arrive(smem_u32(&bars->in_empty[s]));
                fence_proxy_async();             // generic-proxy writes -> visible to the tensor core / the bulk copies (async proxy)
                __syncwarp();
                if (lane == 0) mbar_arrive(CL ? smem_u32(&bars->dw_done[own & 3u]) : smem_u32(&bars->a_full[sa]));
                ++own;
                if (tracer) { TC_TRACE(3, tr); ++tr; }
            }
        }
    } else {
        // =========================== consumer warpgroups: wgmma + epilogue ===========================
        // Warpgroup wg owns pixel rows [64 wg, 64 wg + 64) of every item; a thread holds rows r0 and r0 + 8 of each 64-column
        // accumulator block (fragment layout: see the wgmma wrappers).  Both warpgroups fill every staging tile together.
        const int ew = rwarp - TC_WARP_EPI0;               // 0..7 (rwarp = warp ^ 8 keeps the warpgroups intact)
        const int wg = ew >> 2, wq = ew & 3;
        const int r0 = wg * 64 + wq * 16 + (lane >> 2), cq = (lane & 3) * 2;
        const bool leader = wq == 0 && lane == 0;          // releases this warpgroup's operand stages
        const bool elected = ew == 0 && lane == 0;         // issues the tensor stores (and, in cluster mode, arms the A ring)
        constexpr uint32_t bar_id = 1u, bar_n = 256u;      // named barrier of the eight consumer warps
        T* __restrict__ outp = reinterpret_cast<T*>(p.out);
        const T* __restrict__ skipp = reinterpret_cast<const T*>(p.skip);
        const int n_stg = p.n_stg < 2 ? 1 : 2;
        const int nch = (p.n_cta + 63) >> 6;               // 64-column accumulator blocks of an item
        const int bn_ch = p.bn >> 6;                       // ... per weight stage (1 or 2); nb = nch / bn_ch stages per K-block
        const uint32_t a_lo0 = sw128_desc_lo(smem_base + a_off + (uint32_t)wg * 8192u), b_lo0 = sw128_desc_lo(smem_base + b_off);
        const uint32_t a_step = TC_A_STAGE_BYTES >> 4, b_step = (uint32_t)p.b_stage_bytes >> 4;
        Ring ra, rb;
        int tr = 0;
        uint32_t stg_flip = 0;
        bool first = true;
        // cluster mode: operand tiles of K-blocks another CTA owns arrive by bulk copy; the elected thread arms a stage's barrier
        // with the expected bytes for its NEXT use as soon as the current use has been observed complete (kb_arm = K-block of
        // that next use, q_left = K-block uses of this CTA's whole run that are not armed yet)
        int kb_arm = 0;
        long q_left = 0;
        if constexpr (CL) {
            if (elected) {
                const int n_it = u_first < u_count ? (u_count - 1 - u_first) / u_stride + 1 : 0;
                q_left = (long)n_it * p.kblocks;
                for (int s = 0; s < p.s_a && q_left > 0; ++s, --q_left) {
                    if ((uint32_t)kb_arm % cs != crank) mbar_expect_tx(smem_u32(&bars->a_full[s]), (uint32_t)TC_A_STAGE_BYTES);
                    if (++kb_arm == p.kblocks) kb_arm = 0;
                }
            }
        }
        mbar_wait_sel<kHint>(smem_u32(&bars->aff_full), 0);      // BN affine in place (bulk copy of the prologue)
        for (int u = u_first; u < u_count; u += u_stride, first = false) {
            const int w = item_of(u);
            const ItemCoord c = decode_item(p, w, NI, TH, TW);
            float acc[TC_NCH][32];
#pragma unroll
            for (int j = 0; j < TC_NCH; ++j)
#pragma unroll
                for (int i = 0; i < 32; ++i) acc[j][i] = 0.f;
            for (int kb = 0; kb < p.kblocks; ++kb, ra.next((uint32_t)p.s_a)) {
                mbar_wait_sleep_sel<kHint>(smem_u32(&bars->a_full[ra.s]), ra.ph, (uint32_t)p.mma_sleep_ns);
                if constexpr (CL) {
                    if (elected && q_left > 0) {
                        if ((uint32_t)kb_arm % cs != crank) mbar_expect_tx(smem_u32(&bars->a_full[ra.s]), (uint32_t)TC_A_STAGE_BYTES);
                        if (++kb_arm == p.kblocks) kb_arm = 0;
                        --q_left;
                    }
                }
                if (elected) TC_TRACE(4, tr);
                uint32_t sbs[TC_NCH] = {0u, 0u};                  // weight stage of each 64-column block
                for (int nbi = 0; nbi * bn_ch < nch; ++nbi) {
                    uint32_t sb;
                    if (p.b_resident) {
                        sb = (uint32_t)(kb * (nch / bn_ch) + nbi);
                        if (first) mbar_wait_sel<kHint>(smem_u32(&bars->b_full[sb]), 0);
                    } else {
                        sb = rb.s;
                        mbar_wait_sel<kHint>(smem_u32(&bars->b_full[sb]), rb.ph);
                        rb.next((uint32_t)p.s_b);
                    }
                    sbs[nbi] = sb;
                }
                const uint32_t a_lo = a_lo0 + ra.s * a_step;
                wgmma_fence();
#pragma unroll
                for (int j = 0; j < TC_NCH; ++j) {
                    if (j < nch) {
                        const uint32_t b_lo = b_lo0 + (bn_ch == 2 ? sbs[0] * b_step + (uint32_t)j * 512u : sbs[j] * b_step);
#pragma unroll
                        for (int k4 = 0; k4 < 4; ++k4)        // +32 B (16 elements) per K step
                            wgmma_n64<T>(acc[j], sw128_desc(a_lo + 2u * k4), sw128_desc(b_lo + 2u * k4), (kb > 0 || k4 > 0) ? 1u : 0u);
                    }
                }
                wgmma_commit();
                wgmma_wait0();
                if (leader) {                                    // this warpgroup is done reading the stages
                    const uint32_t bar_a = smem_u32(&bars->a_empty[ra.s]);
                    if constexpr (CL) { for (uint32_t r = 0; r < cs; ++r) mbar_arrive_cluster(mapa_u32(bar_a, r)); }
                    else mbar_arrive(bar_a);
                    if (!p.b_resident)
                        for (int nbi = 0; nbi * bn_ch < nch; ++nbi) {
                            const uint32_t bar_b = smem_u32(&bars->b_empty[sbs[nbi]]);
                            if constexpr (CW) { for (uint32_t r = 0; r < wmc; ++r) mbar_arrive_cluster(mapa_u32(bar_b, r)); }
                            else mbar_arrive(bar_b);
                        }
                }
                if (elected) { TC_TRACE(5, tr); ++tr; }
            }

            if (!p.head) {
                // per block of 64 output channels:
                //  A: registers -> BN affine + act -> 16-bit -> shared staging tile [128 pixels][64 ch] (16-byte chunks XOR-swizzled
                //     exactly like a SWIZZLE_128B tensor-map box)
                //  B: the tile leaves through TMA tensor stores (or coalesced 16-byte LSU stores)
                const float2* aff = s_pw_affine + c.n0;                  // this item's BN affine, 8 bytes per channel
#pragma unroll
                for (int cb = 0; cb < TC_NCH; ++cb) {
                    if (cb >= nch) break;
                    uint8_t* stg = smem + stg_off + (n_stg == 2 ? (stg_flip & 1u) * 16384u : 0u);
                    ++stg_flip;
                    if (n_stg == 1 && stg_flip > 1) {                    // single staging buffer: wait until it is free again
                        if (p.epi_tma && elected) bulk_wait_read0();
                        asm volatile("bar.sync %0, %1;" ::"r"(bar_id), "r"(bar_n) : "memory");
                    }
#pragma unroll
                    for (int i = 0; i < 8; ++i) {                        // 8-column group i: this thread's channel pair of rows r0, r0 + 8
                        if (cb * 64 + i * 8 < p.n_cta) {                 // n_cta is a multiple of 16
                            const float4 af = *reinterpret_cast<const float4*>(aff + cb * 64 + i * 8 + cq);   // (s0, s1, b0, b1)
                            const f32x2 sc = f32x2_make(af.x, af.y), bi = f32x2_make(af.z, af.w);
#pragma unroll
                            for (int h = 0; h < 2; ++h) {
                                const int r = r0 + 8 * h;
                                *reinterpret_cast<uint32_t*>(stg + r * 128 + ((i ^ (r & 7)) << 4) + cq * 2) =
                                    MF::template pack_act<RELU6>(ffma2_abc(f32x2_make(acc[cb][4 * i + 2 * h], acc[cb][4 * i + 2 * h + 1]), sc, bi));
                            }
                        }
                    }
                    if (p.epi_tma) {
                        // one elected thread, asynchronous, whole 128-byte lines, image borders and channel tails clipped by the
                        // hardware.  Before anyone may overwrite the other staging buffer its previous store must have finished
                        // READING shared memory.
                        fence_proxy_async();
                        if (elected && cb == 0) TC_TRACE(9, tr);
                        if (elected) bulk_wait_read0();
                        asm volatile("bar.sync %0, %1;" ::"r"(bar_id), "r"(bar_n) : "memory");    // staging tile complete + other buffer free
                        if (elected && cb == 0) TC_TRACE(10, tr);
                        if (elected) {
                            const uint32_t src = smem_u32(stg);
                            const int cc = c.n0 + cb * 64;
                            if (!p.upsample) {
                                tma_store_4d(&tm_o0, src, cc, c.ox0, c.oy0, c.img0);
                            } else if (!p.epi_red) {
                                tma_store_4d(&tm_o0, src, cc, c.ox0, c.oy0, c.img0);
                                tma_store_4d(&tm_o1, src, cc, c.ox0, c.oy0, c.img0);
                                tma_store_4d(&tm_o2, src, cc, c.ox0, c.oy0, c.img0);
                                tma_store_4d(&tm_o3, src, cc, c.ox0, c.oy0, c.img0);
                            } else {
                                tma_reduce_add_4d(&tm_o0, src, cc, c.ox0, c.oy0, c.img0);
                                tma_reduce_add_4d(&tm_o1, src, cc, c.ox0, c.oy0, c.img0);
                                tma_reduce_add_4d(&tm_o2, src, cc, c.ox0, c.oy0, c.img0);
                                tma_reduce_add_4d(&tm_o3, src, cc, c.ox0, c.oy0, c.img0);
                            }
                            bulk_commit_group();
                            if (cb == 0) TC_TRACE(11, tr);
                        }
                        continue;
                    }
                    asm volatile("bar.sync %0, %1;" ::"r"(bar_id), "r"(bar_n) : "memory");        // staging tile complete
                    const int et = ew * 32 + lane;                        // 0..255 over the consumer warps
                    const int ch = et & 7;                                // 16-byte chunk within the 64-channel block
                    const int ccol = cb * 64 + ch * 8;                    // accumulator column of that chunk
                    const bool cok = ccol < p.n_cta && c.n0 + ccol + 8 <= p.c_out;
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        const int rr = (et >> 3) + 32 * k;                // pixel row of the tile
                        const int r_ni = rr / (TH * TW), r_ty = (rr / TW) % TH, r_tx = rr % TW;
                        const int pimg = c.img0 + r_ni, poy = c.oy0 + r_ty, pox = c.ox0 + r_tx;
                        if (!(cok && pimg < p.n && poy < p.h_out && pox < p.w_out)) continue;
                        const uint4 v = *reinterpret_cast<const uint4*>(stg + rr * 128 + ((ch ^ (rr & 7)) << 4));
                        if (!p.upsample) {
                            *reinterpret_cast<uint4*>(outp + (((size_t)pimg * p.h_out + poy) * p.w_out + pox) * p.out_pitch + c.n0 + ccol) = v;
                        } else {
                            const int w2 = 2 * p.w_out;
                            const size_t pix00 = ((size_t)pimg * 2 * p.h_out + 2 * poy) * w2 + 2 * pox;
                            size_t off[4], soff[4];
#pragma unroll
                            for (int d = 0; d < 4; ++d) {
                                const size_t pix = pix00 + (size_t)(d >> 1) * w2 + (d & 1);
                                off[d] = pix * p.out_pitch + c.n0 + ccol;
                                soff[d] = pix * p.skip_pitch + c.n0 + ccol;
                            }
                            if (skipp != nullptr) {
                                // x = interpolate(x) (already rounded to the storage dtype); x = x + skip (models.py:723-729)
                                uint4 sv[4];
#pragma unroll
                                for (int d = 0; d < 4; ++d) sv[d] = __ldg(reinterpret_cast<const uint4*>(skipp + soff[d]));
                                const uint32_t vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                                for (int d = 0; d < 4; ++d) {
                                    const uint32_t sk[4] = {sv[d].x, sv[d].y, sv[d].z, sv[d].w};
                                    uint32_t z[4];
#pragma unroll
                                    for (int j = 0; j < 4; ++j) {
                                        const float2 a = MF::unpack(vv[j]), bq = MF::unpack(sk[j]);
                                        z[j] = MF::pack(a.x + bq.x, a.y + bq.y);
                                    }
                                    *reinterpret_cast<uint4*>(outp + off[d]) = make_uint4(z[0], z[1], z[2], z[3]);
                                }
                            } else {
#pragma unroll
                                for (int d = 0; d < 4; ++d) *reinterpret_cast<uint4*>(outp + off[d]) = v;
                            }
                        }
                    }
                }
            } else {
                // decode_conv6 folded below the last upsample: dot over the block's (<= 64) output channels, on channel PAIRS:
                // BN affine, ReLU folded into the 16-bit rounding (decode_conv5's output IS stored in 16 bits in the reference),
                // then the head's 16-bit weights times the 16-bit activations (exact products, fp32 accumulation); the four
                // threads that share a row add their partial dots
                float dot[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const int c0 = i * 8 + cq;
                    if (i * 8 < p.n_cta) {
                        const float4 af = *reinterpret_cast<const float4*>(s_pw_affine + c0);
                        const f32x2 sc = f32x2_make(af.x, af.y), bi = f32x2_make(af.z, af.w);
                        const uint32_t hw = s_head_w2[c0 >> 1];
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            const uint32_t hv = MF::template pack_act<RELU6>(ffma2_abc(f32x2_make(acc[0][4 * i + 2 * h], acc[0][4 * i + 2 * h + 1]), sc, bi));
                            MF::fma2(dot[h][0], dot[h][1], hv, hw);
                        }
                    }
                }
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    float d = dot[h][0] + dot[h][1];
                    d += __shfl_xor_sync(0xffffffffu, d, 1);
                    d += __shfl_xor_sync(0xffffffffu, d, 2);
                    const int r = r0 + 8 * h;
                    const int img = c.img0 + r / (TH * TW), oy = c.oy0 + (r / TW) % TH, ox = c.ox0 + r % TW;
                    if ((lane & 3) == 0 && img < p.n && oy < p.h_out && ox < p.w_out) {
                        const float y = apply_act(fmaf(d, p.head_scale, p.head_bias), p.head_act);
                        const uint32_t yy = MF::pack(y, y);
                        T* ho = reinterpret_cast<T*>(p.head_out) + ((size_t)img * 2 * p.h_out + 2 * oy) * (2 * p.w_out) + 2 * ox;
                        *reinterpret_cast<uint32_t*>(ho) = yy;
                        *reinterpret_cast<uint32_t*>(ho + 2 * p.w_out) = yy;
                    }
                }
            }
            if (elected) TC_TRACE(7, tr);
        }
        if (p.epi_tma && elected) bulk_wait_all();                       // all tensor stores have landed
    }

    if constexpr (CLM != 0) cluster_sync_all();    // nobody leaves while a peer may still copy into / signal this CTA
}

// ----------------------------------------------------------------------------------------------
// host side
// ----------------------------------------------------------------------------------------------
PFN_encodeTiled get_tensor_map_encoder() {
    static PFN_encodeTiled fn = nullptr;
    if (fn) return fn;
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) != cudaSuccess || !ptr) return nullptr;
    fn = reinterpret_cast<PFN_encodeTiled>(ptr);
    return fn;
}
static PFN_encodeTiled get_encode() { return get_tensor_map_encoder(); }

struct BlockTcPlan {
    CUtensorMap tm_in, tm_w, tm_o[4];
    TcParams p;
    dim3 grid;
    size_t smem_bytes;
    int dtype, ks, stride, tile;           // tile: 0 = (1,8,16), 1 = (2,8,8)
    int halfk = 0;                         // 1: c_in <= 32, the HALFK instance of the 3x3 stride-1 kernel
    int tiles = 0;                         // 128-pixel tiles of the block (items / splits)
    bool grid_final = false;               // cluster mode: the grid is sized by the occupancy query at the first launch
    TcLaunchOpts opts;                     // the plan's launch options at the time this block was prepared
    void* dwp = nullptr;                   // owned device copies (packed / padded)
    float2* pw_affine = nullptr;
    float* head_w = nullptr;
    std::string name;
};

// experiment knobs (environment, read when a plan is built): FD_TC_MAX_NCTA=<n>, FD_TC_CLUSTER=1|2|4, FD_TC_CLUSTER_MULTIWAVE=1
static void plan_env_knobs(BlockPlanIn& q) {
    const char* a = getenv("FD_TC_MAX_NCTA");
    const char* d = getenv("FD_TC_CLUSTER");          // 1 = never, 2 / 4 = force that cluster size where the block admits it
    if (d && *d) q.cluster = atoi(d);
    { const char* m = getenv("FD_TC_CLUSTER_MULTIWAVE"); q.cluster_multiwave = (m && *m == '1') ? 1 : 0; }
    q.max_n_cta = a ? atoi(a) : 0;
}

static int pick_tile(const StageGeom& g) {
    // 2 images x 8x8 when a whole image fits an 8x8 box (7x7 stages), else 1 image x 8 rows x 16 cols
    return (g.h_out <= 8 && g.w_out <= 8) ? 1 : 0;
}

bool block_tc_supported(int dtype, const StageGeom& g, bool head_fused) {
    if (dtype != FD_F16 && dtype != FD_BF16) return false;
    if (!((g.ksize == 3 && (g.stride == 1 || g.stride == 2)) || (g.ksize == 5 && g.stride == 1))) return false;
    if (g.c_in % 8 || g.c_out % 8) return false;
    if (head_fused && g.c_out > 64) return false;
    return get_encode() != nullptr;
}

template <typename T, int KS, int STRIDE, int NI, int TH, int TW, bool RELU6, bool HALFK = false, int CLM = 0>
static int launch_inst2(BlockTcPlan* bp, cudaStream_t st) {
    auto kern = block_tc_kernel<T, KS, STRIDE, NI, TH, TW, RELU6, HALFK, CLM>;
    constexpr bool CL = CLM != 0;                      // launched on clusters (either mode)
    const int csize = CLM == 1 ? bp->p.cs : bp->p.wmc; // CTAs per cluster
    const int units = CLM == 1 ? bp->tiles : bp->p.items / (bp->p.wmc > 0 ? bp->p.wmc : 1);   // what a cluster walks
    static PerDeviceOnce attr_set;             // the opt-in is per device (and per kernel instance)
    int dev = -1;
    FD_CUDA_OK(cudaGetDevice(&dev));
    if (attr_set.need(dev)) {
        FD_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        attr_set.done(dev);
    }
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = bp->grid; cfg.blockDim = dim3(CLM == 1 ? TC_THREADS_CL : TC_THREADS); cfg.dynamicSmemBytes = bp->smem_bytes; cfg.stream = st;
    cudaLaunchAttribute attr[2];
    int na = 0;
    if (CL) {
        attr[na].id = cudaLaunchAttributeClusterDimension;
        attr[na].val.clusterDim.x = (unsigned)csize; attr[na].val.clusterDim.y = 1; attr[na].val.clusterDim.z = 1;
        ++na;
    }
    if (CL && !bp->grid_final) {
        // one CTA per SM and whole clusters per GPC: ask the runtime how many clusters of this shape are resident at once and
        // let that many walk the tiles (a larger grid would still be correct -- clusters are independent -- only slower)
        cfg.attrs = attr; cfg.numAttrs = (unsigned)na;
        cfg.gridDim = dim3((unsigned)(units * csize), 1, 1);
        int n_cl = 0;
        FD_CUDA_OK(cudaOccupancyMaxActiveClusters(&n_cl, kern, &cfg));
        if (n_cl < 1) return fail(FD_ERR_UNSUPPORTED, "cluster-mode block kernel: no cluster of this shape fits the device");
        if (n_cl > units) n_cl = units;
        bp->grid = dim3((unsigned)(n_cl * csize), 1, 1);
        bp->grid_final = true;
        cfg.gridDim = bp->grid;
    }
    if (bp->opts.pdl) {
        attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[na].val.programmaticStreamSerializationAllowed = 1;
        ++na;
    }
    cfg.attrs = attr; cfg.numAttrs = (unsigned)na;
    FD_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, bp->tm_in, bp->tm_w, bp->tm_o[0], bp->tm_o[1], bp->tm_o[2], bp->tm_o[3], bp->p));
    FD_CUDA_OK(cudaGetLastError());
    return FD_OK;
}
template <typename T, int KS, int STRIDE, int NI, int TH, int TW, bool HALFK = false>
static int launch_inst(BlockTcPlan* bp, cudaStream_t st) {
    if constexpr (!HALFK) {
        if (bp->p.cs > 1)
            return bp->p.act == FD_ACT_RELU6 ? launch_inst2<T, KS, STRIDE, NI, TH, TW, true, false, 1>(bp, st)
                                             : launch_inst2<T, KS, STRIDE, NI, TH, TW, false, false, 1>(bp, st);
        if (bp->p.wmc > 1)
            return bp->p.act == FD_ACT_RELU6 ? launch_inst2<T, KS, STRIDE, NI, TH, TW, true, false, 2>(bp, st)
                                             : launch_inst2<T, KS, STRIDE, NI, TH, TW, false, false, 2>(bp, st);
    }
    return bp->p.act == FD_ACT_RELU6 ? launch_inst2<T, KS, STRIDE, NI, TH, TW, true, HALFK>(bp, st)
                                     : launch_inst2<T, KS, STRIDE, NI, TH, TW, false, HALFK>(bp, st);
}

template <typename T>
static int launch_t(BlockTcPlan* bp, cudaStream_t st) {
    const int key = bp->halfk * 1000 + bp->ks * 100 + bp->stride * 10 + bp->tile;
    switch (key) {
        case 1310: return launch_inst<T, 3, 1, 1, 8, 16, true>(bp, st);
        case 310: return launch_inst<T, 3, 1, 1, 8, 16>(bp, st);
        case 311: return launch_inst<T, 3, 1, 2, 8, 8>(bp, st);
        case 320: return launch_inst<T, 3, 2, 1, 8, 16>(bp, st);
        case 321: return launch_inst<T, 3, 2, 2, 8, 8>(bp, st);
        case 510: return launch_inst<T, 5, 1, 1, 8, 16>(bp, st);
        case 511: return launch_inst<T, 5, 1, 2, 8, 8>(bp, st);
        default: return fail(FD_ERR_UNSUPPORTED, "no fused kernel instance for this block");
    }
}

int block_tc_launch(BlockTcPlan* bp, cudaStream_t st, void* head_out) {
    if (bp->p.head) {
        if (!head_out) return fail(FD_ERR_INVALID, "head-fused block needs the output pointer");
        bp->p.head_out = head_out;
    }
    return bp->dtype == FD_F16 ? launch_t<__half>(bp, st) : launch_t<__nv_bfloat16>(bp, st);
}

size_t block_tc_param_bytes(BlockTcPlan* bp) {
    return (size_t)bp->p.kblocks * bp->p.dwp_bytes + (size_t)bp->p.cpad_all * (sizeof(float2) + sizeof(float));
}
const char* block_tc_name(BlockTcPlan* bp) { return bp->name.c_str(); }

BlockPlanOut block_tc_debug_plan(int ksize, int stride, int h_out, int w_out, int n, int c_in, int c_out, int head) {
    StageGeom g{};
    g.h_out = h_out; g.w_out = w_out;
    BlockPlanIn q{};
    q.ksize = ksize; q.stride = stride; q.tile = pick_tile(g); q.c_in = c_in; q.c_out = c_out; q.head = head;
    const int NI = q.tile ? 2 : 1, TW = q.tile ? 8 : 16;
    q.n_tiles = ((w_out + TW - 1) / TW) * ((h_out + 7) / 8) * ((n + NI - 1) / NI);
    q.barrier_bytes = (int)sizeof(TcBarriers); q.n_sms = 132;
    q.cluster = 0;
    { const char* e = getenv("FD_TC_DW_TEAMS"); q.even_rings = (e && *e == '1') ? 0 : ((e && *e == '2') ? 1 : 2); }
    if (q.even_rings == 2 && ksize == 5 && (c_in + TC_KBLK - 1) / TC_KBLK <= 2) q.even_rings = 1;
    plan_env_knobs(q);
    return plan_block(q);
}

// debug: run once with the timeline enabled; out_host[8 * TC_TRACE_N] SM clocks of CTA 0 (0 = slot unused)
int block_tc_trace(BlockTcPlan* bp, cudaStream_t st, void* head_out, unsigned long long* out_host, int* rows, int* cols) {
    unsigned long long* dev = nullptr;
    const size_t bytes = 12 * TC_TRACE_N * sizeof(unsigned long long);
    FD_CUDA_OK(cudaMalloc(&dev, bytes));
    FD_CUDA_OK(cudaMemsetAsync(dev, 0, bytes, st));
    bp->p.trace = dev;
    int rc = block_tc_launch(bp, st, head_out);
    bp->p.trace = nullptr;
    if (rc == FD_OK && cudaStreamSynchronize(st) != cudaSuccess) rc = fail(FD_ERR_CUDA, "trace run failed");
    if (rc == FD_OK) cudaMemcpy(out_host, dev, bytes, cudaMemcpyDeviceToHost);
    cudaFree(dev);
    *rows = 12; *cols = TC_TRACE_N;
    return rc;
}

void block_tc_destroy(BlockTcPlan* bp) {
    if (!bp) return;
    cudaFree(bp->dwp); cudaFree(bp->pw_affine); cudaFree(bp->head_w);
    delete bp;
}

// per-K-block depthwise parameter block: taps | [64] fp32 scale | [64] fp32 bias (zero padded).  Taps are rounded to the storage
// dtype; 3x3: kept in it as [9][64]; 5x5: widened exactly to fp32 as [5 rows][32 lanes][6 pairs] (see dw_taps_bytes).
template <typename T>
__global__ void pack_dwp_kernel(const float* __restrict__ w, const float* __restrict__ scale, const float* __restrict__ bias,
                                uint8_t* __restrict__ dst, int taps, int c_in, int kblocks, int block_bytes, float post) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= kblocks * 64) return;
    const int kb = i / 64, cl = i % 64, c = kb * 64 + cl;
    uint8_t* blk = dst + (size_t)kb * block_bytes;
    for (int t = 0; t < taps; ++t) {
        const T v = Traits<T>::from_f(c < c_in ? w[t * c_in + c] : 0.f);
        if (taps == 25) {
            float* row = reinterpret_cast<float*>(blk) + ((t / 5) * 32 + (cl >> 1)) * 12;    // kernel row t / 5 of lane cl / 2
            row[(t % 5) * 2 + (cl & 1)] = Traits<T>::to_f(v);
            if (t % 5 == 0) row[10 + (cl & 1)] = 0.f;
        } else {
            reinterpret_cast<T*>(blk)[t * 64 + cl] = v;
        }
    }
    const int tb = taps == 25 ? dw_taps_bytes(5) : dw_taps_bytes(3);
    reinterpret_cast<float*>(blk + tb)[cl] = c < c_in ? scale[c] * post : 0.f;
    reinterpret_cast<float*>(blk + tb + 256)[cl] = c < c_in ? bias[c] * post : 0.f;
}
__global__ void pack_affine_kernel(const float* __restrict__ scale, const float* __restrict__ bias, float2* __restrict__ dst,
                                   int n_src, int n_dst, float post) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    // per channel PAIR (2j, 2j+1): (scale, scale, bias, bias), so that one 16-byte load feeds the pair's affine
    if (i < n_dst) {
        const int pair = i >> 1, odd = i & 1;
        float* d = reinterpret_cast<float*>(dst) + pair * 4;
        d[odd] = i < n_src ? scale[i] * post : 0.f;
        d[2 + odd] = i < n_src ? bias[i] * post : 0.f;
    }
}
__global__ void pad_copy_kernel(const float* __restrict__ src, float* __restrict__ dst, int n_src, int n_dst) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_dst) dst[i] = i < n_src ? src[i] : 0.f;
}

static int padded_copy(const float* src, int n_src, int n_dst, float** out) {
    FD_CUDA_OK(cudaMalloc(out, (size_t)n_dst * 4));
    pad_copy_kernel<<<(n_dst + 255) / 256, 256>>>(src, *out, n_src, n_dst);
    FD_CUDA_OK(cudaGetLastError());
    return FD_OK;
}

// Default choice of the weight-multicast cluster size for a block (1 = none); FD_TC_WMC overrides.
static int block_wmc_auto(const StageGeom& g, const BlockPlanOut& po, int n_tiles) {
    (void)g; (void)po; (void)n_tiles;
    return 1;
}

// what the planner is asked for a block: its geometry, the plan's options and the environment's experiment knobs
static BlockPlanIn block_plan_in(const StageGeom& g, int tile, int halfk, int n_tiles, int head, const TcLaunchOpts& opts) {
    BlockPlanIn pin{};
    pin.ksize = g.ksize; pin.stride = g.stride; pin.tile = tile; pin.c_in = g.c_in; pin.c_out = g.c_out; pin.n_tiles = n_tiles;
    pin.head = head; pin.barrier_bytes = (int)sizeof(TcBarriers); pin.n_sms = opts.n_sms;
    pin.cluster = (opts.cluster && !halfk) ? 0 : 1;
    { const char* e = getenv("FD_TC_DW_TEAMS"); pin.even_rings = (e && *e == '1') ? 0 : ((e && *e == '2') ? 1 : 2); }   // 1 = never, 2 = wherever even rings fit
    if (pin.even_rings == 2 && g.ksize == 5 && (g.c_in + TC_KBLK - 1) / TC_KBLK <= 2) pin.even_rings = 1;   // 5x5 blocks of <= 2 K-blocks
    plan_env_knobs(pin);
    if (halfk) pin.cluster = 1;
    return pin;
}

// The plan block_tc_prepare would build for this (unfolded) block, without building it.  *pinned: an experiment knob of the
// environment asks for a particular block-kernel plan (FD_TC_MAX_NCTA, FD_TC_CLUSTER >= 2, FD_TC_WMC, FD_TC_DW_TEAMS).
BlockPlanOut block_tc_plan_for(const StageGeom& g, const TcLaunchOpts& opts, bool* pinned) {
    const int tile = pick_tile(g);
    const int NI = tile ? 2 : 1, TW = tile ? 8 : 16;
    const int n_tiles = ((g.w_out + TW - 1) / TW) * ((g.h_out + 7) / 8) * ((g.n + NI - 1) / NI);
    const char* e = getenv("FD_TC_NO_HALFK");
    const int halfk = (g.c_in <= 32 && g.ksize == 3 && g.stride == 1 && tile == 0 && !(e && *e == '1')) ? 1 : 0;
    const BlockPlanIn pin = block_plan_in(g, tile, halfk, n_tiles, 0, opts);
    auto set = [](const char* name) { const char* v = getenv(name); return v && *v; };
    *pinned = pin.max_n_cta > 0 || pin.cluster >= 2 || set("FD_TC_WMC") || set("FD_TC_DW_TEAMS");
    return plan_block(pin);
}

int block_tc_prepare(int dtype, const BlockArgs& a, const float* head_w, float head_scale, float head_bias, int head_act,
                     void* head_out, bool tma_epilogue, const TcLaunchOpts& opts, BlockTcPlan** out) {
    PFN_encodeTiled encode = get_encode();
    if (!encode) return fail(FD_ERR_CUDA, "cuTensorMapEncodeTiled is not available from this driver");
    const StageGeom& g = a.g;
    BlockTcPlan* bp = new (std::nothrow) BlockTcPlan();
    if (!bp) return fail(FD_ERR_CUDA, "out of host memory");
    bp->dtype = dtype; bp->ks = g.ksize; bp->stride = g.stride; bp->tile = pick_tile(g);
    bp->opts = opts;
    {
        const char* e = getenv("FD_TC_NO_HALFK");            // experiment knob
        bp->halfk = (g.c_in <= 32 && g.ksize == 3 && g.stride == 1 && bp->tile == 0 && !(e && *e == '1')) ? 1 : 0;
    }
    const int NI = bp->tile ? 2 : 1, TH = 8, TW = bp->tile ? 8 : 16;
    const int IH = (TH - 1) * g.stride + g.ksize, IW = (TW - 1) * g.stride + g.ksize;
    TcParams& p = bp->p;
    memset(&p, 0, sizeof(p));
    p.n = g.n; p.h_in = g.h_in; p.w_in = g.w_in; p.h_out = g.h_out; p.w_out = g.w_out; p.c_in = g.c_in; p.c_out = g.c_out;
    p.tiles_x = (g.w_out + TW - 1) / TW; p.tiles_y = (g.h_out + TH - 1) / TH;
    const int tiles_img = (g.n + NI - 1) / NI;
    const int n_tiles = p.tiles_x * p.tiles_y * tiles_img;
    p.kblocks = (g.c_in + TC_KBLK - 1) / TC_KBLK; p.cin_pad = p.kblocks * TC_KBLK;
    p.act = g.act; p.upsample = g.upsample;
    p.head = head_w != nullptr; p.head_act = head_act; p.head_scale = head_scale; p.head_bias = head_bias;
    p.skip = a.skip; p.out = a.out; p.head_out = head_out;
    p.out_pitch = g.out_pitch > 0 ? g.out_pitch : g.c_out; p.skip_pitch = g.skip_pitch > 0 ? g.skip_pitch : g.c_out;
    const int in_pitch = g.in_pitch > 0 ? g.in_pitch : g.c_in;

    const BlockPlanOut po = plan_block(block_plan_in(g, bp->tile, bp->halfk, n_tiles, p.head, opts));
    if (!po.ok) { delete bp; return fail(FD_ERR_UNSUPPORTED, "fused block does not fit shared memory"); }
    const int splits = po.splits;
    p.n_cta = po.n_cta; p.splits = po.splits; p.items = po.items;
    p.in_stage_bytes = po.in_stage_bytes; p.dwp_bytes = po.dwp_bytes; p.in_stage_stride = po.in_stage_stride; p.cpad_all = po.cpad_all;
    p.s_a = po.s_a; p.n_stg = po.n_stg; p.s_in = po.s_in; p.s_b = po.s_b; p.bn = po.bn; p.nb = po.nb;
    p.b_resident = po.b_resident; p.b_stage_bytes = po.b_stage_bytes;
    p.cs = po.cs; bp->tiles = n_tiles;
    // Weight-multicast clusters (mode 2): wmc consecutive tiles with the same output-channel split stream ONE copy of the weights
    // out of the L2 instead of every CTA fetching the same weight blocks again.
    { const char* e = getenv("FD_TC_EPI_HIGH"); p.epi_high = (e && *e) ? atoi(e) : 0; }
    // Two depthwise teams (see the kernel) need even ring depths, which can cost the plan a staging tile or a weight stage, so
    // they are automatic only for one-K-block blocks whose unconstrained plan already has even rings; FD_TC_DW_TEAMS=2 forces
    // even rings.
    p.dw_teams = po.dw_teams;
    p.wmc = 1;
    {
        const char* e = getenv("FD_TC_WMC");               // 1 = never, 2 / 4 = force where the block admits it
        int want = e && *e ? atoi(e) : 0;
        if (!opts.cluster || bp->halfk) want = 1;
        if (want == 0) want = block_wmc_auto(g, po, n_tiles);
        while (want > 1 && !(p.cs == 1 && !p.b_resident && n_tiles % want == 0 && p.bn % (8 * want) == 0 && n_tiles / want >= 1)) want >>= 1;
        p.wmc = want < 1 ? 1 : want;
    }
    bp->smem_bytes = (size_t)po.smem_bytes;
    const int taps = g.ksize * g.ksize;
    (void)splits;
    const int sms = opts.n_sms;
    p.sleep_ns = opts.sleep_ns;
    {   // experiment knobs (environment, read when a plan is built)
        const char* a = getenv("FD_TC_MMA_SLEEP"); const char* b = getenv("FD_TC_DW_SLEEP");
        p.mma_sleep_ns = a ? atoi(a) : 0;
        p.dw_sleep_ns = b ? atoi(b) : 0;
    }
    bp->grid = dim3((unsigned)(p.items < sms ? p.items : sms), 1, 1);
    if (p.cs > 1) {                                   // whole clusters; refined by the occupancy query at the first launch
        int n_cl = sms / p.cs; if (n_cl > n_tiles) n_cl = n_tiles; if (n_cl < 1) n_cl = 1;
        bp->grid = dim3((unsigned)(n_cl * p.cs), 1, 1);
    } else if (p.wmc > 1) {
        int n_cl = sms / p.wmc; if (n_cl > p.items / p.wmc) n_cl = p.items / p.wmc; if (n_cl < 1) n_cl = 1;
        bp->grid = dim3((unsigned)(n_cl * p.wmc), 1, 1);
    }

    // packed / padded parameter copies (device -> device)
    int rc = FD_OK;
    const float post = 1.0f;
    auto magic = [](int d) { return (unsigned long long)((1ULL << 40) / (unsigned long long)d) + 1ULL; };
    p.mg_splits = magic(p.splits); p.mg_tx = magic(p.tiles_x); p.mg_ty = magic(p.tiles_y);
    if (cudaMalloc(&bp->dwp, (size_t)p.kblocks * p.dwp_bytes) != cudaSuccess) rc = fail(FD_ERR_CUDA, "cudaMalloc failed");
    if (rc == FD_OK) {
        const int tot = p.kblocks * 64;
        if (dtype == FD_F16) pack_dwp_kernel<__half><<<(tot + 127) / 128, 128>>>(a.dw_w, a.dw_scale, a.dw_bias, (uint8_t*)bp->dwp, taps, g.c_in, p.kblocks, p.dwp_bytes, post);
        else pack_dwp_kernel<__nv_bfloat16><<<(tot + 127) / 128, 128>>>(a.dw_w, a.dw_scale, a.dw_bias, (uint8_t*)bp->dwp, taps, g.c_in, p.kblocks, p.dwp_bytes, post);
        if (cudaGetLastError() != cudaSuccess) rc = fail(FD_ERR_CUDA, "pack_dwp_kernel launch failed");
    }
    if (rc == FD_OK && cudaMalloc(&bp->pw_affine, (size_t)p.cpad_all * sizeof(float2)) != cudaSuccess) rc = fail(FD_ERR_CUDA, "cudaMalloc failed");
    if (rc == FD_OK) {
        pack_affine_kernel<<<(p.cpad_all + 127) / 128, 128>>>(a.pw_scale, a.pw_bias, bp->pw_affine, g.c_out, p.cpad_all, post);
        if (cudaGetLastError() != cudaSuccess) rc = fail(FD_ERR_CUDA, "pack_affine_kernel launch failed");
    }
    if (rc == FD_OK) rc = padded_copy(p.head ? head_w : a.pw_scale, p.head ? g.c_out : 0, p.cpad_all, &bp->head_w);
    if (rc == FD_OK && cudaDeviceSynchronize() != cudaSuccess) rc = fail(FD_ERR_CUDA, "parameter packing failed");
    if (rc != FD_OK) { block_tc_destroy(bp); return rc; }
    p.dwp = bp->dwp; p.pw_affine = bp->pw_affine; p.head_w = bp->head_w;

    // tensor maps
    const size_t es = 2;
    const CUtensorMapDataType dt = dtype == FD_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
    {   // input: NHWC viewed as (C, W, H, N); box (64, IW, IH, NI); no swizzle; OOB -> 0 (== zero padding)
        cuuint64_t dims[4] = {(cuuint64_t)g.c_in, (cuuint64_t)g.w_in, (cuuint64_t)g.h_in, (cuuint64_t)g.n};
        cuuint64_t strides[3] = {(cuuint64_t)in_pitch * es, (cuuint64_t)g.w_in * in_pitch * es, (cuuint64_t)g.h_in * g.w_in * in_pitch * es};
        cuuint32_t box[4] = {(cuuint32_t)TC_KBLK, (cuuint32_t)IW, (cuuint32_t)IH, (cuuint32_t)NI};
        cuuint32_t estr[4] = {1, 1, 1, 1};
        CUresult r = encode(&bp->tm_in, dt, 4, const_cast<void*>(a.in), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { block_tc_destroy(bp); return fail(FD_ERR_CUDA, "cuTensorMapEncodeTiled(input) failed: " + std::to_string((int)r)); }
    }
    {   // pointwise weights [c_out][c_in] viewed as (K = c_in, N = c_out); box (64, bn); 128B swizzle
        cuuint64_t dims[2] = {(cuuint64_t)g.c_in, (cuuint64_t)g.c_out};
        cuuint64_t strides[1] = {(cuuint64_t)g.c_in * es};
        cuuint32_t box[2] = {(cuuint32_t)TC_KBLK, (cuuint32_t)(p.bn / p.wmc)};      // multicast mode: each CTA loads its share of a block
        cuuint32_t estr[2] = {1, 1};
        CUresult r = encode(&bp->tm_w, dt, 2, const_cast<void*>(a.pw_w), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { block_tc_destroy(bp); return fail(FD_ERR_CUDA, "cuTensorMapEncodeTiled(weights) failed: " + std::to_string((int)r)); }
    }
    // output views for the TMA epilogue: plain NHWC, or the four (dy, dx) phases of the 2x nearest-upsampled tensor
    memset(bp->tm_o, 0, sizeof(bp->tm_o));
    p.epi_tma = (!p.head && tma_epilogue) ? 1 : 0;
    p.epi_red = (p.epi_tma && a.skip != nullptr) ? 1 : 0;
    if (p.epi_red && (a.skip != a.out || p.skip_pitch != p.out_pitch)) { block_tc_destroy(bp); return fail(FD_ERR_STATE, "in-place skip accumulation needs out == skip"); }
    if (p.epi_tma) {
        const int up = g.upsample ? 2 : 1;
        const cuuint64_t C = (cuuint64_t)g.c_out, P = (cuuint64_t)p.out_pitch, W2 = (cuuint64_t)g.w_out * up, H2 = (cuuint64_t)g.h_out * up;
        for (int d = 0; d < (g.upsample ? 4 : 1); ++d) {
            char* base = reinterpret_cast<char*>(a.out) + ((size_t)(d >> 1) * W2 + (d & 1)) * P * es;
            cuuint64_t dims[4] = {C, (cuuint64_t)g.w_out, (cuuint64_t)g.h_out, (cuuint64_t)g.n};
            cuuint64_t strides[3] = {up * P * es, up * W2 * P * es, H2 * W2 * P * es};
            cuuint32_t box[4] = {64, (cuuint32_t)TW, (cuuint32_t)TH, (cuuint32_t)NI};
            cuuint32_t estr[4] = {1, 1, 1, 1};
            CUresult r = encode(&bp->tm_o[d], dt, 4, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            if (r != CUDA_SUCCESS) { block_tc_destroy(bp); return fail(FD_ERR_CUDA, "cuTensorMapEncodeTiled(output) failed: " + std::to_string((int)r)); }
        }
    }
    char buf[160];
    char clbuf[16] = "";
    if (p.cs > 1) snprintf(clbuf, sizeof(clbuf), ",cl%d", p.cs);
    else if (p.wmc > 1) snprintf(clbuf, sizeof(clbuf), ",wmc%d", p.wmc);
    if (p.dw_teams == 2) strncat(clbuf, ",t2", sizeof(clbuf) - strlen(clbuf) - 1);
    snprintf(buf, sizeof(buf), "block_tc<k%d,s%d,%s%s%s>%s%s%s[n%dx%d,bn%d%s,kb%d,in%d,a%d,b%d,e%d]", g.ksize, g.stride, bp->tile ? "2x8x8" : "1x8x16", bp->halfk ? ",k32" : "", clbuf,
             g.upsample ? "+up2x" : "", a.skip ? (p.epi_red ? "+skip(red)" : "+skip") : "", p.head ? "+head" : (p.epi_tma ? "+tmast" : ""), p.n_cta, p.splits, p.bn,
             p.b_resident ? "r" : "", p.kblocks, p.s_in, p.s_a, p.s_b, p.head ? 0 : p.n_stg);
    bp->name = buf;
    *out = bp;
    return FD_OK;
}

}  // namespace fd
