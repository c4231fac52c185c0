// Stem (conv_bn(c_in, C0, stride 2) + BN + ReLU6, reference imagenet/mobilenet.py:22-27, 41 and models.py:443-453) on
// wgmma, for 1 <= c_in <= 7 input channels (RGB: 3, depth only: 1, RGB-D: 4).
//
// A dense 3x3 convolution over c_in planes is a K = 9*c_in contraction per output pixel: on SIMT that is 27*C0 FMAs per
// pixel at c_in = 3 (694 MMAC per batch of 64, more than twice the HBM time of the stage), on the tensor core it is a
// M=128 x N=C0 x K=16*ceil(9*c_in/16) product per 128-pixel tile once the im2col rows sit in shared memory.  9*c_in <= 63,
// so one pixel's im2col row is one 128-byte SW128 K-major row for every c_in.  So:
//   warp 8     TMA producer : 4-D box [1 img][c_in planes][17 rows][40 cols] of the NCHW input per 8x16 output tile
//                             (OOB zero fill == the conv's zero padding); stem weights [C0pad x 64] loaded once
//   warps 0-3  im2col       : thread = output pixel; gathers its 9*c_in taps from the staged planes and writes the
//                             128B-swizzled K-major A row, K = ci*9 + ky*3 + kx, zero past 9*c_in
//   warps 4-7  consumer     : one warpgroup: wgmma m64n32k16 (two row halves x C0 / 32 column blocks x ceil(9*c_in/16)
//                             K steps: 2 at c_in = 3) into register accumulators -> BN affine + ReLU6 -> 16-bit NHWC store
// Persistent: one CTA per SM walks tiles blockIdx.x, +gridDim.x, ...
#include <cstdio>
#include <cstring>
#include <new>
#include <string>

#include "fd_tc_common.cuh"

namespace fd {

constexpr int ST_WARP_EPI0 = 4, ST_WARP_TMA = 8, ST_THREADS = 288;
constexpr int ST_MAX_N = 64;                          // output channels the register accumulators hold
constexpr int ST_TH = 8, ST_TW = 16;
constexpr int ST_IH = 17, ST_IW = 40;                 // rows 2*7+3 = 17; cols: the 33 needed ones sit at box columns 7..39 because
                                                      // the box starts 8 elements (16 bytes) left of column 2*ox0 (aligned start)
constexpr int ST_XSHIFT = 8;
constexpr int ST_MAX_CIN = 7;                        // K = 9*c_in fits one 64-element K-major row
__host__ __device__ constexpr int st_in_bytes(int cin) { return cin * ST_IH * ST_IW * 2; }                  // 4080 at c_in = 3
__host__ __device__ constexpr int st_in_stride(int cin) { return (st_in_bytes(cin) + 1023) / 1024 * 1024; } // 4096 at c_in = 3
__host__ __device__ constexpr int st_ksteps(int cin) { return (9 * cin + 15) / 16; }                        // k16 steps: 2 at c_in = 3
constexpr int ST_A_BYTES = 128 * 128;
constexpr int ST_S_IN = 8, ST_S_A = 3;

struct StemParams {
    int n, h_in, w_in, h_out, w_out, c_out, n_pad;   // n_pad: c_out rounded up to 32 (one wgmma column block)
    int out_pitch;                                   // elements between output pixels (>= c_out)
    int tiles_x, tiles_y, items;
    unsigned long long mg_tx, mg_ty;
    void* out;
    const float2* affine;    // [n_pad / 2] x (scale, scale, bias, bias) of a channel pair
};

struct StemBarriers {
    uint64_t in_full[ST_S_IN], in_empty[ST_S_IN];
    uint64_t a_full[ST_S_A], a_empty[ST_S_A];
    uint64_t b_full;
};

template <typename T, int CIN>
__global__ void __launch_bounds__(ST_THREADS, 1)
stem_tc_kernel(const __grid_constant__ CUtensorMap tm_in, const __grid_constant__ CUtensorMap tm_w, const StemParams p) {
    using MF = MixFma<T>;
    constexpr int ST_IN_BYTES = st_in_bytes(CIN), ST_IN_STRIDE = st_in_stride(CIN), KS = st_ksteps(CIN);
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* smem = smem_raw + (smem_base - smem_u32(smem_raw));
    const uint32_t a_off = 0;
    const uint32_t b_off = a_off + ST_S_A * ST_A_BYTES;            // weights: n_pad rows x 128 B
    const uint32_t in_off = b_off + (uint32_t)p.n_pad * 128u;
    const uint32_t af_off = in_off + ST_S_IN * ST_IN_STRIDE;
    const uint32_t bar_off = af_off + (uint32_t)p.n_pad * 8u;
    StemBarriers* bars = reinterpret_cast<StemBarriers*>(smem + bar_off);
    float2* s_affine = reinterpret_cast<float2*>(smem + af_off);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        for (int i = 0; i < ST_S_IN; ++i) { mbar_init(smem_u32(&bars->in_full[i]), 1); mbar_init(smem_u32(&bars->in_empty[i]), 4); }
        for (int i = 0; i < ST_S_A; ++i) { mbar_init(smem_u32(&bars->a_full[i]), 4); mbar_init(smem_u32(&bars->a_empty[i]), 1); }
        mbar_init(smem_u32(&bars->b_full), 1);
        fence_barrier_init();
    }
    if (warp == ST_WARP_TMA && lane == 0) { tma_prefetch_desc(&tm_in); tma_prefetch_desc(&tm_w); }
    for (int i = threadIdx.x; i < p.n_pad; i += ST_THREADS) s_affine[i] = p.affine[i];
    // an A row gets the K positions its KS k16 steps read (zeros past 9*c_in); the rest of the 128-byte row is never read
    pdl_launch_dependents();                       // the next kernel may begin its own prologue
    pdl_wait_prior_grid();                         // everything below reads what the previous kernel wrote
    __syncthreads();

    auto decode = [&](int w, int& img, int& oy0, int& ox0) {
        const uint32_t t2 = fdiv40((uint32_t)w, p.mg_tx);
        ox0 = (int)((uint32_t)w - t2 * (uint32_t)p.tiles_x) * ST_TW;
        const uint32_t t3 = fdiv40(t2, p.mg_ty);
        oy0 = (int)(t2 - t3 * (uint32_t)p.tiles_y) * ST_TH;
        img = (int)t3;
    };

    if (warp == ST_WARP_TMA) {
        if (lane == 0) {
            mbar_expect_tx(smem_u32(&bars->b_full), (uint32_t)p.n_pad * 128u);
            tma_load_2d(smem_base + b_off, &tm_w, smem_u32(&bars->b_full), 0, 0);
            Ring rin;
            for (int w = blockIdx.x; w < p.items; w += gridDim.x, rin.next(ST_S_IN)) {
                int img, oy0, ox0;
                decode(w, img, oy0, ox0);
                mbar_wait(smem_u32(&bars->in_empty[rin.s]), rin.ph ^ 1u);
                mbar_expect_tx(smem_u32(&bars->in_full[rin.s]), ST_IN_BYTES);
                tma_load_4d(smem_base + in_off + rin.s * ST_IN_STRIDE, &tm_in, smem_u32(&bars->in_full[rin.s]), 2 * ox0 - ST_XSHIFT, 2 * oy0 - 1, 0, img);
            }
        }
    } else if (warp < ST_WARP_EPI0) {
        // =========================== im2col workers: thread = output pixel ===========================
        const int m = threadIdx.x;                       // 0..127
        const int ty = m / ST_TW, tx = m % ST_TW;
        Ring rin, ra;
        for (int w = blockIdx.x; w < p.items; w += gridDim.x, rin.next(ST_S_IN), ra.next(ST_S_A)) {
            mbar_wait(smem_u32(&bars->in_full[rin.s]), rin.ph);
            // tap kx of pixel tx is box column 2*tx + kx + 7: words (tx+3) [high half] and (tx+4) [both halves]
            const uint8_t* in_s = smem + in_off + rin.s * ST_IN_STRIDE + (2 * ty * ST_IW + 2 * tx + ST_XSHIFT - 2) * 2;
            // 3*c_in (plane, ky) rows of 3 taps from two aligned 32-bit words
            constexpr int NK = 9 * CIN;
            uint32_t h[NK];
#pragma unroll
            for (int r = 0; r < 3 * CIN; ++r) {
                const int ci = r / 3, ky = r % 3;
                const uint32_t* q = reinterpret_cast<const uint32_t*>(in_s + ((ci * ST_IH + ky) * ST_IW) * 2);
                const uint32_t w0 = q[0], w1 = q[1];
                h[3 * r] = w0 >> 16; h[3 * r + 1] = w1 & 0xffffu; h[3 * r + 2] = w1 >> 16;
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(smem_u32(&bars->in_empty[rin.s]));
            uint32_t wd[8 * KS];                       // the KS k16 steps' K positions, two per word
#pragma unroll
            for (int j = 0; j < 8 * KS; ++j) {
                const uint32_t lo = (2 * j < NK) ? h[(2 * j < NK) ? 2 * j : 0] : 0u;
                const uint32_t hi = (2 * j + 1 < NK) ? h[(2 * j + 1 < NK) ? 2 * j + 1 : 0] : 0u;
                wd[j] = lo | (hi << 16);
            }
            mbar_wait(smem_u32(&bars->a_empty[ra.s]), ra.ph ^ 1u);
            uint8_t* a_row = smem + a_off + ra.s * ST_A_BYTES + m * 128;
#pragma unroll
            for (int c = 0; c < 2 * KS; ++c)
                *reinterpret_cast<uint4*>(a_row + ((c ^ (m & 7)) << 4)) = make_uint4(wd[4 * c], wd[4 * c + 1], wd[4 * c + 2], wd[4 * c + 3]);
            fence_proxy_async();
            __syncwarp();
            if (lane == 0) mbar_arrive(smem_u32(&bars->a_full[ra.s]));
        }
    } else {
        // =========================== consumer warpgroup: wgmma + epilogue ===========================
        const int wq = warp - ST_WARP_EPI0, cq = (lane & 3) * 2;
        T* __restrict__ outp = reinterpret_cast<T*>(p.out);
        const int nch = p.n_pad >> 5;                    // 32-column blocks
        mbar_wait(smem_u32(&bars->b_full), 0);
        const uint32_t b_lo = sw128_desc_lo(smem_base + b_off);
        Ring ra;
        for (int w = blockIdx.x; w < p.items; w += gridDim.x, ra.next(ST_S_A)) {
            int img, oy0, ox0;
            decode(w, img, oy0, ox0);
            float acc[2][ST_MAX_N / 32][16];              // [row half][column block]
            mbar_wait(smem_u32(&bars->a_full[ra.s]), ra.ph);
            const uint32_t a_lo = sw128_desc_lo(smem_base + a_off + ra.s * ST_A_BYTES);
            wgmma_fence();
#pragma unroll
            for (int mh = 0; mh < 2; ++mh)
#pragma unroll
                for (int j = 0; j < ST_MAX_N / 32; ++j) {
                    if (j < nch) {                        // KS steps of 16 (+32 B each) from a zero accumulator; B rows of block j at +j * 4 KB
#pragma unroll
                        for (int ks = 0; ks < KS; ++ks)
                            wgmma_n32<T>(acc[mh][j], sw128_desc(a_lo + (uint32_t)mh * 512u + 2u * ks),
                                         sw128_desc(b_lo + (uint32_t)j * 256u + 2u * ks), ks > 0 ? 1u : 0u);
                    }
                }
            wgmma_commit();
            wgmma_wait0();
            if (wq == 0 && lane == 0) mbar_arrive(smem_u32(&bars->a_empty[ra.s]));
#pragma unroll
            for (int mh = 0; mh < 2; ++mh)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int m = mh * 64 + wq * 16 + (lane >> 2) + 8 * h;     // pixel of the tile
                    const int oy = oy0 + m / ST_TW, ox = ox0 + m % ST_TW;
                    if (oy >= p.h_out || ox >= p.w_out) continue;
                    T* o = outp + (((size_t)img * p.h_out + oy) * p.w_out + ox) * p.out_pitch;
#pragma unroll
                    for (int j = 0; j < ST_MAX_N / 32; ++j)
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            const int c0 = j * 32 + i * 8;            // 8-channel group; this thread's pair is c0 + cq
                            if (j < nch && c0 < p.c_out) {
                                const float4 af = *reinterpret_cast<const float4*>(s_affine + c0 + cq);     // (s0, s1, b0, b1)
                                *reinterpret_cast<uint32_t*>(o + c0 + cq) = MF::template pack_act<true>(ffma2_abc(
                                    f32x2_make(acc[mh][j][4 * i + 2 * h], acc[mh][j][4 * i + 2 * h + 1]), f32x2_make(af.x, af.y), f32x2_make(af.z, af.w)));
                            }
                        }
                }
        }
    }
}

// ----------------------------------------------------------------------------------------------
// host side
// ----------------------------------------------------------------------------------------------
struct StemTcPlan {
    CUtensorMap tm_in, tm_w;
    StemParams p;
    dim3 grid;
    size_t smem_bytes;
    int dtype, c_in;
    TcLaunchOpts opts;
    const void* x_bound = nullptr;       // input pointer the tensor map was encoded for
    void* w16 = nullptr;                 // [n_pad][64] 16-bit, K = (ci, ky, kx) padded
    float2* affine = nullptr;
    int n, h_in, w_in;
    std::string name;
};

template <typename T>
__global__ void pack_stem_w_kernel(const float* __restrict__ wk, T* __restrict__ dst, int c_in, int c_out, int n_pad) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;           // dst[co][k], src tap-major [9 c_in][c_out]
    if (i >= n_pad * 64) return;
    const int co = i / 64, k = i % 64;
    dst[i] = Traits<T>::from_f((co < c_out && k < 9 * c_in) ? wk[k * c_out + co] : 0.f);
}
__global__ void pack_stem_affine_kernel(const float* __restrict__ scale, const float* __restrict__ bias, float2* __restrict__ dst,
                                        int c_out, int n_pad) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    // per channel PAIR (2j, 2j+1): (scale, scale, bias, bias), one 16-byte load feeds the pair (same layout as the block kernel)
    if (i < n_pad) {
        float* d = reinterpret_cast<float*>(dst) + (i >> 1) * 4;
        d[i & 1] = i < c_out ? scale[i] : 0.f;
        d[2 + (i & 1)] = i < c_out ? bias[i] : 0.f;
    }
}

bool stem_tc_supported(int dtype, const StageGeom& g) {
    if (dtype != FD_F16 && dtype != FD_BF16) return false;
    if (g.ksize != 3 || g.stride != 2 || g.c_in < 1 || g.c_in > ST_MAX_CIN || g.act != FD_ACT_RELU6) return false;
    if (g.c_out % 8 || g.c_out > ST_MAX_N || (g.w_in % 8)) return false;       // W*2 bytes must be a 16-byte multiple for TMA
    return get_tensor_map_encoder() != nullptr;
}

void stem_tc_destroy(StemTcPlan* sp) {
    if (!sp) return;
    cudaFree(sp->w16); cudaFree(sp->affine);
    delete sp;
}

static int encode_input_map(StemTcPlan* sp, const void* x) {
    PFN_encodeTiled encode = get_tensor_map_encoder();
    const CUtensorMapDataType dt = sp->dtype == FD_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
    const cuuint64_t plane = (cuuint64_t)sp->w_in * sp->h_in * 2;
    cuuint64_t dims[4] = {(cuuint64_t)sp->w_in, (cuuint64_t)sp->h_in, (cuuint64_t)sp->c_in, (cuuint64_t)sp->n};
    cuuint64_t strides[3] = {(cuuint64_t)sp->w_in * 2, plane, plane * (cuuint64_t)sp->c_in};
    cuuint32_t box[4] = {ST_IW, ST_IH, (cuuint32_t)sp->c_in, 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = encode(&sp->tm_in, dt, 4, const_cast<void*>(x), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(FD_ERR_CUDA, "cuTensorMapEncodeTiled(stem input) failed: " + std::to_string((int)r));
    sp->x_bound = x;
    return FD_OK;
}

int stem_tc_prepare(int dtype, const StageGeom& g, const float* wk_dev, const float* scale_dev, const float* bias_dev, void* out,
                    const TcLaunchOpts& opts, StemTcPlan** res) {
    PFN_encodeTiled encode = get_tensor_map_encoder();
    if (!encode) return fail(FD_ERR_CUDA, "cuTensorMapEncodeTiled is not available from this driver");
    StemTcPlan* sp = new (std::nothrow) StemTcPlan();
    if (!sp) return fail(FD_ERR_CUDA, "out of host memory");
    sp->dtype = dtype; sp->c_in = g.c_in; sp->n = g.n; sp->h_in = g.h_in; sp->w_in = g.w_in;
    StemParams& p = sp->p;
    memset(&p, 0, sizeof(p));
    p.n = g.n; p.h_in = g.h_in; p.w_in = g.w_in; p.h_out = g.h_out; p.w_out = g.w_out; p.c_out = g.c_out;
    p.n_pad = (g.c_out + 31) / 32 * 32;
    p.out_pitch = g.out_pitch > 0 ? g.out_pitch : g.c_out;
    p.tiles_x = (g.w_out + ST_TW - 1) / ST_TW; p.tiles_y = (g.h_out + ST_TH - 1) / ST_TH;
    p.items = p.tiles_x * p.tiles_y * g.n;
    auto magic = [](int d) { return (unsigned long long)((1ULL << 40) / (unsigned long long)d) + 1ULL; };
    p.mg_tx = magic(p.tiles_x); p.mg_ty = magic(p.tiles_y);
    p.out = out;
    int rc = FD_OK;
    if (cudaMalloc(&sp->w16, (size_t)p.n_pad * 64 * 2) != cudaSuccess || cudaMalloc(&sp->affine, (size_t)p.n_pad * sizeof(float2)) != cudaSuccess)
        rc = fail(FD_ERR_CUDA, "cudaMalloc failed");
    if (rc == FD_OK) {
        const int tot = p.n_pad * 64;
        if (dtype == FD_F16) pack_stem_w_kernel<__half><<<(tot + 127) / 128, 128>>>(wk_dev, (__half*)sp->w16, g.c_in, g.c_out, p.n_pad);
        else pack_stem_w_kernel<__nv_bfloat16><<<(tot + 127) / 128, 128>>>(wk_dev, (__nv_bfloat16*)sp->w16, g.c_in, g.c_out, p.n_pad);
        pack_stem_affine_kernel<<<(p.n_pad + 127) / 128, 128>>>(scale_dev, bias_dev, sp->affine, g.c_out, p.n_pad);
        if (cudaGetLastError() != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) rc = fail(FD_ERR_CUDA, "stem parameter packing failed");
    }
    if (rc != FD_OK) { stem_tc_destroy(sp); return rc; }
    p.affine = sp->affine;
    {
        const CUtensorMapDataType dt = dtype == FD_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
        cuuint64_t dims[2] = {64, (cuuint64_t)p.n_pad};
        cuuint64_t strides[1] = {128};
        cuuint32_t box[2] = {64, (cuuint32_t)p.n_pad};
        cuuint32_t estr[2] = {1, 1};
        CUresult r = encode(&sp->tm_w, dt, 2, sp->w16, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { stem_tc_destroy(sp); return fail(FD_ERR_CUDA, "cuTensorMapEncodeTiled(stem weights) failed"); }
    }
    sp->smem_bytes = (size_t)ST_S_A * ST_A_BYTES + (size_t)p.n_pad * 128 + (size_t)ST_S_IN * st_in_stride(g.c_in) + (size_t)p.n_pad * 8 +
                     sizeof(StemBarriers) + 1024;
    const int sms = opts.n_sms;
    sp->opts = opts;
    sp->grid = dim3((unsigned)(p.items < sms ? p.items : sms), 1, 1);
    char buf[96];
    if (g.c_in == 3) snprintf(buf, sizeof(buf), "stem_tc<k3,s2,1x8x16>[n%d]", p.n_pad);
    else snprintf(buf, sizeof(buf), "stem_tc<k3,s2,1x8x16,cin%d>[n%d]", g.c_in, p.n_pad);
    sp->name = buf;
    *res = sp;
    return FD_OK;
}

size_t stem_tc_param_bytes(StemTcPlan* sp) { return (size_t)sp->p.n_pad * (64 * 2 + sizeof(float2)); }
const char* stem_tc_name(StemTcPlan* sp) { return sp->name.c_str(); }

template <typename T, int CIN>
static int launch_stem_tc(StemTcPlan* sp, cudaLaunchConfig_t& cfg) {
    static PerDeviceOnce attr_done;            // the dynamic shared-memory opt-in is per device and per kernel instance
    int dev = -1;
    FD_CUDA_OK(cudaGetDevice(&dev));
    if (attr_done.need(dev)) {
        FD_CUDA_OK(cudaFuncSetAttribute(stem_tc_kernel<T, CIN>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        attr_done.done(dev);
    }
    FD_CUDA_OK(cudaLaunchKernelEx(&cfg, stem_tc_kernel<T, CIN>, sp->tm_in, sp->tm_w, sp->p));
    return FD_OK;
}

template <typename T>
static int launch_stem_cin(StemTcPlan* sp, cudaLaunchConfig_t& cfg) {
    switch (sp->c_in) {
        case 1: return launch_stem_tc<T, 1>(sp, cfg);
        case 2: return launch_stem_tc<T, 2>(sp, cfg);
        case 3: return launch_stem_tc<T, 3>(sp, cfg);
        case 4: return launch_stem_tc<T, 4>(sp, cfg);
        case 5: return launch_stem_tc<T, 5>(sp, cfg);
        case 6: return launch_stem_tc<T, 6>(sp, cfg);
        case 7: return launch_stem_tc<T, 7>(sp, cfg);
        default: return fail(FD_ERR_UNSUPPORTED, "stem_tc_kernel: c_in must be 1..7");
    }
}

// x may change from call to call (the caller's tensor): re-encode the input tensor map when it does.  Under CUDA-graph
// capture the map is baked into the captured launch, which is keyed on (x, y) by the caller.
int stem_tc_launch(StemTcPlan* sp, const void* x, cudaStream_t st) {
    if ((reinterpret_cast<uintptr_t>(x) & 15) != 0) return fail(FD_ERR_INVALID, "stem input must be 16-byte aligned");
    if (x != sp->x_bound) {
        int rc = encode_input_map(sp, x);
        if (rc) return rc;
    }
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = sp->grid; cfg.blockDim = dim3(ST_THREADS); cfg.dynamicSmemBytes = sp->smem_bytes; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = sp->opts.pdl ? 1 : 0;
    int rc;
    if (sp->dtype == FD_F16) rc = launch_stem_cin<__half>(sp, cfg);
    else rc = launch_stem_cin<__nv_bfloat16>(sp, cfg);
    if (rc) return rc;
    FD_CUDA_OK(cudaGetLastError());
    return FD_OK;
}

}  // namespace fd
