// SIMT kernels of the FastDepth forward path (all dtypes).
//
//  * stem_kernel  : conv_bn(c_in,C0,s2)+BN+ReLU6, NCHW in -> NHWC out, c_in 1..7
//                                                                      (reference imagenet/mobilenet.py:22-27,41; models.py:443-453)
//  * dw_kernel    : depthwise kxk(stride)+BN+act, NHWC                (reference imagenet/mobilenet.py:31-33; models.py:61-68)
//  * pw_kernel    : pointwise 1x1+BN+act as a tiled SIMT GEMM, with the decoder's nearest-x2
//                   upsample + skip add in the epilogue               (reference imagenet/mobilenet.py:35-37; models.py:70-75,723-729)
//  * conv_kernel  : dense kxk stride-1 conv+BN+act (+ nearest x2 upsample) of the dense NNConv decoder
//                                                                      (reference models.py:52-59, 245-270)
//  * convt_kernel : transposed conv / unpool + 5x5 conv, +BN+act, of the DeConv and UpConv decoders, one output phase per
//                   grid z                                            (reference models.py:18-34, 77-107, 145-201)
//  * head_kernel  : pointwise(C,1)+BN+ReLU -> [N,1,H,W] (optionally below the last upsample)
//                                                                      (reference models.py:698,731)
//
// dw_kernel + pw_kernel are "path 0": the unfused, reference-quality implementation every
// dtype can run (it is the fp32 path and the on-device cross-check for the fused wgmma
// block kernel in fd_block_tc.cu).  All accumulate in fp32 and apply BN as a folded fp32
// per-channel affine, then round once to the storage dtype.
#include "fd_common.cuh"
#include "fd_conv_plan.h"

namespace fd {

// ----------------------------------------------------------------------------------------
// stem
// ----------------------------------------------------------------------------------------
template <typename T, int CIN>
__global__ void __launch_bounds__(256)
stem_kernel(const T* __restrict__ x, T* __restrict__ out, const float* __restrict__ w,
            const float* __restrict__ scale, const float* __restrict__ bias,
            int n, int h_in, int w_in, int h_out, int w_out, int c_out, int out_pitch, int stride, int act) {
    extern __shared__ float s_w[];                 // [9 c_in][c_out] tap-major, then scale, bias
    const int nw = 9 * CIN * c_out;
    for (int i = threadIdx.x; i < nw; i += blockDim.x) s_w[i] = w[i];
    float* s_scale = s_w + nw;
    float* s_bias = s_scale + c_out;
    for (int i = threadIdx.x; i < c_out; i += blockDim.x) { s_scale[i] = scale[i]; s_bias[i] = bias[i]; }
    __syncthreads();

    const int groups = c_out >> 3;
    const long long total = (long long)n * h_out * w_out * groups;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int g = (int)(idx % groups);
    long long p = idx / groups;
    const int ox = (int)(p % w_out); p /= w_out;
    const int oy = (int)(p % h_out);
    const int img = (int)(p / h_out);

    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    const size_t plane = (size_t)h_in * w_in;
    const T* xi = x + (size_t)img * CIN * plane;
#pragma unroll
    for (int ci = 0; ci < CIN; ++ci) {
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) {
            const int iy = oy * stride - 1 + ky;
            if (iy < 0 || iy >= h_in) continue;
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
                const int ix = ox * stride - 1 + kx;
                if (ix < 0 || ix >= w_in) continue;
                const float v = Traits<T>::to_f(xi[ci * plane + (size_t)iy * w_in + ix]);
                const float* wp = s_w + ((ci * 3 + ky) * 3 + kx) * c_out + g * 8;
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[j] = fmaf(v, wp[j], acc[j]);
            }
        }
    }
    float y[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) y[j] = apply_act(fmaf(acc[j], s_scale[g * 8 + j], s_bias[g * 8 + j]), act);
    T* op = out + (((size_t)img * h_out + oy) * w_out + ox) * out_pitch + g * 8;
    store8<T>(op, y);
}

// ----------------------------------------------------------------------------------------
// depthwise (unfused path)
// ----------------------------------------------------------------------------------------
template <typename T, int K>
__global__ void __launch_bounds__(256)
dw_kernel(const T* __restrict__ in, T* __restrict__ out, const float* __restrict__ w,
          const float* __restrict__ scale, const float* __restrict__ bias,
          int n, int h_in, int w_in, int h_out, int w_out, int c, int in_pitch, int stride, int act) {
    const int groups = c >> 3;
    const long long total = (long long)n * h_out * w_out * groups;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int g = (int)(idx % groups);
    long long p = idx / groups;
    const int ox = (int)(p % w_out); p /= w_out;
    const int oy = (int)(p % h_out);
    const int img = (int)(p / h_out);
    constexpr int PAD = (K - 1) / 2;

    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    const T* base = in + (size_t)img * h_in * w_in * in_pitch + g * 8;
#pragma unroll
    for (int ky = 0; ky < K; ++ky) {
        const int iy = oy * stride - PAD + ky;
        if (iy < 0 || iy >= h_in) continue;
#pragma unroll
        for (int kx = 0; kx < K; ++kx) {
            const int ix = ox * stride - PAD + kx;
            if (ix < 0 || ix >= w_in) continue;
            float v[8], wv[8];
            load8<T>(base + ((size_t)iy * w_in + ix) * in_pitch, v);
            load8<float>(w + (size_t)(ky * K + kx) * c + g * 8, wv);
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j] = fmaf(v[j], wv[j], acc[j]);
        }
    }
    float sc[8], bi[8], y[8];
    load8<float>(scale + g * 8, sc);
    load8<float>(bias + g * 8, bi);
#pragma unroll
    for (int j = 0; j < 8; ++j) y[j] = apply_act(fmaf(acc[j], sc[j], bi[j]), act);
    store8<T>(out + (((size_t)img * h_out + oy) * w_out + ox) * c + g * 8, y);
}

// ----------------------------------------------------------------------------------------
// pointwise GEMM (unfused path): out[m, co] = act(scale[co] * sum_k A[m,k] W[co,k] + bias[co])
// optional epilogue: nearest-x2 upsample (+ skip add at the upsampled resolution)
// ----------------------------------------------------------------------------------------
constexpr int PW_BM = 64, PW_BN = 64, PW_BK = 16, PW_THREADS = 256;

template <typename T>
__device__ __forceinline__ void load4f(const T* p, float (&o)[4]);
template <> __device__ __forceinline__ void load4f<float>(const float* p, float (&o)[4]) {
    float4 a = __ldg(reinterpret_cast<const float4*>(p)); o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.w;
}
template <> __device__ __forceinline__ void load4f<__half>(const __half* p, float (&o)[4]) {
    uint2 r = __ldg(reinterpret_cast<const uint2*>(p));
    const __half2* h = reinterpret_cast<const __half2*>(&r);
    float2 a = __half22float2(h[0]), b = __half22float2(h[1]); o[0] = a.x; o[1] = a.y; o[2] = b.x; o[3] = b.y;
}
template <> __device__ __forceinline__ void load4f<__nv_bfloat16>(const __nv_bfloat16* p, float (&o)[4]) {
    uint2 r = __ldg(reinterpret_cast<const uint2*>(p));
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&r);
    float2 a = __bfloat1622float2(h[0]), b = __bfloat1622float2(h[1]); o[0] = a.x; o[1] = a.y; o[2] = b.x; o[3] = b.y;
}
template <typename T>
__device__ __forceinline__ void store4f(T* p, const float (&v)[4]);
template <> __device__ __forceinline__ void store4f<float>(float* p, const float (&v)[4]) {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
}
template <> __device__ __forceinline__ void store4f<__half>(__half* p, const float (&v)[4]) {
    uint2 r; __half2* h = reinterpret_cast<__half2*>(&r);
    h[0] = __floats2half2_rn(v[0], v[1]); h[1] = __floats2half2_rn(v[2], v[3]);
    *reinterpret_cast<uint2*>(p) = r;
}
template <> __device__ __forceinline__ void store4f<__nv_bfloat16>(__nv_bfloat16* p, const float (&v)[4]) {
    uint2 r; __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&r);
    h[0] = __floats2bfloat162_rn(v[0], v[1]); h[1] = __floats2bfloat162_rn(v[2], v[3]);
    *reinterpret_cast<uint2*>(p) = r;
}

template <typename T>
__global__ void __launch_bounds__(PW_THREADS)
pw_kernel(const T* __restrict__ a, const T* __restrict__ wgt, T* __restrict__ out, const T* __restrict__ skip,
          const float* __restrict__ scale, const float* __restrict__ bias,
          long long m_total, int c_in, int c_out, int out_pitch, int skip_pitch, int h, int w, int upsample, int act) {
    __shared__ float As[PW_BK][PW_BM + 4];
    __shared__ float Ws[PW_BK][PW_BN + 4];
    const int tid = threadIdx.x;
    const long long m0 = (long long)blockIdx.x * PW_BM;
    const int n0 = blockIdx.y * PW_BN;
    const int lr = tid >> 2;            // 0..63: tile row this thread loads
    const int lk = (tid & 3) * 4;       // k offset within the BK slab
    const int ty = tid >> 4, tx = tid & 15;   // 16x16 threads, 4x4 outputs each

    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    for (int k0 = 0; k0 < c_in; k0 += PW_BK) {
        float va[4] = {0.f, 0.f, 0.f, 0.f}, vw[4] = {0.f, 0.f, 0.f, 0.f};
        if (m0 + lr < m_total && k0 + lk < c_in) load4f<T>(a + (size_t)(m0 + lr) * c_in + k0 + lk, va);
        if (n0 + lr < c_out && k0 + lk < c_in) load4f<T>(wgt + (size_t)(n0 + lr) * c_in + k0 + lk, vw);
#pragma unroll
        for (int j = 0; j < 4; ++j) { As[lk + j][lr] = va[j]; Ws[lk + j][lr] = vw[j]; }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < PW_BK; ++k) {
            float ra[4], rw[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) { ra[i] = As[k][ty * 4 + i]; rw[i] = Ws[k][tx * 4 + i]; }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(ra[i], rw[j], acc[i][j]);
        }
        __syncthreads();
    }

    const int co = n0 + tx * 4;
    if (co >= c_out) return;            // c_out % 8 == 0 and co % 4 == 0 -> the 4 columns are all valid
    float sc[4], bi[4];
    load4f<float>(scale + co, sc);
    load4f<float>(bias + co, bi);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const long long m = m0 + ty * 4 + i;
        if (m >= m_total) continue;
        float y[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) y[j] = apply_act(fmaf(acc[i][j], sc[j], bi[j]), act);
        if (!upsample) {
            store4f<T>(out + (size_t)m * out_pitch + co, y);
        } else {
            const int px = (int)(m % w);
            const long long t = m / w;
            const int py = (int)(t % h);
            const long long img = t / h;
            const int w2 = 2 * w;
#pragma unroll
            for (int dy = 0; dy < 2; ++dy)
#pragma unroll
                for (int dx = 0; dx < 2; ++dx) {
                    const size_t pix = ((size_t)img * 2 * h + 2 * py + dy) * w2 + 2 * px + dx;
                    const size_t o = pix * out_pitch + co;
                    float z[4] = {y[0], y[1], y[2], y[3]};
                    if (skip != nullptr) {
                        float s[4];
                        load4f<T>(skip + pix * skip_pitch + co, s);
                        // the reference rounds the upsampled tensor to the storage dtype BEFORE the
                        // add (x = F.interpolate(x); x = x + skip, models.py:723-729)
#pragma unroll
                        for (int j = 0; j < 4; ++j) z[j] = Traits<T>::to_f(Traits<T>::from_f(z[j])) + s[j];
                    }
                    store4f<T>(out + o, z);
                }
        }
    }
}

// ----------------------------------------------------------------------------------------
// dense kxk stride-1 conv (padding (k-1)/2) + BN + act (+ nearest x2 upsample), path 0: the pointwise GEMM above with the
// A rows gathered straight from the NHWC input (K = k*k*c_in, tap-major; c_in % 8 == 0, so a 4-channel load never
// straddles two taps).  Weights [c_out][k*k][c_in] in the plan dtype.
// ----------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(PW_THREADS)
conv_kernel(const T* __restrict__ in, const T* __restrict__ wgt, T* __restrict__ out,
            const float* __restrict__ scale, const float* __restrict__ bias,
            int n, int h, int w, int c_in, int c_out, int in_pitch, int out_pitch, int ks, int upsample, int act) {
    __shared__ float As[PW_BK][PW_BM + 4];
    __shared__ float Ws[PW_BK][PW_BN + 4];
    const int tid = threadIdx.x;
    const long long m_total = (long long)n * h * w;
    const long long m0 = (long long)blockIdx.x * PW_BM;
    const int n0 = blockIdx.y * PW_BN;
    const int lr = tid >> 2;
    const int lk = (tid & 3) * 4;
    const int ty = tid >> 4, tx = tid & 15;
    const int pad = (ks - 1) / 2;
    const int k_total = ks * ks * c_in;
    // the pixel this thread loads A rows for
    const long long lm = m0 + lr;
    const int lx = (int)(lm % w);
    const int ly = (int)((lm / w) % h);
    const long long limg = lm / ((long long)w * h);

    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    for (int k0 = 0; k0 < k_total; k0 += PW_BK) {
        float va[4] = {0.f, 0.f, 0.f, 0.f}, vw[4] = {0.f, 0.f, 0.f, 0.f};
        const int kk = k0 + lk;
        if (kk < k_total) {
            const int tap = kk / c_in, ci = kk - tap * c_in;
            const int iy = ly + tap / ks - pad, ix = lx + tap % ks - pad;
            if (lm < m_total && iy >= 0 && iy < h && ix >= 0 && ix < w)
                load4f<T>(in + (((size_t)limg * h + iy) * w + ix) * in_pitch + ci, va);
            if (n0 + lr < c_out) load4f<T>(wgt + (size_t)(n0 + lr) * k_total + kk, vw);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) { As[lk + j][lr] = va[j]; Ws[lk + j][lr] = vw[j]; }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < PW_BK; ++k) {
            float ra[4], rw[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) { ra[i] = As[k][ty * 4 + i]; rw[i] = Ws[k][tx * 4 + i]; }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(ra[i], rw[j], acc[i][j]);
        }
        __syncthreads();
    }

    const int co = n0 + tx * 4;
    if (co >= c_out) return;
    float sc[4], bi[4];
    load4f<float>(scale + co, sc);
    load4f<float>(bias + co, bi);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const long long m = m0 + ty * 4 + i;
        if (m >= m_total) continue;
        float y[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) y[j] = apply_act(fmaf(acc[i][j], sc[j], bi[j]), act);
        if (!upsample) {
            store4f<T>(out + (size_t)m * out_pitch + co, y);
        } else {
            const int px = (int)(m % w);
            const long long t = m / w;
            const int py = (int)(t % h);
            const long long img = t / h;
#pragma unroll
            for (int dy = 0; dy < 2; ++dy)
#pragma unroll
                for (int dx = 0; dx < 2; ++dx)
                    store4f<T>(out + (((size_t)img * 2 * h + 2 * py + dy) * (2 * w) + 2 * px + dx) * out_pitch + co, y);
        }
    }
}

// ----------------------------------------------------------------------------------------
// transposed conv (DECONV) / unpool + conv (UPCONV) + BN + act, path 0: blockIdx.z is the output phase q = 2 ry + rx; the GEMM
// above over the n*h*w input-resolution pixels (Y, X) with K = that phase's taps * c_in, the A row of (Y, X) gathered at
// (Y + dy, X + dx) (only the taps the phase really has), the result stored at output pixel (2 Y + ry, 2 X + rx).  Weights
// [c_out][k*k][c_in] with phase-major taps (fd_conv_plan.h).
// ----------------------------------------------------------------------------------------
struct ConvPhases { ConvPhase ph[4]; };

template <typename T>
__global__ void __launch_bounds__(PW_THREADS)
convt_kernel(const T* __restrict__ in, const T* __restrict__ wgt, T* __restrict__ out,
             const float* __restrict__ scale, const float* __restrict__ bias,
             int n, int h, int w, int c_in, int c_out, int in_pitch, int out_pitch, int taps, const ConvPhases phs, int act) {
    __shared__ float As[PW_BK][PW_BM + 4];
    __shared__ float Ws[PW_BK][PW_BN + 4];
    const int q = blockIdx.z;
    const ConvPhase f = phs.ph[q];
    const int tid = threadIdx.x;
    const long long m_total = (long long)n * h * w;
    const long long m0 = (long long)blockIdx.x * PW_BM;
    const int n0 = blockIdx.y * PW_BN;
    const int lr = tid >> 2;
    const int lk = (tid & 3) * 4;
    const int ty = tid >> 4, tx = tid & 15;
    const int k_total = f.ny * f.nx * c_in;
    const long long lm = m0 + lr;
    const int lx = (int)(lm % w);
    const int ly = (int)((lm / w) % h);
    const long long limg = lm / ((long long)w * h);

    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    for (int k0 = 0; k0 < k_total; k0 += PW_BK) {
        float va[4] = {0.f, 0.f, 0.f, 0.f}, vw[4] = {0.f, 0.f, 0.f, 0.f};
        const int kk = k0 + lk;
        if (kk < k_total) {
            const int tap = kk / c_in, ci = kk - tap * c_in;
            const int iy = ly + f.dy0 + tap / f.nx, ix = lx + f.dx0 + tap % f.nx;
            if (lm < m_total && iy >= 0 && iy < h && ix >= 0 && ix < w)
                load4f<T>(in + (((size_t)limg * h + iy) * w + ix) * in_pitch + ci, va);
            if (n0 + lr < c_out) load4f<T>(wgt + ((size_t)(n0 + lr) * taps + f.tap0 + tap) * c_in + ci, vw);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) { As[lk + j][lr] = va[j]; Ws[lk + j][lr] = vw[j]; }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < PW_BK; ++k) {
            float ra[4], rw[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) { ra[i] = As[k][ty * 4 + i]; rw[i] = Ws[k][tx * 4 + i]; }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(ra[i], rw[j], acc[i][j]);
        }
        __syncthreads();
    }

    const int co = n0 + tx * 4;
    if (co >= c_out) return;
    float sc[4], bi[4];
    load4f<float>(scale + co, sc);
    load4f<float>(bias + co, bi);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const long long m = m0 + ty * 4 + i;
        if (m >= m_total) continue;
        float y[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) y[j] = apply_act(fmaf(acc[i][j], sc[j], bi[j]), act);
        const int px = (int)(m % w);
        const long long t = m / w;
        const int py = (int)(t % h);
        const long long img = t / h;
        store4f<T>(out + (((size_t)img * 2 * h + 2 * py + (q >> 1)) * (2 * w) + 2 * px + (q & 1)) * out_pitch + co, y);
    }
}

// ----------------------------------------------------------------------------------------
// head: C -> 1 pointwise + BN + ReLU, written as [N,1,H,W]; with up=1 every low-res result is
// replicated to its 2x2 block (decode_conv6 commutes with the last nearest upsample)
// ----------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256)
head_kernel(const T* __restrict__ in, T* __restrict__ out, const float* __restrict__ w, float scale, float bias,
            long long m_total, int c, int in_pitch, int h, int wd, int up, int act) {
    const long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= m_total) return;
    const T* p = in + (size_t)m * in_pitch;
    float acc = 0.f;
    for (int k = 0; k < c; k += 8) {
        float v[8], wv[8];
        load8<T>(p + k, v);
        load8<float>(w + k, wv);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc = fmaf(v[j], wv[j], acc);
    }
    const T y = Traits<T>::from_f(apply_act(fmaf(acc, scale, bias), act));
    if (!up) {
        out[m] = y;
    } else {
        const int px = (int)(m % wd);
        const long long t = m / wd;
        const int py = (int)(t % h);
        const long long img = t / h;
        T* o = out + ((size_t)img * 2 * h + 2 * py) * (2 * wd) + 2 * px;
        o[0] = y; o[1] = y; o[2 * wd] = y; o[2 * wd + 1] = y;
    }
}

// ----------------------------------------------------------------------------------------
// launchers (host)
// ----------------------------------------------------------------------------------------
template <typename T>
static int launch_stem_t(const void* x, void* out, const float* w, const float* scale, const float* bias,
                         const StageGeom& g, cudaStream_t st) {
    const long long total = (long long)g.n * g.h_out * g.w_out * (g.c_out / 8);
    const int threads = 256;
    const long long blocks = (total + threads - 1) / threads;
    const size_t smem = (size_t)(9 * g.c_in + 2) * g.c_out * sizeof(float);
    decltype(&stem_kernel<T, 3>) k;
    switch (g.c_in) {
        case 1: k = stem_kernel<T, 1>; break;
        case 2: k = stem_kernel<T, 2>; break;
        case 3: k = stem_kernel<T, 3>; break;
        case 4: k = stem_kernel<T, 4>; break;
        case 5: k = stem_kernel<T, 5>; break;
        case 6: k = stem_kernel<T, 6>; break;
        case 7: k = stem_kernel<T, 7>; break;
        default: return fail(FD_ERR_UNSUPPORTED, "stem_kernel: c_in must be 1..7");
    }
    if (smem > 48 * 1024) FD_CUDA_OK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k<<<(unsigned)blocks, threads, smem, st>>>((const T*)x, (T*)out, w, scale, bias, g.n, g.h_in, g.w_in, g.h_out, g.w_out,
                                               g.c_out, g.out_pitch, g.stride, g.act);
    FD_CUDA_OK(cudaGetLastError());
    return FD_OK;
}

template <typename T>
static int launch_dw_t(const BlockArgs& a, cudaStream_t st) {
    const StageGeom& g = a.g;
    const long long total = (long long)g.n * g.h_out * g.w_out * (g.c_in / 8);
    const int threads = 256;
    const unsigned blocks = (unsigned)((total + threads - 1) / threads);
    if (g.ksize == 3)
        dw_kernel<T, 3><<<blocks, threads, 0, st>>>((const T*)a.in, (T*)a.mid, a.dw_w, a.dw_scale, a.dw_bias, g.n, g.h_in,
                                                    g.w_in, g.h_out, g.w_out, g.c_in, g.in_pitch, g.stride, g.act);
    else if (g.ksize == 5)
        dw_kernel<T, 5><<<blocks, threads, 0, st>>>((const T*)a.in, (T*)a.mid, a.dw_w, a.dw_scale, a.dw_bias, g.n, g.h_in,
                                                    g.w_in, g.h_out, g.w_out, g.c_in, g.in_pitch, g.stride, g.act);
    else
        return fail(FD_ERR_UNSUPPORTED, "depthwise kernel size must be 3 or 5");
    FD_CUDA_OK(cudaGetLastError());
    return FD_OK;
}

template <typename T>
static int launch_pw_t(const BlockArgs& a, cudaStream_t st) {
    const StageGeom& g = a.g;
    const long long m_total = (long long)g.n * g.h_out * g.w_out;
    dim3 grid((unsigned)((m_total + PW_BM - 1) / PW_BM), (unsigned)((g.c_out + PW_BN - 1) / PW_BN));
    pw_kernel<T><<<grid, PW_THREADS, 0, st>>>((const T*)a.mid, (const T*)a.pw_w, (T*)a.out, (const T*)a.skip, a.pw_scale,
                                              a.pw_bias, m_total, g.c_in, g.c_out, g.out_pitch, g.skip_pitch, g.h_out, g.w_out, g.upsample, g.act);
    FD_CUDA_OK(cudaGetLastError());
    return FD_OK;
}

template <typename T>
static int launch_conv_t(const void* in, const void* w, void* out, const float* scale, const float* bias, const StageGeom& g,
                         cudaStream_t st) {
    const long long m_total = (long long)g.n * g.h_out * g.w_out;
    dim3 grid((unsigned)((m_total + PW_BM - 1) / PW_BM), (unsigned)((g.c_out + PW_BN - 1) / PW_BN));
    conv_kernel<T><<<grid, PW_THREADS, 0, st>>>((const T*)in, (const T*)w, (T*)out, scale, bias, g.n, g.h_out, g.w_out, g.c_in,
                                                g.c_out, g.in_pitch > 0 ? g.in_pitch : g.c_in, g.out_pitch > 0 ? g.out_pitch : g.c_out,
                                                g.ksize, g.upsample, g.act);
    FD_CUDA_OK(cudaGetLastError());
    return FD_OK;
}

template <typename T>
static int launch_convt_t(int kind, const void* in, const void* w, void* out, const float* scale, const float* bias,
                          const StageGeom& g, cudaStream_t st) {
    ConvPhases phs;
    conv_phases(kind, g.ksize, phs.ph);
    const long long m_total = (long long)g.n * g.h_out * g.w_out;
    dim3 grid((unsigned)((m_total + PW_BM - 1) / PW_BM), (unsigned)((g.c_out + PW_BN - 1) / PW_BN), 4);
    convt_kernel<T><<<grid, PW_THREADS, 0, st>>>((const T*)in, (const T*)w, (T*)out, scale, bias, g.n, g.h_out, g.w_out, g.c_in,
                                                 g.c_out, g.in_pitch > 0 ? g.in_pitch : g.c_in,
                                                 g.out_pitch > 0 ? g.out_pitch : g.c_out, g.ksize * g.ksize, phs, g.act);
    FD_CUDA_OK(cudaGetLastError());
    return FD_OK;
}

template <typename T>
static int launch_head_t(const void* in, void* out, const float* w, float scale, float bias, long long m_total, int c,
                         int in_pitch, int h, int wd, int up, int act, cudaStream_t st) {
    const int threads = 256;
    const unsigned blocks = (unsigned)((m_total + threads - 1) / threads);
    head_kernel<T><<<blocks, threads, 0, st>>>((const T*)in, (T*)out, w, scale, bias, m_total, c, in_pitch, h, wd, up, act);
    FD_CUDA_OK(cudaGetLastError());
    return FD_OK;
}

#define FD_DISPATCH(dtype, CALL)                                          \
    switch (dtype) {                                                      \
        case FD_F32: { using T = float; return CALL; }                    \
        case FD_F16: { using T = __half; return CALL; }                   \
        case FD_BF16: { using T = __nv_bfloat16; return CALL; }           \
        default: return fail(FD_ERR_INVALID, "bad dtype");                \
    }

int launch_stem(int dtype, const void* x, void* out, const float* w, const float* scale, const float* bias,
                const StageGeom& g, cudaStream_t st) {
    FD_DISPATCH(dtype, launch_stem_t<T>(x, out, w, scale, bias, g, st));
}
int launch_dw(int dtype, const BlockArgs& a, cudaStream_t st) { FD_DISPATCH(dtype, launch_dw_t<T>(a, st)); }
int launch_pw(int dtype, const BlockArgs& a, cudaStream_t st) { FD_DISPATCH(dtype, launch_pw_t<T>(a, st)); }
int launch_conv(int dtype, const void* in, const void* w, void* out, const float* scale, const float* bias, const StageGeom& g,
                cudaStream_t st) {
    FD_DISPATCH(dtype, launch_conv_t<T>(in, w, out, scale, bias, g, st));
}
int launch_convt(int dtype, int kind, const void* in, const void* w, void* out, const float* scale, const float* bias,
                 const StageGeom& g, cudaStream_t st) {
    FD_DISPATCH(dtype, launch_convt_t<T>(kind, in, w, out, scale, bias, g, st));
}
int launch_head(int dtype, const void* in, void* out, const float* w, float scale, float bias, long long m_total, int c,
                int in_pitch, int h, int wd, int up, int act, cudaStream_t st) {
    FD_DISPATCH(dtype, launch_head_t<T>(in, out, w, scale, bias, m_total, c, in_pitch, h, wd, up, act, st));
}

}  // namespace fd
