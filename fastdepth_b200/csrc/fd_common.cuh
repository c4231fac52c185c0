// Shared device/host helpers for the fastdepth_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <string>

#include "../../include/fastdepth_b200.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "fastdepth_b200 targets sm_90a only (-gencode arch=compute_90a,code=sm_90a)"
#endif

namespace fd {

// ----------------------------------------------------------------------------------------
// error plumbing (thread-local message behind fd_last_error())
// ----------------------------------------------------------------------------------------
void set_error(const std::string& msg);
int fail(int code, const std::string& msg);

#define FD_CUDA_OK(expr)                                                                         \
    do {                                                                                         \
        cudaError_t _e = (expr);                                                                 \
        if (_e != cudaSuccess)                                                                   \
            return ::fd::fail(FD_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e));  \
    } while (0)

// ----------------------------------------------------------------------------------------
// dtype traits: storage type T in {float, __half, __nv_bfloat16}; math always fp32
// ----------------------------------------------------------------------------------------
template <typename T> struct Traits;
template <> struct Traits<float> {
    static constexpr int kDtype = FD_F32;
    static constexpr int kVec = 4;                     // elements per 16-byte vector
    __device__ __forceinline__ static float to_f(float v) { return v; }
    __device__ __forceinline__ static float from_f(float v) { return v; }
};
template <> struct Traits<__half> {
    static constexpr int kDtype = FD_F16;
    static constexpr int kVec = 8;
    __device__ __forceinline__ static float to_f(__half v) { return __half2float(v); }
    __device__ __forceinline__ static __half from_f(float v) { return __float2half_rn(v); }
};
template <> struct Traits<__nv_bfloat16> {
    static constexpr int kDtype = FD_BF16;
    static constexpr int kVec = 8;
    __device__ __forceinline__ static float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
    __device__ __forceinline__ static __nv_bfloat16 from_f(float v) { return __float2bfloat16_rn(v); }
};

// 8 consecutive channels as fp32, loaded/stored with the widest aligned vectors.
template <typename T> struct Vec8 { float v[8]; };

template <typename T>
__device__ __forceinline__ void load8(const T* __restrict__ p, float (&out)[8]);
template <>
__device__ __forceinline__ void load8<float>(const float* __restrict__ p, float (&out)[8]) {
    float4 a = __ldg(reinterpret_cast<const float4*>(p));
    float4 b = __ldg(reinterpret_cast<const float4*>(p) + 1);
    out[0] = a.x; out[1] = a.y; out[2] = a.z; out[3] = a.w;
    out[4] = b.x; out[5] = b.y; out[6] = b.z; out[7] = b.w;
}
template <>
__device__ __forceinline__ void load8<__half>(const __half* __restrict__ p, float (&out)[8]) {
    uint4 r = __ldg(reinterpret_cast<const uint4*>(p));
    const __half2* h = reinterpret_cast<const __half2*>(&r);
#pragma unroll
    for (int i = 0; i < 4; ++i) { float2 f = __half22float2(h[i]); out[2 * i] = f.x; out[2 * i + 1] = f.y; }
}
template <>
__device__ __forceinline__ void load8<__nv_bfloat16>(const __nv_bfloat16* __restrict__ p, float (&out)[8]) {
    uint4 r = __ldg(reinterpret_cast<const uint4*>(p));
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&r);
#pragma unroll
    for (int i = 0; i < 4; ++i) { float2 f = __bfloat1622float2(h[i]); out[2 * i] = f.x; out[2 * i + 1] = f.y; }
}

template <typename T>
__device__ __forceinline__ void store8(T* __restrict__ p, const float (&in)[8]);
template <>
__device__ __forceinline__ void store8<float>(float* __restrict__ p, const float (&in)[8]) {
    reinterpret_cast<float4*>(p)[0] = make_float4(in[0], in[1], in[2], in[3]);
    reinterpret_cast<float4*>(p)[1] = make_float4(in[4], in[5], in[6], in[7]);
}
template <>
__device__ __forceinline__ void store8<__half>(__half* __restrict__ p, const float (&in)[8]) {
    uint4 r;
    __half2* h = reinterpret_cast<__half2*>(&r);
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(in[2 * i], in[2 * i + 1]);
    *reinterpret_cast<uint4*>(p) = r;
}
template <>
__device__ __forceinline__ void store8<__nv_bfloat16>(__nv_bfloat16* __restrict__ p, const float (&in)[8]) {
    uint4 r;
    __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&r);
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(in[2 * i], in[2 * i + 1]);
    *reinterpret_cast<uint4*>(p) = r;
}

__device__ __forceinline__ float apply_act(float v, int act) {
    v = fmaxf(v, 0.0f);
    return act == FD_ACT_RELU6 ? fminf(v, 6.0f) : v;
}

// ----------------------------------------------------------------------------------------
// stage description shared by host planning code and kernel launchers
// ----------------------------------------------------------------------------------------
struct StageGeom {
    int n, h_in, w_in, h_out, w_out;   // h_out/w_out: spatial size of the conv output (pre-upsample)
    int c_in, c_out;
    int ksize, stride, act;
    int upsample;                      // 0/1
    int in_pitch, out_pitch;           // elements between consecutive pixels of the input / output tensor (>= channels;
                                       // larger when the tensor is a channel slice of a wider concat buffer)
    int skip_pitch;                    // same for the skip tensor of an ADD stage
};

// Launch-time options of a plan (fd_plan_set_option), copied into every kernel plan when it is built so that two plans with
// different options never share mutable state.
struct TcLaunchOpts {
    int pdl = 1;             // programmatic dependent launch attribute on every launch
    int sleep_ns = 0;        // > 0: latency-tolerant mbarrier waits back off with nanosleep instead of spinning
    int n_sms = 132;         // SMs of the plan's device (grid size and the planner's wave model)
    int cluster = 1;         // 1: the block planner may run small-map blocks on thread-block clusters that share the depthwise half
};

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) is a per-DEVICE property of a kernel: remember which devices have it.
struct PerDeviceOnce {
    unsigned long long mask = 0;
    bool need(int dev) const { return dev < 0 || dev >= 64 || !((mask >> dev) & 1ull); }
    void done(int dev) { if (dev >= 0 && dev < 64) mask |= 1ull << dev; }
};

// Launch argument bundle for one fused / unfused block stage.
struct BlockArgs {
    StageGeom g;
    const void* in;          // NHWC [n, h_in, w_in, c_in]
    void* mid;               // NHWC [n, h_out, w_out, c_in]   (path 0 only)
    void* out;               // NHWC [n, h_out*(1+up), w_out*(1+up), c_out]
    const void* skip;        // NHWC same shape as out, or nullptr
    const float* dw_w;       // [k*k][c_in] fp32 (tap-major so 8 channels are contiguous)
    const float* dw_scale;   // [c_in]
    const float* dw_bias;    // [c_in]
    const void* pw_w;        // [c_out][c_in] plan dtype
    const float* pw_scale;   // [c_out]
    const float* pw_bias;    // [c_out]
};

}  // namespace fd
