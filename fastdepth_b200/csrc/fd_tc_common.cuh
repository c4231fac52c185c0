// wgmma / TMA / mbarrier / cluster PTX wrappers shared by the sm_90a tensor-core kernels
// (fd_block_tc.cu: fused depthwise->pointwise blocks; fd_stem_tc.cu: im2col stem; fd_conv_tc.cu: dense kxk conv).
#pragma once
#include <cuda.h>
#include <cstdio>

#include "fd_common.cuh"

namespace fd {

// ----------------------------------------------------------------------------------------------
// PTX wrappers
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// Blocking wait with a suspend-time hint: the thread is parked by the hardware (no issue slots burnt) until the phase
// completes or the hint (ns) expires, instead of spinning on short default time-outs, so that waiting warps take few issue slots
// from the warps that compute.
#ifdef FD_TC_WATCHDOG
// Debug build (-DFD_TC_WATCHDOG): every blocking barrier wait gives up after ~50 ms, reports who waited for what and traps, so a
// protocol dead-lock shows up as a launch failure with a message instead of a hung GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    const long long t0 = clock64();
    for (;;) {
        uint32_t ok;
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
        if (ok) return;
        if (clock64() - t0 > 100000000ll) {
            printf("WATCHDOG block %d warp %d lane %d: barrier at smem offset %u parity %u never completed\n", (int)blockIdx.x, (int)(threadIdx.x >> 5),
                   (int)(threadIdx.x & 31), bar, parity);
            __trap();
        }
    }
}
#else
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, %2;\n\t"
        "@p bra WAIT_DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "WAIT_DONE:\n\t}" ::"r"(bar), "r"(parity), "r"(1000000u) : "memory");
}
#endif
// Wait for roles that can afford wake-up latency (the TMA producer waiting for a free stage): a plain timed sleep between
// probes parks the warp whatever the hardware does with the suspend-time hint.
__device__ __forceinline__ void mbar_wait_sleep(uint32_t bar, uint32_t parity, uint32_t ns) {
    if (ns == 0u) { mbar_wait(bar, parity); return; }
    for (;;) {
        uint32_t ok;
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
        if (ok) break;
        __nanosleep(ns);
    }
}
// A plain probe loop with a pause between probes, used by the tile-sharing cluster instance of the block kernel (its waiters
// sit on barriers that are completed from OTHER SMs: bulk-copy bytes, remote arrivals).  The planner admits that mode on
// one-wave launches only (FD_TC_CLUSTER_MULTIWAVE=1 lifts the limit for experiments).
__device__ __forceinline__ void mbar_wait_nohint(uint32_t bar, uint32_t parity) {
#ifdef FD_TC_WATCHDOG
    mbar_wait(bar, parity);          // the watchdog form is a plain probe loop already
#else
    for (;;) {
        uint32_t ok;
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
        if (ok) return;
        __nanosleep(40);
    }
#endif
}
template <bool HINT>
__device__ __forceinline__ void mbar_wait_sel(uint32_t bar, uint32_t parity) {
    if constexpr (HINT) mbar_wait(bar, parity); else mbar_wait_nohint(bar, parity);
}
template <bool HINT>
__device__ __forceinline__ void mbar_wait_sleep_sel(uint32_t bar, uint32_t parity, uint32_t ns) {
    if (ns == 0u) { mbar_wait_sel<HINT>(bar, parity); return; }
    mbar_wait_sleep(bar, parity, ns);
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
// tile load delivered to the same shared-memory offset (and signalled on the barrier at the same offset) in every CTA of `mask`
__device__ __forceinline__ void tma_load_2d_multicast(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, uint16_t mask) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;"
        ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "h"(mask) : "memory");
}
// plain (non-tensor) bulk copy global -> shared, completion on an mbarrier (SASS UBLKCP)
__device__ __forceinline__ void bulk_load(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
// shared -> global tensor stores (bulk async group); OOB parts of the box are clipped by the hardware
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* map, uint32_t src, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                 ::"l"(map), "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
// same, but element-wise ADD into global memory (performed at L2 in the tensor's dtype, round-to-nearest)
__device__ __forceinline__ void tma_reduce_add_4d(const CUtensorMap* map, uint32_t src, int c0, int c1, int c2, int c3) {
    asm volatile("cp.reduce.async.bulk.tensor.4d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                 ::"l"(map), "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read1() { asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}

// ---- Hopper warpgroup MMA (wgmma): D[regs] (+)= A[smem] * B[smem]^T, both operands K-major 128B-swizzled, fp32 accumulate.
// A warpgroup (four consecutive warps, the first one's id a multiple of four) computes a 64-row slice; thread t of it holds rows
// 16 * (t / 32) + (t % 32) / 4 (+ 8) and, per 8-column group j, the columns 8 j + 2 (t % 4) (+ 1):
//   d[4 j + 0], d[4 j + 1] = row r, columns c, c + 1;   d[4 j + 2], d[4 j + 3] = row r + 8, same columns.
// K-major, SWIZZLE_128B shared-memory matrix descriptor: start address >> 4, LBO (unused for swizzled K-major) = 1, SBO = 1024 B
// between 8-row groups, layout type 1 (128B swizzle) in bits 62-63.  The start address advances by 32 B (2 in the low word) per
// K step of 16 elements inside the 128-byte swizzle row.
constexpr uint32_t kSw128DescHi = (1024u >> 4) | (1u << 30);
__device__ __forceinline__ uint32_t sw128_desc_lo(uint32_t saddr) { return ((saddr >> 4) & 0x3FFFu) | (1u << 16); }
__device__ __forceinline__ uint64_t sw128_desc(uint32_t lo) { return ((uint64_t)kSw128DescHi << 32) | lo; }
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait1() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }
#define FD_WGMMA_N64(TY)                                                                                                        \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"                                                          \
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32." TY "." TY " "                                                   \
                 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,"  \
                 "%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}"                                                                  \
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),    \
                   "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),         \
                   "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),        \
                   "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])                      \
                 : "l"(a), "l"(b), "r"(acc))
#define FD_WGMMA_N32(TY)                                                                                                        \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"                                                          \
                 "wgmma.mma_async.sync.aligned.m64n32k16.f32." TY "." TY " "                                                   \
                 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n\t}"                      \
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),    \
                   "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])                       \
                 : "l"(a), "l"(b), "r"(acc))
// m64 x n64 x k16 (or n32), accumulate when acc != 0, else overwrite
template <typename T> __device__ __forceinline__ void wgmma_n64(float (&d)[32], uint64_t a, uint64_t b, uint32_t acc);
template <> __device__ __forceinline__ void wgmma_n64<__half>(float (&d)[32], uint64_t a, uint64_t b, uint32_t acc) { FD_WGMMA_N64("f16"); }
template <> __device__ __forceinline__ void wgmma_n64<__nv_bfloat16>(float (&d)[32], uint64_t a, uint64_t b, uint32_t acc) { FD_WGMMA_N64("bf16"); }
template <typename T> __device__ __forceinline__ void wgmma_n32(float (&d)[16], uint64_t a, uint64_t b, uint32_t acc);
template <> __device__ __forceinline__ void wgmma_n32<__half>(float (&d)[16], uint64_t a, uint64_t b, uint32_t acc) { FD_WGMMA_N32("f16"); }
template <> __device__ __forceinline__ void wgmma_n32<__nv_bfloat16>(float (&d)[16], uint64_t a, uint64_t b, uint32_t acc) { FD_WGMMA_N32("bf16"); }
// m64 x n128 / n256 x k16 in ONE instruction (the dense conv kernel): the A tile is read from shared memory once per
// instruction, so wider instructions need fewer shared-memory bytes per MAC than several n64 ones
#define FD_WGMMA_N128(TY) \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t" \
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32." TY "." TY " " \
                 "{" \
                 "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15," \
                 "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31," \
                 "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47," \
                 "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63" \
                 "}, %64, %65, p, 1, 1, 0, 0;\n\t}" \
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), \
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), \
                   "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), \
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), \
                   "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), \
                   "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), \
                   "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), \
                   "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]) \
                 : "l"(a), "l"(b), "r"(acc))
#define FD_WGMMA_N256(TY) \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t" \
                 "wgmma.mma_async.sync.aligned.m64n256k16.f32." TY "." TY " " \
                 "{" \
                 "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15," \
                 "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31," \
                 "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47," \
                 "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63," \
                 "%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79," \
                 "%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95," \
                 "%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111," \
                 "%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127" \
                 "}, %128, %129, p, 1, 1, 0, 0;\n\t}" \
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), \
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), \
                   "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), \
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), \
                   "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), \
                   "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), \
                   "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), \
                   "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), \
                   "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), \
                   "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), \
                   "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), \
                   "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), \
                   "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), \
                   "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), \
                   "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), \
                   "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127]) \
                 : "l"(a), "l"(b), "r"(acc))
template <typename T> __device__ __forceinline__ void wgmma_n128(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc);
template <> __device__ __forceinline__ void wgmma_n128<__half>(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc) { FD_WGMMA_N128("f16"); }
template <> __device__ __forceinline__ void wgmma_n128<__nv_bfloat16>(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc) { FD_WGMMA_N128("bf16"); }
template <typename T> __device__ __forceinline__ void wgmma_n256(float (&d)[128], uint64_t a, uint64_t b, uint32_t acc);
template <> __device__ __forceinline__ void wgmma_n256<__half>(float (&d)[128], uint64_t a, uint64_t b, uint32_t acc) { FD_WGMMA_N256("f16"); }
template <> __device__ __forceinline__ void wgmma_n256<__nv_bfloat16>(float (&d)[128], uint64_t a, uint64_t b, uint32_t acc) { FD_WGMMA_N256("bf16"); }
// one instruction of width BN (64, 128 or 256 output columns); d holds BN / 2 accumulators per thread
template <typename T, int BN> __device__ __forceinline__ void wgmma_bn(float (&d)[BN / 2], uint64_t a, uint64_t b, uint32_t acc) {
    if constexpr (BN == 64) wgmma_n64<T>(d, a, b, acc);
    else if constexpr (BN == 128) wgmma_n128<T>(d, a, b, acc);
    else wgmma_n256<T>(d, a, b, acc);
}
#undef FD_WGMMA_N64
#undef FD_WGMMA_N32
#undef FD_WGMMA_N128
#undef FD_WGMMA_N256
// ---- TF32 wgmma with A from registers (the split-TF32 pointwise kernel): D[regs] += A[regs] * B[smem]^T, m64 x n(N) x k8.
// A: per warp of the warpgroup a 16 x 8 slice in four registers, the mma.m16n8k8 tf32 layout: a[0] = (row g, column t),
// a[1] = (g + 8, t), a[2] = (g, t + 4), a[3] = (g + 8, t + 4) with g = lane / 4, t = lane % 4.  The tensor core reads only the
// top 19 bits of every 32-bit operand, so the operands are rounded to TF32 (cvt.rna) before they get here.  B as for the 16-bit
// forms: K-major, 128B-swizzled; one k8 step is 32 bytes of the 128-byte row, like one k16 step of 16-bit data.
#define FD_WGMMA_TF32_N64 \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t" \
                 "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 " \
                 "{" \
                 "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15," \
                 "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31" \
                 "}, {%32, %33, %34, %35}, %36, p, 1, 1;\n\t}" \
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), \
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), \
                   "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), \
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]) \
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc))
#define FD_WGMMA_TF32_N128 \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t" \
                 "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 " \
                 "{" \
                 "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15," \
                 "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31," \
                 "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47," \
                 "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63" \
                 "}, {%64, %65, %66, %67}, %68, p, 1, 1;\n\t}" \
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), \
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), \
                   "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), \
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), \
                   "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), \
                   "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), \
                   "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), \
                   "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]) \
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc))
#define FD_WGMMA_TF32_N256 \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %133, 0;\n\t" \
                 "wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 " \
                 "{" \
                 "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15," \
                 "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31," \
                 "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47," \
                 "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63," \
                 "%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79," \
                 "%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95," \
                 "%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111," \
                 "%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127" \
                 "}, {%128, %129, %130, %131}, %132, p, 1, 1;\n\t}" \
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), \
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), \
                   "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), \
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), \
                   "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), \
                   "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), \
                   "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), \
                   "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), \
                   "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), \
                   "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), \
                   "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), \
                   "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), \
                   "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), \
                   "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), \
                   "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), \
                   "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127]) \
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc))
// m64 x n(BN) x k8, TF32 inputs; accumulate when acc != 0, else overwrite
template <int BN> __device__ __forceinline__ void wgmma_tf32_bn(float (&d)[BN / 2], const uint32_t (&a)[4], uint64_t b, uint32_t acc) {
    if constexpr (BN == 64) FD_WGMMA_TF32_N64;
    else if constexpr (BN == 128) FD_WGMMA_TF32_N128;
    else FD_WGMMA_TF32_N256;
}
#undef FD_WGMMA_TF32_N64
#undef FD_WGMMA_TF32_N128
#undef FD_WGMMA_TF32_N256
// fp32 -> TF32, round to nearest with ties away from zero; the low 13 bits of the result are zero
__device__ __forceinline__ uint32_t rna_tf32(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return r;
}

// ---- thread-block clusters: rank, cluster barrier, DSMEM addresses, remote mbarrier arrives ---------------
__device__ __forceinline__ uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t mapa_u32(uint32_t addr, uint32_t rank) {
    uint32_t r; asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank)); return r;
}
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t cluster_addr) {
    asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(cluster_addr) : "memory");
}
// wait on a LOCAL barrier whose arrivals come (also) from the peer CTA: acquire at cluster scope
__device__ __forceinline__ void mbar_wait_cluster(uint32_t bar, uint32_t parity, uint32_t ns) {
    for (;;) {
        uint32_t ok;
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
        if (ok) break;
        if (ns) __nanosleep(ns);
    }
}
__device__ __forceinline__ void st_cluster_v4(uint32_t cluster_addr, uint4 v) {
    asm volatile("st.shared::cluster.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(cluster_addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
// Bulk copy from this CTA's shared memory into a peer CTA's (SM -> SM over the cluster network, async proxy on both ends): the
// completion bytes are posted on an mbarrier in the DESTINATION CTA.  dst / bar are shared::cluster addresses (mapa_u32).
__device__ __forceinline__ void bulk_copy_to_peer(uint32_t dst_cluster, uint32_t src_cta, uint32_t bytes, uint32_t bar_cluster) {
    asm volatile("cp.async.bulk.shared::cluster.shared::cta.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst_cluster), "r"(src_cta), "r"(bytes), "r"(bar_cluster) : "memory");
}
// Packed fp32 pair (channel pair of one lane).  The pair travels as one 64-bit value and is computed as two FMAs; a 16-bit x
// 16-bit product is exact in fp32, so widening first and using the fp32 FMA gives the mixed-precision result bit for bit.
typedef unsigned long long f32x2;
__device__ __forceinline__ f32x2 f32x2_make(float lo, float hi) { return ((f32x2)__float_as_uint(hi) << 32) | (f32x2)__float_as_uint(lo); }
__device__ __forceinline__ float f32x2_lo(f32x2 v) { return __uint_as_float((uint32_t)v); }
__device__ __forceinline__ float f32x2_hi(f32x2 v) { return __uint_as_float((uint32_t)(v >> 32)); }
__device__ __forceinline__ f32x2 ffma2_abc(f32x2 a, f32x2 b, f32x2 c) {
    return f32x2_make(fmaf(f32x2_lo(a), f32x2_lo(b), f32x2_lo(c)), fmaf(f32x2_hi(a), f32x2_hi(b), f32x2_hi(c)));
}
__device__ __forceinline__ void ffma2(f32x2& acc, f32x2 a, f32x2 b) { acc = ffma2_abc(a, b, acc); }
// 16 bytes from shared memory, loaded where the call stands: the compiler neither hoists it nor merges it with an earlier load
// of the same address, so it cannot decide to keep a whole tap table live in registers (and spill) to save the reloads
__device__ __forceinline__ uint4 lds_u4_here(const void* p) {
    uint4 v;
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(smem_u32(p)));
    return v;
}

// mixed-precision FMA: exact 16-bit x 16-bit product added into fp32
template <typename T> struct MixFma;
template <> struct MixFma<__half> {
    __device__ __forceinline__ static f32x2 widen(uint32_t v) {           // two HADD2.F32
        const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&v));
        return f32x2_make(f.x, f.y);
    }
    __device__ __forceinline__ static void fma2(float& lo, float& hi, uint32_t a, uint32_t b) {
        const f32x2 x = widen(a), y = widen(b);
        lo = fmaf(f32x2_lo(x), f32x2_lo(y), lo);
        hi = fmaf(f32x2_hi(x), f32x2_hi(y), hi);
    }
    __device__ __forceinline__ static uint32_t pack(float lo, float hi) {
        __half2 h = __floats2half2_rn(lo, hi);
        return *reinterpret_cast<uint32_t*>(&h);
    }
    __device__ __forceinline__ static float2 unpack(uint32_t v) { return __half22float2(*reinterpret_cast<__half2*>(&v)); }
    // round the fp32 pair to 16 bits with ReLU folded into the conversion (F2FP.RELU), ReLU6's upper clamp on the packed
    // result (HMNMX2): clamping after rounding equals rounding after clamping because 0 and 6 are representable
    template <bool RELU6>
    __device__ __forceinline__ static uint32_t pack_act(f32x2 v) {
        uint32_t h;
        asm("cvt.rn.relu.f16x2.f32 %0, %1, %2;" : "=r"(h) : "f"(f32x2_hi(v)), "f"(f32x2_lo(v)));
        if (RELU6) asm("min.f16x2 %0, %0, %1;" : "+r"(h) : "r"(0x46004600u));
        return h;
    }
};
template <> struct MixFma<__nv_bfloat16> {
    __device__ __forceinline__ static f32x2 widen(uint32_t v) {           // bf16 -> fp32 is a 16-bit shift
        return f32x2_make(__uint_as_float(v << 16), __uint_as_float(v & 0xffff0000u));
    }
    __device__ __forceinline__ static void fma2(float& lo, float& hi, uint32_t a, uint32_t b) {
        const f32x2 x = widen(a), y = widen(b);
        lo = fmaf(f32x2_lo(x), f32x2_lo(y), lo);
        hi = fmaf(f32x2_hi(x), f32x2_hi(y), hi);
    }
    __device__ __forceinline__ static uint32_t pack(float lo, float hi) {
        __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
        return *reinterpret_cast<uint32_t*>(&h);
    }
    __device__ __forceinline__ static float2 unpack(uint32_t v) { return __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&v)); }
    template <bool RELU6>
    __device__ __forceinline__ static uint32_t pack_act(f32x2 v) {
        uint32_t h;
        asm("cvt.rn.relu.bf16x2.f32 %0, %1, %2;" : "=r"(h) : "f"(f32x2_hi(v)), "f"(f32x2_lo(v)));
        if (RELU6) asm("min.bf16x2 %0, %0, %1;" : "+r"(h) : "r"(0x40C040C0u));
        return h;
    }
};

// programmatic dependent launch: let the next kernel of the stream start its prologue on SMs this grid has already left,
// and make this kernel's first global access wait for the previous grid's memory to be visible
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait_prior_grid() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// stage index + phase parity of an mbarrier ring, advanced without div/mod
struct Ring {
    uint32_t s = 0, ph = 0;
    __device__ __forceinline__ void next(uint32_t n) { if (++s == n) { s = 0; ph ^= 1u; } }
};
// exact w / d for w, d < 2^20 with mg = floor(2^40 / d) + 1
__device__ __forceinline__ uint32_t fdiv40(uint32_t w, unsigned long long mg) { return (uint32_t)(((unsigned long long)w * mg) >> 40); }

// scalar BN affine + activation (head path only; the block paths do channel PAIRS: ffma2_abc + MixFma::pack_act)
template <bool RELU6>
__device__ __forceinline__ float affine_act(float acc, float s, float b) {
    const float v = fmaxf(fmaf(acc, s, b), 0.0f);
    return RELU6 ? fminf(v, 6.0f) : v;
}


typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
PFN_encodeTiled get_tensor_map_encoder();       // cuTensorMapEncodeTiled through cudaGetDriverEntryPoint (no libcuda link)

}  // namespace fd
