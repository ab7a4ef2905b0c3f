// Device-only helpers: TMA bulk staging of the scene blob into shared memory (cp.async.bulk + mbarrier,
// SASS: UBLKCP / SYNCS), 128-bit cache-hinted global accesses, warp helpers.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "tpt_types.h"
#include "tpt_scene_pack.h"

namespace tpt {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init()
{
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity)
{
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE;\n"
        "bra WAIT_LOOP;\n"
        "DONE:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// Producer/consumer waits of warps that share an SM with working warps: try_wait with a suspend-time hint, and a
// nanosleep between attempts, so that a waiting warp issues a handful of instructions per microsecond instead of spinning
// (measured in the split exact kernel: the plain try_wait loop was 23 % of all issued instructions).
// CLUSTER: the barrier is arrived at from another CTA of the cluster, so the wait acquires at cluster scope.
template <bool CLUSTER = false>
__device__ __forceinline__ void mbar_wait_sleep(uint64_t* bar, uint32_t parity)
{
#define TPT_WAIT_SLEEP(TRY_WAIT)                                                                                              \
    asm volatile(                                                                                                             \
        "{\n"                                                                                                                 \
        ".reg .pred p;\n" TRY_WAIT " p, [%0], %1, %2;\n"                                                                      \
        "@p bra DONE_S;\n"                                                                                                    \
        "WAIT_LOOP_S:\n"                                                                                                      \
        "nanosleep.u32 128;\n" /* 32 .. 1024 ns measured: no difference in frame time */                                     \
        TRY_WAIT " p, [%0], %1, %2;\n"                                                                                        \
        "@!p bra WAIT_LOOP_S;\n"                                                                                              \
        "DONE_S:\n"                                                                                                           \
        "}\n" ::"r"(smem_u32(bar)), "r"(parity), "r"(100000u) : "memory")
    if constexpr (CLUSTER) TPT_WAIT_SLEEP("mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64");
    else TPT_WAIT_SLEEP("mbarrier.try_wait.parity.shared::cta.b64");
#undef TPT_WAIT_SLEEP
}
// 1-D bulk copy global -> shared through the TMA unit; bytes % 16 == 0, both addresses 16 B aligned.
__device__ __forceinline__ void tma_bulk_g2s(void* dstSmem, const void* srcGlobal, uint32_t bytes, uint64_t* bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dstSmem)),
                 "l"(srcGlobal), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// Stages `bytes` of the scene blob into shared memory with TMA bulk copies issued by one thread; every
// thread of the CTA returns only after the data has landed. `bar` must live in shared memory.
__device__ __forceinline__ void stage_blob(unsigned char* dst, const unsigned char* src, uint32_t bytes, uint64_t* bar)
{
    if (threadIdx.x == 0)
    {
        mbar_init(bar, 1);
        mbar_fence_init();
    }
    __syncthreads();
    if (threadIdx.x == 0)
    {
        mbar_expect_tx(bar, bytes);
        const uint32_t kChunk = 32768;
        for (uint32_t off = 0; off < bytes; off += kChunk)
        {
            uint32_t n = bytes - off < kChunk ? bytes - off : kChunk;
            tma_bulk_g2s(dst + off, src + off, n, bar);
        }
    }
    mbar_wait(bar, 0);
}

// Scene view: sections inside the staged prefix point to shared memory, the rest to global memory.
// ALL_STAGED: the caller guarantees stagedBytes == L.totalBytes; every pointer is then derived from the shared-memory base
// alone, which lets the compiler prove the address space (LDS instead of generic LD with 64-bit address arithmetic).
template <bool ALL_STAGED = false>
__device__ __forceinline__ SceneView make_view(const unsigned char* smemBase, const unsigned char* globalBase,
                                               const SceneBlobLayout& L, uint32_t stagedBytes, int count, int nLights)
{
    SceneView v;
    auto pick = [&](uint32_t off) -> const unsigned char* { return (ALL_STAGED || off < stagedBytes) ? smemBase + off : globalBase + off; };
    v.sph = (const Q4*)pick(L.offSph);
    v.invRadius = (const float*)pick(L.offInvRadius);
    v.lights = (const LightRec*)pick(L.offLights);
    v.matA = (const Q4*)pick(L.offMatA);
    v.matB = (const Q4*)pick(L.offMatB);
    v.matRi = (const float*)pick(L.offMatRi);
    v.media = (const Q4*)pick(media_offset(L.offMatRi, count));
    v.fog = (const Q4*)pick(fog_offset(L.offMatRi, count, L.flags));
    v.count = count;
    v.simdCount = (count + 3) / 4 * 4;
    v.nLights = nLights;
    v.flags = L.flags;
    v.maxDepth = scene_max_depth(L.flags);
    v.sphShared = smem_u32(smemBase + L.offSph);   // geometry is always inside the staged prefix
    v.envLo = L.envLo;
    v.envHi = L.envHi;
    v.envW = L.envW;
    v.envH = L.envH;
    v.tex = L.tex;
    v.emit = L.emit;
    return v;
}

// Adds the warp's ray counts to *counter with one atomic per warp; all 32 lanes must call it.
__device__ __forceinline__ void flush_ray_count(unsigned long long* counter, unsigned rc, int lane)
{
    for (int off = 16; off > 0; off >>= 1) rc += __shfl_xor_sync(0xffffffffu, rc, off);
    if (lane == 0 && rc) atomicAdd(counter, (unsigned long long)rc);
}

__device__ __forceinline__ float4 ld_stream_f4(const float* p)
{
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ void st_stream_f4(float* p, float4 v)
{
    asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

} // namespace tpt
