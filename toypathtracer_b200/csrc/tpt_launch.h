// Internal interface between the C-ABI (tpt_api.cu) and the two kernel translation units.
#pragma once
#include <cuda_runtime.h>
#include "tpt_types.h"

namespace tpt {

struct SceneDev
{
    const unsigned char* blob;   // device copy of the packed scene (tpt_scene_pack.h)
    SceneBlobLayout layout;
    int count, nLights;
    uint32_t stagedBytes;        // prefix of the blob every CTA stages into shared memory via TMA
    int kformMode;               // fast kernels: 2 = expanded form on the pair array where it fits (kernel parameter up to
                                 // kParamPairSpheres, else shared memory; form 5 where halfOk), 3 = the same always in
                                 // shared memory (A/B), 4 = as 2 but form 4 never runs form 5's pass 1 (A/B), 1 = expanded form, scalar
    bool kformOk;                // every sphere satisfies |c|^2 <= 128 + 2 r^2: the expanded-form sweep of the fast kernels
                                 // then rounds no worse than the reference form (see FastHitterK)
    ParamPairs pairs;            // pass-1 operands of sweep forms 4 and 5 (all zero for scenes of more than kParamPairSpheres)
    bool halfOk;                 // pairs.h holds form 5's half-precision pass 1 (build_half_pairs)
};

// lanes: 0 = choose from the number of (frame,row) chains; 1, 2, 8, 9, 32 or 64..71 to force (see tpt_exact.cu).
// resolve = false: with numFrames > 1 only the per-frame colours are written to p.scratch (no blend into the image)
cudaError_t launch_exact(const DrawParams& p, const SceneDev& sc, int lanes, int numSMs, cudaStream_t stream, bool resolve = true);
// the reference's progressive blend (Test.cpp:272-276,293-295) of p.numFrames frames of per-frame colours in p.scratch
cudaError_t launch_resolve_exact(const DrawParams& p, cudaStream_t stream);
cudaError_t launch_debug_libm(int fn, const float* dIn, float* dOut, long long n, cudaStream_t stream);
// sweep form variants 3/4 run for this scene (0 reference, 1 expanded, 2 packed pairs, 3 conservative packed)
int fast_queue_kform(const SceneDev& sc);
// nearest hit of n rays {o.xyz, d.xyz} with one sweep form of the fast kernels (0 reference, 1 expanded, 2 packed pairs, 3 conservative,
// 4 packed pairs in the kernel parameter, 5 form 4 with the half-precision pass 1)
cudaError_t launch_debug_hit(const SceneDev& sc, int kform, const float* dRays, int* dId, float* dT, long long n, int numSMs, cudaStream_t stream);
constexpr int kMaxFramesPerDraw = 256;  // frames per fast launch: per-frame blend weights live in shared memory

// What a host-buffer draw needs to know about a fast variant.
struct FastVariantInfo
{
    bool writesFinalPixels;   // the trace kernel stores finished pixels itself (no L2 reductions), also into mapped host memory
    bool rowBands;            // a draw can be split into row bands, one launch per band
    bool progressCounters;    // the trace kernel can publish per-band completion counters (launch_fast's bandDone)
    bool referenceQueue;      // runs the slab queue's reference-form instances, which alone sample the environment
                              // ("environment_sampling") and look up textures (tpt_set_textures)
};
FastVariantInfo fast_variant_info(int variant);
// The variant a draw with "fast_variant" -1 runs over regionPix pixels of numFrames frames at spp; zeroCopy: the draw
// stores straight into mapped host memory.
int fast_auto_variant(const SceneDev& sc, long long regionPix, int spp, int numFrames, bool zeroCopy);
// variant: see tpt_fast.cu
// bandDone (optional, variants with progressCounters only): device counters [numBands]; the kernel publishes finished
// paths per band of macro-tiles, bandExpected[b] receives the final count of band b (host array) and
// kSlabPix*ceil(mtiles/numBands) pixels form a band.
cudaError_t launch_fast(const DrawParams& p, const SceneDev& sc, int variant, int numSMs, cudaStream_t stream,
                        unsigned int* bandDone = nullptr, int numBands = 0, unsigned int* bandExpected = nullptr);
// tpt_trace_rays: fast-mode radiance of p.numRays (>= 1) caller rays p.rays, p.spp samples each with streams
// pixel_seed(ray * spp + sample, p.frame0), mean written to the float4 p.image[ray] (zeroed first); p.numFrames = 1, p.flags = 0.
// Runs the slab-queue instance variant 3 would run for the scene. tpt_trace_irradiance: the same launch with p.pointStart
// set, p.rays holding surface points {p, n} and p.pointIds their sphere ids (or null); the mean is then scaled by pi.
// tpt_trace_samples: the same launch with p.sums set, adding (v, 1) and, with p.sq4, (v^2, 0) per sample to the
// caller's sums (not zeroed), v being the path's radiance (x pi for points); with the list p.entries of p.numRays indices
// into the numIn inputs, whose check lands in *badPixel (device) as for launch_fast_samples before anything is traced.
cudaError_t launch_fast_rays(const DrawParams& p, const SceneDev& sc, long long numIn, unsigned long long* badPixel, int numSMs,
                             cudaStream_t stream);
// tpt_draw_samples: p.spp samples of each of the p.numRays (>= 1) entries of the pixel list p.pixels (null: pixels 0 ..
// numRays - 1 of the width x height image), sample s of pixel i being the fast draw's camera ray with stream
// pixel_seed(i * spp + s, p.frame0). Adds (sum of col, spp) to the float4 p.image[entry] and, when p.sq4 is not null,
// (sum of col^2, 0) to p.sq4[entry]; p.numFrames = 1, p.flags = 0. A list is checked first: the smallest
// (entry << 32 | index) of an index outside the image lands in *badPixel (device; ~0 when there is none) and then nothing
// is traced. Runs the slab-queue instance variant 3 would run for the scene.
cudaError_t launch_fast_samples(const DrawParams& p, const SceneDev& sc, unsigned long long* badPixel, int numSMs,
                                cudaStream_t stream);
// The check of n int32 `list` against [0, limit) that the caller lists get before their trace kernel: the smallest
// (entry << 32 | value) of an entry outside lands in *bad (device; ~0 when there is none). tpt_set_environment and
// tpt_set_textures check device texels' channels with it, as their bits.
cudaError_t launch_list_check(const int* list, long long n, long long limit, unsigned long long* bad, int numSMs,
                              cudaStream_t stream);
// tpt_draw_aovs (rays = false: the region of p, frames [p.frame0, p.frame0 + p.numFrames) at p.spp, blended over the outputs
// with the weight of `prev`) and tpt_trace_aovs (rays = true: p.numRays >= 1 caller rays p.rays): first-hit albedo4,
// normal4 and ids (each may be null) with the slab queue's sweep form, one ray counted per traced sample.
cudaError_t launch_fast_aovs(const DrawParams& p, const SceneDev& sc, bool rays, float* albedo4, float* normal4, int* ids,
                             int numSMs, cudaStream_t stream);
// TPT_MODE_REFGPU (tpt_refgpu.cuh): strict arithmetic (tpt_exact.cu) / GPU-native arithmetic (tpt_fast.cu)
cudaError_t launch_refgpu_exact(const DrawParams& p, const SceneDev& sc, int numSMs, cudaStream_t stream);
cudaError_t launch_refgpu_fast(const DrawParams& p, const SceneDev& sc, int numSMs, cudaStream_t stream);
int fast_slab_pixels();
// weight of `prev` when frames [frame0, frame0 + numFrames) are blended into it: the product of their lerp_fac
float prev_weight(int frame0, int numFrames, unsigned flags);

// The kernels the calling thread's current library call launched; start_kernels clears the record. `launches` counts every
// launch (tpt_last_launch_count): trace kernels, and through note_launch the helpers that clear, blend or count.
// Diagnostic (tpt_debug_last_kernels): the trace kernels, as the function pointers launch_trace passed to note_kernel
// (a launch only stores a pointer); n counts them, the first kCap are kept (the count is reported, so a cut-off list shows).
struct KernelRecord
{
    static constexpr int kCap = 16;
    const void* fn[kCap];
    int n;
    int launches;
};
extern thread_local KernelRecord t_lastKernels;
inline void clear_kernels() { t_lastKernels.n = 0; t_lastKernels.launches = 0; }
inline void note_launch() { ++t_lastKernels.launches; }
inline void note_kernel(const void* fn)
{
    if (t_lastKernels.n < KernelRecord::kCap) t_lastKernels.fn[t_lastKernels.n] = fn;
    ++t_lastKernels.n;
    note_launch();
}
// Records a trace kernel (note_kernel) and launches it, so that the record and the launch cannot drift apart. The
// diagnostic kernels (k_debug_hit, k_debug_libm) are launched directly and stay out of the record.
template <class Kernel, class... Args>
cudaError_t launch_trace(Kernel kern, dim3 grid, dim3 block, size_t dyn, cudaStream_t stream, const Args&... args)
{
    note_kernel((const void*)kern);
    kern<<<grid, block, dyn, stream>>>(args...);
    return cudaGetLastError();
}

// Launch set-up of a persistent kernel: allows `dyn` bytes of dynamic shared memory, sizes the grid to the CTAs that stay
// resident on numSMs SMs (at least one per SM) but no more than `ctasNeeded`, and zeroes the work counter.
template <class Kernel>
cudaError_t persistent_grid(Kernel kern, int threads, size_t dyn, int numSMs, long long ctasNeeded, const DrawParams& p,
                            cudaStream_t stream, long long& grid)
{
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn);
    if (e != cudaSuccess) return e;
    int perSM = 0;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSM, kern, threads, dyn);
    if (e != cudaSuccess) return e;
    grid = (long long)numSMs * (perSM < 1 ? 1 : perSM);
    if (grid > ctasNeeded) grid = ctasNeeded;
    return cudaMemsetAsync(p.workCounter, 0, sizeof(unsigned int), stream);
}

} // namespace tpt
