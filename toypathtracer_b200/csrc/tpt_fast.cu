// Fast (throughput) mode kernels: same estimator as the reference's Trace/Scatter (Cpp/Source/Test.cpp:83-234),
// one independent XorShift32 stream per (pixel, frame) instead of the reference's per-row stream, FMA
// contraction and fast intrinsics allowed. Results agree with the reference statistically (same expectation,
// same rays/sample), not bitwise — bitwise parity is the exact mode's job (tpt_exact.cu).
//
// The estimator is written once, as path_step (one step of a per-lane path state machine on a QPath): every variant and
// entry point shades with it; the block wavefront (variants 6/7) runs its last part, lambert_next, in a phase of its own.
// The variants differ in how they deal work and write pixels:
// variant 0  "megakernel": one thread per pixel, loops over frames x spp with one stream per pixel and frame (what
//            the reference's own GPU shaders do, Cpp/Windows/ComputeShader.hlsl:353-395). Baseline for the
//            persistent design.
// variant 1  "persistent wavefront" (variant 2: the same kernel at 3 instead of 2 CTAs per SM): one CTA per SM
//            slot, resident for the whole draw. The CTA pulls tiles of
//            kTilePix pixels from a global counter; inside a tile every lane runs a path and refills itself with the
//            next (pixel, sample) from a warp-aggregated shared counter as soon as its path ends (ray regeneration),
//            so the ray-vs-all-spheres sweep — 85 % of the instructions — always runs with full warps. Radiance is
//            accumulated per pixel in shared memory; finished tiles are written with coalesced 128-bit stores (and
//            128-bit loads of `prev` when accumulating).
// variants 3-9: see their sections below.
#include <climits>
#include <cstdio>
#include <cstdlib>
#include <type_traits>
#include <vector>
#include <cuda_fp16.h>
#include "tpt_integrator.cuh"
#include "tpt_device_utils.cuh"
#include "tpt_launch.h"
#include "tpt_fastdiv.h"

namespace tpt {

constexpr int kFastThreads = 256;
constexpr int kTilePix = 1024;          // pixels per tile (12 KB of float3 accumulators)

__device__ __forceinline__ uint32_t fmix32(uint32_t h)
{
    h ^= h >> 16; h *= 0x85ebca6bu; h ^= h >> 13; h *= 0xc2b2ae35u; h ^= h >> 16;
    return h;
}
__device__ __forceinline__ uint32_t pixel_seed(uint32_t pixelIndex, uint32_t frame)
{
    return fmix32(pixelIndex * 0x9E3779B9u + fmix32(frame + 0x7F4A7C15u)) | 1u;
}

// Per-frame weights of the progressive blend (Test.cpp:272-276,293-295) when `numFrames` frames are fused in
// one launch: image = prev*wPrev + sum_f mean_f * w[f], w[f] = (1-lerp_f) * prod_{g>f} lerp_g.
// Fast mode draws its lens and roughness samples analytically instead of by rejection (Maths.cpp:20-37): the same
// distributions (uniform on the unit disk / in the unit ball) from a fixed number of draws, so no lane of a warp waits in
// a rejection loop for its neighbours (ncu: the two loops were 23 + ~25 warp instructions per path step at 18 / 3.5 active
// lanes). The reference's own GPU ports sample analytically as well (ComputeShader.hlsl:18-35). TPT_FAST_ANALYTIC=0
// restores the rejection loops for A/B runs.
#ifndef TPT_FAST_ANALYTIC
#define TPT_FAST_ANALYTIC 1
#endif
__device__ __forceinline__ int opaque_int(int x) { asm volatile("" : "+r"(x)); return x; }
__device__ __forceinline__ V3 fast_in_unit_disk(uint32_t& state)
{
#if TPT_FAST_ANALYTIC
    const float r = M<false>::sqrt_(RandomFloat01(state));
    float sa, ca;
    __sincosf(2.0f * TPT_PI * RandomFloat01(state), &sa, &ca);
    return v3(r * ca, r * sa, 0.0f);
#else
    return RandomInUnitDisk(state);
#endif
}
__device__ __forceinline__ V3 fast_in_unit_sphere(uint32_t& state)
{
#if TPT_FAST_ANALYTIC
    const float z = 1.0f - 2.0f * RandomFloat01(state);
    float sa, ca;
    __sincosf(2.0f * TPT_PI * RandomFloat01(state), &sa, &ca);
    const float rad = __powf(RandomFloat01(state), 1.0f / 3.0f);                 // radius = u^(1/3) as ex2(lg2(u)/3); u = 0 -> 0
    const float r = M<false>::sqrt_(fmaxf(1.0f - z * z, 0.0f)) * rad;
    return v3(r * ca, r * sa, z * rad);
#else
    return RandomInUnitSphere(state);
#endif
}
// Maths.h:437-442 with the analytic lens sample
__device__ __forceinline__ Ray fast_get_ray(const Camera88& c, float s, float t, uint32_t& state)
{
    V3 rd = c.lensRadius * fast_in_unit_disk(state);
    V3 offset = ld3(c.uu) * rd.x + ld3(c.vv) * rd.y;
    Ray r;
    r.orig = ld3(c.origin) + offset;
    r.dir = M<false>::normalize(ld3(c.lowerLeftCorner) + s * ld3(c.horizontal) + t * ld3(c.vertical) - ld3(c.origin) - offset);
    return r;
}
// The camera ray of one fast-mode sample of pixel (x, y), drawn from the sample's stream: the pixel jitter, then the lens
// sample (Test.cpp:286-288 + Maths.h:437-442). The image kernels and the AOV pass build their primary rays with it.
__device__ __forceinline__ Ray fast_camera_ray(const DrawParams& p, int x, int y, uint32_t& rng)
{
    float u = ((float)x + RandomFloat01(rng)) * p.invWidth;
    float v = ((float)y + RandomFloat01(rng)) * p.invHeight;
    return fast_get_ray(p.cam, u, v, rng);
}

__device__ __forceinline__ void blend_weights(const DrawParams& p, float* w, float& wPrev)
{
    float suffix = 1.0f;
    for (int fi = p.numFrames - 1; fi >= 0; --fi)
    {
        float lf = lerp_fac(p.frame0 + fi, p.flags);
        w[fi] = (1.0f - lf) * suffix;
        suffix *= lf;
    }
    wPrev = suffix;
}

// prev*wPrev + acc for one pixel (Test.cpp:293-295 with the frames of this draw folded into acc). A zero weight must
// not read `prev` as a number (NaN * 0), but the pixel's alpha is still the buffer's: the reference never writes it
// (Maths.h:38).
__device__ __forceinline__ float4 blend_prev(const DrawParams& p, const float* px, float wPrev, float ax, float ay, float az)
{
    if (wPrev != 0.0f)
    {
        float4 prev = ld_stream_f4(px);
        prev.x = prev.x * wPrev + ax; prev.y = prev.y * wPrev + ay; prev.z = prev.z * wPrev + az;
        return prev;
    }
    return make_float4(ax, ay, az, p.zeroAlpha ? 0.0f : __ldg(px + 3));
}

// Pixel (x, row ri) of the draw's region: image row y = row0 + ri * rowStep, and the pixel's float4 offset in the caller's
// buffer (row ri of a packed band, row y otherwise).
struct RegionPixel { int x, y; size_t off; };
__device__ __forceinline__ RegionPixel region_pixel(const DrawParams& p, int ri, int x)
{
    const int y = p.row0 + ri * p.rowStep;
    return {x, y, (size_t)(p.packed ? ri : y) * p.width + x};
}
// Pixel i of the region, counted row-major over its numRows rows; the division is done in i's type.
template <class I>
__device__ __forceinline__ RegionPixel region_pixel(const DrawParams& p, I i)
{
    const int ri = (int)(i / (I)p.width);
    return region_pixel(p, ri, (int)(i - (I)ri * (I)p.width));
}

// A finished tile of region pixels [pix0, pix0 + tilePix) whose radiance sits in acc[3 i ..]: prev * wPrev + acc with one
// coalesced 128-bit store per pixel (a 128-bit load of prev when it has weight), the accumulators zeroed for the next
// tile. The CTA's `stride` threads share the loop.
template <class I, class N>
__device__ __forceinline__ void write_tile(const DrawParams& p, float* acc, I pix0, N tilePix, float wPrev, N stride)
{
    for (N i = threadIdx.x; i < tilePix; i += stride)
    {
        float* px = p.image + region_pixel(p, pix0 + (I)i).off * 4;
        st_stream_f4(px, blend_prev(p, px, wPrev, acc[i * 3 + 0], acc[i * 3 + 1], acc[i * 3 + 2]));
        acc[i * 3 + 0] = 0.0f; acc[i * 3 + 1] = 0.0f; acc[i * 3 + 2] = 0.0f;
    }
}

// ---- variant 3 ------------------------------------------------------------------------------------------------
// "persistent queue": no tiles, no block barriers after the prologue. Every WARP pulls slabs of kSlabPix pixels x
// one sample index from a global counter (one atomic per 128 paths), deals the slab's paths to its idle lanes
// (ray regeneration, no atomics inside the warp: the slab cursor is warp-uniform), and every finished path adds
// its weighted radiance to the float4 accumulation buffer with ONE 128-bit vector reduction
// (red.global.add.v4.f32, SASS REDG.E.ADD.F32x4) that resolves in L2. A tiny prepare kernel first scales the
// buffer by the weight of `prev` (or zeroes it). End-of-kernel tail = one slab per warp instead of one 1024-pixel
// tile per CTA, which matters at 1280x720x4spp where a warp's share of the whole frame is only ~1000 paths.
#ifndef TPT_SLAB_PIX
#define TPT_SLAB_PIX 64
#endif
constexpr int kSlabPix = TPT_SLAB_PIX;     // paths per slab (pixels x one sample index)
#ifndef TPT_QUEUE_THREADS
#define TPT_QUEUE_THREADS 128
#define TPT_QUEUE_MINB 6
#endif
#ifndef TPT_BIG_THREADS
#define TPT_BIG_THREADS 768      // one CTA per SM for scenes that fill the shared memory (A/B: 1024 = 32 warps at 64 registers)
#endif
#ifndef TPT_P1_GROUP
#define TPT_P1_GROUP 16
#endif
constexpr int kQueueThreads = TPT_QUEUE_THREADS;

__global__ void k_prepare_image(DrawParams p, float wPrev)
{
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long n = (long long)p.numRows * p.width;
    if (idx >= n) return;
    float* px = p.image + region_pixel(p, idx).off * 4;
    float4 v = blend_prev(p, px, wPrev, 0.0f, 0.0f, 0.0f);
    *reinterpret_cast<float4*>(px) = v;   // stays in L2 for the reductions that follow
}

__device__ __forceinline__ void red_add_f4(float* addr, float x, float y, float z, float w = 0.0f)
{
    asm volatile("red.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(addr), "f"(x), "f"(y), "f"(z), "f"(w) : "memory");
}

// Camera rays of one slab (<= kSlabPix consecutive pixels of the region, one sample index), generated by the whole warp
// in one convergent burst (Test.cpp:286-288 + Maths.h:437-442) into the warp's shared buffer:
// {origin.xyz, rng state} {direction.xyz, tag}; tag = image float4 offset (tileBase < 0) or tileBase + q.
__device__ __forceinline__ void generate_slab_rays(const DrawParams& p, float4 (*rays)[2], int lane, uint32_t count,
                                                   int x0, int ri0, uint32_t sample, uint32_t frame, int tileBase)
{
    for (uint32_t q = (uint32_t)lane; q < count; q += 32)
    {
        int x = x0 + (int)q, ri = ri0;
        while (x >= p.width) { x -= p.width; ++ri; }
        const RegionPixel pix = region_pixel(p, ri, x);
        uint32_t rng = pixel_seed((uint32_t)(pix.y * p.width + x) * (uint32_t)p.spp + sample, frame);
        Ray r = fast_camera_ray(p, x, pix.y, rng);
        const uint32_t tag = tileBase < 0 ? (uint32_t)pix.off : (uint32_t)tileBase + q;
        rays[q][0] = make_float4(r.orig.x, r.orig.y, r.orig.z, __uint_as_float(rng));
        rays[q][1] = make_float4(r.dir.x, r.dir.y, r.dir.z, __uint_as_float(tag));
    }
}

// Caller rays of one slab (tpt_trace_rays): rays [r0, r0 + count) of p.rays, count <= kSlabPix. The warp reads their
// 6 * count floats as rows of 32 consecutive floats (coalesced at any 4-byte alignment of p.rays) into its shared buffer, each
// lane then takes rays `lane` and `lane + 32` from there, normalises the direction and seeds the stream with
// pixel_seed(ray * spp + sample, frame). A ray with a non-finite component, or whose direction does not normalise to a finite
// non-zero vector (zero length, or a squared length that underflows or overflows), is dropped: the survivors are written
// compacted, in ray order, as {origin.xyz, rng state} {direction.xyz, ray index}. Returns their number.
// With a list (p.entries, tpt_trace_samples) [r0, r0 + count) are list entries: each lane reads its two indices (32
// consecutive ints per row) and gathers those inputs' 6 floats; the stream is the input's, pixel_seed(input * spp + sample,
// frame), and the tag the entry. The indices were checked against the inputs before the launch (k_check_pixels).
__device__ __forceinline__ uint32_t load_slab_rays(const DrawParams& p, float4 (*rays)[2], int lane, uint32_t count,
                                                   uint32_t r0, uint32_t sample, uint32_t frame)
{
    float v[2][6];
    uint32_t in[2];
    if (p.entries)
    {
#pragma unroll
        for (int h = 0; h < 2; ++h)
        {
            const uint32_t q = (uint32_t)lane + 32u * h;
            in[h] = q < count ? (uint32_t)__ldg(p.entries + r0 + q) : 0u;
#pragma unroll
            for (int j = 0; j < 6; ++j) v[h][j] = q < count ? __ldg(p.rays + (size_t)in[h] * 6 + j) : 0.0f;
        }
    }
    else
    {
        float* raw = reinterpret_cast<float*>(rays);
        const float* src = p.rays + (size_t)r0 * 6;
#pragma unroll
        for (uint32_t k = 0; k < 6 * kSlabPix; k += 32)
            if (k + lane < 6 * count) raw[k + lane] = __ldg(src + k + lane);
        __syncwarp();
#pragma unroll
        for (int h = 0; h < 2; ++h)
        {
            in[h] = r0 + (uint32_t)lane + 32u * h;
#pragma unroll
            for (int j = 0; j < 6; ++j) v[h][j] = (uint32_t)(lane + 32 * h) < count ? raw[(lane + 32 * h) * 6 + j] : 0.0f;
        }
        __syncwarp();
    }
    uint32_t base = 0;
    const unsigned ltMask = (1u << lane) - 1u;
#pragma unroll
    for (int h = 0; h < 2; ++h)
    {
        const uint32_t q = (uint32_t)lane + 32u * h;
        const V3 o = v3(v[h][0], v[h][1], v[h][2]);
        const V3 d = M<false>::normalize(v3(v[h][3], v[h][4], v[h][5]));
        const bool ok = q < count && isfinite(o.x) && isfinite(o.y) && isfinite(o.z) && isfinite(d.x) && isfinite(d.y) &&
                        isfinite(d.z) && (d.x != 0.0f || d.y != 0.0f || d.z != 0.0f);
        const unsigned m = __ballot_sync(0xffffffffu, ok);
        if (ok)
        {
            const uint32_t slot = base + (uint32_t)__popc(m & ltMask);
            const uint32_t rng = pixel_seed(in[h] * (uint32_t)p.spp + sample, frame);
            rays[slot][0] = make_float4(o.x, o.y, o.z, __uint_as_float(rng));
            rays[slot][1] = make_float4(d.x, d.y, d.z, __uint_as_float(r0 + q));
        }
        base += (uint32_t)__popc(m);
    }
    return base;
}

// Camera rays of one slab of a pixel list (tpt_draw_samples): entries [e0, e0 + count) of p.pixels, count <= kSlabPix, or
// the pixels e0, e0 + 1, ... when p.pixels is null. Each pass of the warp reads 32 consecutive indices (one coalesced
// 128-byte row, two for a full slab) and builds each entry's ray exactly as generate_slab_rays builds the draw's ray for
// that pixel and sample: stream pixel_seed(pixel * spp + sample, frame), then fast_camera_ray. Tag = the entry index. The
// indices were checked against the image before the launch (k_check_pixels). (Loading both rows before generating the
// rays kept two more values live and made the 64-register instance spill 68 B instead of 8.)
__device__ __forceinline__ void generate_list_rays(const DrawParams& p, float4 (*rays)[2], int lane, uint32_t count,
                                                   uint32_t e0, uint32_t sample, uint32_t frame)
{
    for (uint32_t q = (uint32_t)lane; q < count; q += 32)
    {
        const uint32_t pix = p.pixels ? (uint32_t)__ldg(p.pixels + e0 + q) : e0 + q;
        const int y = (int)(pix / (uint32_t)p.width);
        const int x = (int)(pix - (uint32_t)y * (uint32_t)p.width);
        uint32_t rng = pixel_seed(pix * (uint32_t)p.spp + sample, frame);
        Ray r = fast_camera_ray(p, x, y, rng);
        rays[q][0] = make_float4(r.orig.x, r.orig.y, r.orig.z, __uint_as_float(rng));
        rays[q][1] = make_float4(r.dir.x, r.dir.y, r.dir.z, __uint_as_float(e0 + q));
    }
}

struct QPath
{
    V3 o, d;
    V3 thr, col;
    V3 nextDir;
    V3 thrAlb;
    V3 nl;
    float pend;       // m * omega / pi of the shadow ray in flight: it adds thrAlb * E_light * pend when it hits its light
    uint32_t rng;
    uint32_t pixOff;  // float4 index of the pixel in the image buffer
    float weight;
    int kind;
    int depth;
    int mid;
    bool doMaterialE;
    bool active;
};

// A new path along camera ray r, its stream continuing from rng. The caller sets pixOff and weight.
__device__ __forceinline__ void begin_path(QPath& st, const Ray& r, uint32_t rng)
{
    st.o = r.orig; st.d = r.dir;
    st.rng = rng;
    st.thr = v3(1, 1, 1); st.col = v3(0, 0, 0);
    st.kind = 0; st.depth = 0; st.doMaterialE = true; st.active = true;
}
// A new path from a ray-buffer entry {origin.xyz, rng state} {direction.xyz, tag}. The caller decodes the tag into
// pixOff and weight.
__device__ __forceinline__ void begin_path(QPath& st, float4 e0, float4 e1)
{
    begin_path(st, Ray{v3(e0.x, e0.y, e0.z), v3(e1.x, e1.y, e1.z)}, __float_as_uint(e0.w));
}

// Ray regeneration of the warp-dealt kernels (slab, tile and group queues): the idle lanes take entries [cur, end) of
// the warp's ray buffer in lane-rank order, the cursor being warp-uniform. When the buffer is used up, refill(p) fetches
// the next batch and returns kDealRefilled (cur and end reset, the buffer written between two __syncwarp), kDealBlocked
// (nothing can be fetched this round; the warp traces what it has) or kDealExhausted (the work counter ran out: set
// `exhausted`, no more fetches). start(tag) decodes an entry's tag for the lane that took it.
// (p is handed to refill rather than captured: a lambda holding the address of the body's by-value DrawParams made
// the compiler load every field into registers at kernel entry, +1 register and up to 8 B of spills.)
enum DealResult { kDealRefilled, kDealBlocked, kDealExhausted };
template <class Refill, class Start>
__device__ __forceinline__ void deal_paths(const DrawParams& p, QPath& st, const float4 (*rays)[2], uint32_t& cur, uint32_t& end,
                                           bool& exhausted, int lane, Refill&& refill, Start&& start)
{
    const unsigned ltMask = (1u << lane) - 1u;
    unsigned need = __ballot_sync(0xffffffffu, !st.active);
    while (need && !exhausted)
    {
        if (cur >= end)
        {
            const DealResult r = refill(p);
            if (r == kDealExhausted) { exhausted = true; break; }
            if (r == kDealBlocked) break;
        }
        const uint32_t avail = end - cur;
        const uint32_t rank = (uint32_t)__popc(need & ltMask);
        if (!st.active && rank < avail)
        {
            const float4 e0 = rays[cur + rank][0];
            const float4 e1 = rays[cur + rank][1];
            begin_path(st, e0, e1);
            start(__float_as_uint(e1.w));
        }
        const uint32_t n = (uint32_t)__popc(need);
        cur += n < avail ? n : avail;
        need = __ballot_sync(0xffffffffu, !st.active);
    }
}

// Fast-mode sweep in expanded form: with od = o.d, oo = o.o and K = |s|^2 - r^2 (per sphere, computed once per CTA in
// double precision) nb = s.d - od and c = K + oo - 2 s.o, i.e. 8 instead of 10 FP32 issue slots per (ray, sphere):
//   nb = fma(sx,dx, fma(sy,dy, fma(sz,dz, -od)));  c = fma(sx,-2ox, fma(sy,-2oy, fma(sz,-2oz, K+oo)));  discr = fma(nb,nb,-c)
// Same two-pass structure and the same behind-the-origin rejection as SerialHitter. Algebraically the reference's
// test (Maths.cpp:97-102); rounding differs (c loses ~|s|^2 * 2^-24 absolute accuracy), which the fast mode's
// statistical tests bound. Padded "impossible" spheres get K = +1e30 so they can never be candidates here.
struct FastHitterK
{
    uint32_t sphK;      // shared-memory address of {sx, sy, sz, K}[simdCount]
    int simdCount;
    __device__ __forceinline__ float4 ld(int i) const
    {
        float4 r;
        asm("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "r"(sphK + (uint32_t)i * 16u));
        return r;
    }
    __device__ __forceinline__ int hit(const SceneView&, V3 o, V3 d, float tMin, float tMax, float& tOut) const
    {
        const float nod = -fmaf(o.x, d.x, fmaf(o.y, d.y, o.z * d.z));
        const float oo = fmaf(o.x, o.x, fmaf(o.y, o.y, o.z * o.z));
        const float ax = -2.0f * o.x, ay = -2.0f * o.y, az = -2.0f * o.z;
        float bestT = tMax;
        int bestId = -1;
        for (int base = 0; base < simdCount; base += 32)
        {
            const int n = simdCount - base < 32 ? simdCount - base : 32;
            uint32_t neg = 0;
#pragma unroll
            for (int k = 0; k < 32; k += 4)
            {
                if (k < n)
                {
#pragma unroll
                    for (int j = 0; j < 4; ++j)
                    {
                        const float4 s = ld(base + k + j);
                        const float nb = fmaf(s.x, d.x, fmaf(s.y, d.y, fmaf(s.z, d.z, nod)));
                        const float c = fmaf(s.x, ax, fmaf(s.y, ay, fmaf(s.z, az, s.w + oo)));
                        const float discr = fmaf(nb, nb, -c);
                        // reject: discr < 0, or centre behind (nb < 0) with the origin outside (c > 0)
                        const uint32_t rej = __float_as_uint(discr) | (__float_as_uint(nb) & ~__float_as_uint(c));
                        neg = __funnelshift_l(rej, neg, 1);
                    }
                }
            }
            uint32_t cand = ~neg & (n == 32 ? 0xffffffffu : ((1u << n) - 1u));
            while (cand)
            {
                const int bit = 31 - __clz((int)cand);
                cand &= ~(1u << bit);
                const int i = base + (n - 1 - bit);
                const float4 s = ld(i);
                const float nb = fmaf(s.x, d.x, fmaf(s.y, d.y, fmaf(s.z, d.z, nod)));
                const float c = fmaf(s.x, ax, fmaf(s.y, ay, fmaf(s.z, az, s.w + oo)));
                const float discr = fmaf(nb, nb, -c);
                if (discr > 0.0f)
                {
                    const float sq = M<false>::sqrt_(discr);
                    float t = nb - sq;
                    if (t <= tMin) t = nb + sq;
                    if (t > tMin && t < bestT) { bestT = t; bestId = i; }
                }
            }
        }
        tOut = bestT;
        return bestId;
    }
};

// Rewrites the staged sphere array IN PLACE from {s, r^2} to {s, K} (one CTA-wide pass, double precision for the
// cancellation |s|^2 - r^2). The fast kernels need r^2 nowhere else (the normal uses the centre and invRadius), so the
// expanded form costs no extra shared memory and works for any sphere count.
__device__ __forceinline__ void build_sphK(const SceneView& sc, float4* sphInSmem)
{
    for (int i = threadIdx.x; i < sc.simdCount; i += blockDim.x)
    {
        const float4 s = sphInSmem[i];
        const double K = (double)s.x * s.x + (double)s.y * s.y + (double)s.z * s.z - (double)s.w;
        sphInSmem[i].w = i < sc.count ? (float)K : 1.0e30f;
    }
}

// Pair form of the expanded sweep: the sphere array is interleaved in pairs so that one LDS.128 brings the same coordinate
// of TWO spheres, and the ray constants are shared by both. Hopper has no packed FP32 instruction, so each pair costs two
// independent scalar chains; the kernels are FP32-issue bound, and the pair layout halves the shared-memory loads and keeps
// two chains in flight per load: per PAIR of spheres
//   2 LDS.128 {x0,x1,y0,y1} {z0,z1,-K0,-K1},  2 FADD (-K - o.o),  6 FFMA (nb),  6 FFMA (-c),  2 FFMA (discr),
//   2 LOP3 + 2 SHF (sign bits into the candidate mask).
// -c and discr are the exact negations/equals of FastHitterK's c and discr (same products, IEEE negation symmetry), so pass
// 2 — unchanged, on the {s, K} array — sees the same candidates it would have computed itself.
// Where pass 1 reads the pair array from: shared memory at address sphP (two LDS.128 per pair), or the kernel parameter
// (ParamPairs, sweep form 4), where every index is a compile-time constant: ptxas (12.9, sm_90a) then loads the values into
// uniform registers (ULDC.64, two per instruction) that the FFMAs read, with no vector register and no shared-memory
// latency per value. kOneChunk: the scene has at most 64 padded spheres, so the sweep is a single chunk at base 0.
struct SmemPairs
{
    static constexpr bool kOneChunk = false;
    uint32_t sphP;
    __device__ __forceinline__ void load(int pair, float& x0, float& x1, float& y0, float& y1, float& z0, float& z1, float& k0, float& k1) const
    {
        const uint32_t a = sphP + (uint32_t)pair * 32u;
        asm("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(x0), "=f"(x1), "=f"(y0), "=f"(y1) : "r"(a));
        asm("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(z0), "=f"(z1), "=f"(k0), "=f"(k1) : "r"(a + 16u));
    }
};
struct ParamPairsRef
{
    static constexpr bool kOneChunk = true;
    const ParamPairs* pp;       // the kernel's __grid_constant__ parameter
    __device__ __forceinline__ void load(int pair, float& x0, float& x1, float& y0, float& y1, float& z0, float& z1, float& k0, float& k1) const
    {
        const float* f = pp->f + pair * 8;
        x0 = f[0]; x1 = f[1]; y0 = f[2]; y1 = f[3]; z0 = f[4]; z1 = f[5]; k0 = f[6]; k1 = f[7];
    }
};

// Packed-pair pass 1 shared by FastHitterK2 / FastHitterKC / FastHitterK2C: spheres [s0, s0+G) = G/2 pairs of the pair
// array; shifts G rejection signs into `neg` (sphere s0 ends up at the highest of the G new bits).
struct SweepConsts { float DX, DY, DZ, NOD, BX, BY, BZ, NOO; };
template <int G, class P>
__device__ __forceinline__ void sweep_full(const P& pairs, int s0, uint32_t& neg, const SweepConsts& c)
{
#pragma unroll
    for (int j = 0; j < G; j += 2)
    {
        float x0, x1, y0, y1, z0, z1, k0, k1;
        pairs.load((s0 + j) >> 1, x0, x1, y0, y1, z0, z1, k0, k1);
        const float nb0 = fmaf(x0, c.DX, fmaf(y0, c.DY, fmaf(z0, c.DZ, c.NOD)));
        const float nb1 = fmaf(x1, c.DX, fmaf(y1, c.DY, fmaf(z1, c.DZ, c.NOD)));
        const float negc0 = fmaf(x0, c.BX, fmaf(y0, c.BY, fmaf(z0, c.BZ, __fadd_rn(k0, c.NOO))));
        const float negc1 = fmaf(x1, c.BX, fmaf(y1, c.BY, fmaf(z1, c.BZ, __fadd_rn(k1, c.NOO))));
        const float discr0 = fmaf(nb0, nb0, negc0), discr1 = fmaf(nb1, nb1, negc1);
        // reject: discr < 0, or centre behind (nb < 0) with the origin outside (-c < 0)
        const uint32_t r0 = __float_as_uint(discr0) | (__float_as_uint(nb0) & __float_as_uint(negc0));
        const uint32_t r1 = __float_as_uint(discr1) | (__float_as_uint(nb1) & __float_as_uint(negc1));
        neg = __funnelshift_l(r0, neg, 1);
        neg = __funnelshift_l(r1, neg, 1);
    }
}
// The straight-line group between two (warp-uniform) bounds checks is the instruction scheduler's window: a group of 16
// spheres keeps sixteen independent chains in flight. Counts that are not a multiple of the group fall through to halved
// groups, down to 4.
template <int G, class P>
__device__ __forceinline__ void sweep_upto(const P& pairs, int s0, int left, uint32_t& neg, const SweepConsts& c)
{
    if (left >= G) sweep_full<G>(pairs, s0, neg, c);
    else if constexpr (G > 4)
    {
        if (left > 0)
        {
            sweep_upto<G / 2>(pairs, s0, left, neg, c);
            sweep_upto<G / 2>(pairs, s0 + G / 2, left - G / 2, neg, c);
        }
    }
}
// 64 spheres [base, base+n) -> candidate mask, sphere base + J <-> bit 63 - J (n a multiple of 4, 4 <= n <= 64)
template <class P>
__device__ __forceinline__ unsigned long long sweep_chunk64(const P& pairs, int base, int n, const SweepConsts& c)
{
    const int n0 = n < 32 ? n : 32, n1 = n - n0;
    uint32_t neg0 = 0, neg1 = 0;
#pragma unroll
    for (int k = 0; k < 32; k += TPT_P1_GROUP) sweep_upto<TPT_P1_GROUP>(pairs, base + k, n0 - k, neg0, c);
    if (n1 > 0)
    {
#pragma unroll
        for (int k = 0; k < 32; k += TPT_P1_GROUP) sweep_upto<TPT_P1_GROUP>(pairs, base + 32 + k, n1 - k, neg1, c);
    }
    // left-align: after n shifts sphere j of the round sits at bit n-1-j
    const uint32_t c0 = ~neg0 << (32 - n0);
    const uint32_t c1 = n1 > 0 ? ~neg1 << (32 - n1) : 0u;
    return ((unsigned long long)c0 << 32) | c1;
}
// Sweep form 5's pass 1: packed half precision on ParamPairs::h (build_half_pairs states the test; DESIGN §3.1c derives its
// error bound). Per pair of spheres: 6 HFMA2 for xu, xv, 2 HFMA2 for q = xu^2 + xv^2 - R'^2, and LOP3 + LEA.HI that shift
// the two sign bits (15: low sphere, 31: high sphere) into the block's mask. There is no "wholly behind the origin" test:
// pass 2 rejects those spheres (t <= tMin), and the study in DESIGN §3.1c found its 5 more slots per pair dearer than the
// pass-2 trips it saves. The candidates contain form 4's, so pass 2 (unchanged, on {s, K}, ascending sphere order) makes
// the same decisions. The form-4 kernels run it (FastHitterKH) when the parameter's `half` is set. The bound assumes
// |o| <= kHalfOriginBound and a unit direction: if any active lane of the warp has a ray outside that, the warp runs
// form 4's FP32 pass 1 on this trip.
struct HalfPairsRef
{
    static constexpr bool kOneChunk = true;
    const ParamPairs* pp;       // the kernel's __grid_constant__ parameter
};
struct HalfRay { __half2 ux, uy, uz, vx, vy, vz, nou, nov; };
__device__ __forceinline__ __half2 u32_h2(uint32_t w) { __half2 h; memcpy(&h, &w, 4); return h; }
__device__ __forceinline__ uint32_t h2_u32(__half2 h) { uint32_t w; memcpy(&w, &h, 4); return w; }
template <int G>
__device__ __forceinline__ void half_sweep_full(const ParamPairs* pp, int p0, uint32_t& acc, const HalfRay& r)
{
#pragma unroll
    for (int j = 0; j < G; ++j)
    {
        const uint32_t* w = pp->h + (p0 + j) * kHalfPairWords;
        const __half2 X = u32_h2(w[0]), Y = u32_h2(w[1]), Z = u32_h2(w[2]);
        const __half2 xu = __hfma2(X, r.ux, __hfma2(Y, r.uy, __hfma2(Z, r.uz, r.nou)));
        const __half2 xv = __hfma2(X, r.vx, __hfma2(Y, r.vy, __hfma2(Z, r.vz, r.nov)));
        const __half2 q = __hfma2(xu, xu, __hfma2(xv, xv, u32_h2(w[3])));
        acc = (acc >> 1) | (h2_u32(q) & 0x80008000u);
    }
}
template <int G>
__device__ __forceinline__ void half_sweep_upto(const ParamPairs* pp, int p0, int left, uint32_t& acc, const HalfRay& r)
{
    if (left >= G) half_sweep_full<G>(pp, p0, acc, r);
    else if constexpr (G > 2)
    {
        if (left > 0)
        {
            half_sweep_upto<G / 2>(pp, p0, left, acc, r);
            half_sweep_upto<G / 2>(pp, p0 + G / 2, left - G / 2, acc, r);
        }
    }
}
// The candidate mask of the block of 2h spheres whose h pairs start at pair p0: sphere j of the block at bit 31 - j.
__device__ __forceinline__ uint32_t half_block_mask(const ParamPairs* pp, int p0, int h, const HalfRay& r)
{
    uint32_t acc = 0;
    half_sweep_upto<TPT_P1_GROUP / 2>(pp, p0, h, acc, r);
    half_sweep_upto<TPT_P1_GROUP / 2>(pp, p0 + TPT_P1_GROUP / 2, h - TPT_P1_GROUP / 2, acc, r);
    // after h pairs, pair p's signs sit at bits 16 - h + p (sphere p) and 32 - h + p (sphere h + p)
    const uint32_t low = (1u << h) - 1u;
    return __brev(((acc >> (16 - h)) & low) | ((acc >> (32 - 2 * h)) & ~low));
}

// Pass 1 of one chunk of n spheres at base: sphere base + J <-> bit 63 - J of the candidate mask.
template <class P>
__device__ __forceinline__ unsigned long long pass1(const P& pairs, int base, int n, const SweepConsts& C, V3, V3)
{
    return sweep_chunk64(pairs, base, n, C);
}
__device__ __forceinline__ unsigned long long pass1(const HalfPairsRef& pairs, int, int n, const SweepConsts& C, V3 o, V3 d)
{
    const bool inBound = dot(o, o) <= kHalfOriginBound * kHalfOriginBound && fabsf(dot(d, d) - 1.0f) <= 0x1p-18f;
    if (!__all_sync(__activemask(), inBound)) return sweep_chunk64(ParamPairsRef{pairs.pp}, 0, n, C);
    // the branch-free orthonormal basis (u, v) around d of sample_light_cone
    const float sgn = copysignf(1.0f, d.z);
    const float a = __fdividef(-1.0f, sgn + d.z);
    const float b = d.x * d.y * a;
    const V3 u = v3(1.0f + sgn * d.x * d.x * a, sgn * b, -sgn * d.x);
    const V3 v = v3(b, sgn + d.y * d.y * a, -d.y);
    HalfRay r;
    r.ux = __float2half2_rn(u.x); r.uy = __float2half2_rn(u.y); r.uz = __float2half2_rn(u.z);
    r.vx = __float2half2_rn(v.x); r.vy = __float2half2_rn(v.y); r.vz = __float2half2_rn(v.z);
    r.nou = __float2half2_rn(-dot(o, u)); r.nov = __float2half2_rn(-dot(o, v));
    const int n0 = n < 32 ? n : 32, n1 = n - n0;
    const uint32_t m0 = half_block_mask(pairs.pp, 0, n0 / 2, r);
    const uint32_t m1 = n1 > 0 ? half_block_mask(pairs.pp, 16, n1 / 2, r) : 0u;
    return ((unsigned long long)m0 << 32) | m1;
}

// FastHitterK2: pass 1 on the pair array in shared memory; FastHitterKC: on the pair array in the kernel parameter (scenes
// of at most 64 padded spheres); FastHitterKH: form 5's half-precision pass 1 on the same parameter (form 4's on a fallback
// trip). Same pass 2 on the same candidates or a superset of them: ids and distances are bit-identical.
template <class P>
struct FastHitterK2T
{
    uint32_t sphK;      // shared-memory address of {sx, sy, sz, K}[simdCount]         (pass 2)
    P pairs;            // the pair array, 32 B per pair                                (pass 1)
    int simdCount;
    __device__ __forceinline__ float4 ld(int i) const
    {
        float4 r;
        asm("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "r"(sphK + (uint32_t)i * 16u));
        return r;
    }
    __device__ __forceinline__ int hit(const SceneView&, V3 o, V3 d, float tMin, float tMax, float& tOut) const
    {
        const float nod = -fmaf(o.x, d.x, fmaf(o.y, d.y, o.z * d.z));
        const float oo = fmaf(o.x, o.x, fmaf(o.y, o.y, o.z * o.z));
        const float ax = -2.0f * o.x, ay = -2.0f * o.y, az = -2.0f * o.z;
        SweepConsts C;
        C.DX = d.x; C.DY = d.y; C.DZ = d.z; C.NOD = nod;
        C.BX = -ax; C.BY = -ay; C.BZ = -az; C.NOO = -oo;
        float bestT = tMax;
        int bestId = -1;
        // chunks of 64 spheres: pass 1 fills a 64-bit candidate mask (sphere base + J <-> bit 63 - J), pass 2 walks it
        for (int base = 0; base < (P::kOneChunk ? 1 : simdCount); base += 64)
        {
            unsigned long long cand = pass1(pairs, base, simdCount - base < 64 ? simdCount - base : 64, C, o, d);
            // pass 2, two candidates per trip (independent LDS.128 / 9 FMA / MUFU chains); ascending sphere order as before
            while (cand)
            {
                const int ja = __clzll((long long)cand);
                cand &= ~(0x8000000000000000ull >> ja);
                const bool hasB = cand != 0ull;
                const int jb = hasB ? __clzll((long long)cand) : ja;
                cand &= ~(0x8000000000000000ull >> jb);
                const float4 sa = ld(base + ja), sb = ld(base + jb);
                const float nba = fmaf(sa.x, d.x, fmaf(sa.y, d.y, fmaf(sa.z, d.z, nod)));
                const float nbb = fmaf(sb.x, d.x, fmaf(sb.y, d.y, fmaf(sb.z, d.z, nod)));
                const float ca = fmaf(sa.x, ax, fmaf(sa.y, ay, fmaf(sa.z, az, sa.w + oo)));
                const float cb = fmaf(sb.x, ax, fmaf(sb.y, ay, fmaf(sb.z, az, sb.w + oo)));
                const float da = fmaf(nba, nba, -ca), db = fmaf(nbb, nbb, -cb);
                const float sqa = M<false>::sqrt_(fmaxf(da, 0.0f)), sqb = M<false>::sqrt_(fmaxf(db, 0.0f));
                float ta = nba - sqa, tb = nbb - sqb;
                if (ta <= tMin) ta = nba + sqa;
                if (tb <= tMin) tb = nbb + sqb;
                if (da > 0.0f && ta > tMin && ta < bestT) { bestT = ta; bestId = base + ja; }
                if (hasB && db > 0.0f && tb > tMin && tb < bestT) { bestT = tb; bestId = base + jb; }
            }
        }
        tOut = bestT;
        return bestId;
    }
};
using FastHitterK2 = FastHitterK2T<SmemPairs>;
using FastHitterKC = FastHitterK2T<ParamPairsRef>;
using FastHitterKH = FastHitterK2T<HalfPairsRef>;
// The sweep of the form-4 kernels: form 5's (FastHitterKH) when the launch's parameter sets `half`, else form 4's. Each
// is a whole sweep, pass 1 and pass 2, so the FP32 one compiles as it does without form 5. (A choice inside pass 1 only
// left the FP32 pass 1 9-14 % slower than without form 5 on H100; two whole queue bodies doubled the kernel's LDS.128.)
struct FastHitterK45
{
    FastHitterKC fp32;
    const ParamPairs* pp;
    __device__ __forceinline__ int hit(const SceneView& sc, V3 o, V3 d, float tMin, float tMax, float& tOut) const
    {
        if (pp->half) return FastHitterKH{fp32.sphK, HalfPairsRef{pp}, fp32.simdCount}.hit(sc, o, d, tMin, tMax, tOut);
        return fp32.hit(sc, o, d, tMin, tMax, tOut);
    }
};

// Conservative form for scenes the expanded form is NOT accurate enough for (centres far from the origin: the gate in
// tpt_set_scene fails, e.g. the 4096-sphere stress scene): pass 1 is the packed expanded-form sweep with an error bound
// folded into its additive constants, so it can only ADD candidates; pass 2 evaluates every candidate in the reference
// form (Maths.cpp:97-102) on the untouched {s, r^2} array, so hit decisions and distances are the reference form's
// (tpt_debug_hit: bit-identical ids and distances on millions of rays). Bound (u = 2^-24, |d| = 1): |d nb| <= 6u(|s|+|o|),
// |d c| <= 9u(|s|+|o|)^2, hence |d discr| <= 22u(|s|+|o|)^2 for the expanded form and <= 12u(|s|+|o|)^2 for the reference
// form; with (|s|+|o|)^2 <= 2(|s|^2 + o.o) the margin eps_i = 2^-17 (|s_i|^2 + o.o) = 64u * 2(...) covers both. It splits
// into a per-sphere constant (stored with -K_i) and a per-ray constant (folded into -o.o): no extra instruction, and a
// far-away sphere (the ground, |s| = 1000) does not loosen the test of the others. The "wholly behind" rejection needs no
// margin of its own: a sphere it drops wrongly has a true nb below 6u(|s|+|o|) << tMin/2, i.e. both roots below tMin.
struct FastHitterK2C
{
    uint32_t sph;       // shared-memory address of the ORIGINAL {sx, sy, sz, r^2}[simdCount]   (pass 2)
    uint32_t sphP;      // pair array {x0,x1,y0,y1}{z0,z1,-K0,-K1}                             (pass 1)
    int simdCount;
    __device__ __forceinline__ int hit(const SceneView&, V3 o, V3 d, float tMin, float tMax, float& tOut) const
    {
        const float nod = -fmaf(o.x, d.x, fmaf(o.y, d.y, o.z * d.z));
        const float oo = fmaf(o.x, o.x, fmaf(o.y, o.y, o.z * o.z));
        SweepConsts C;
        C.DX = d.x; C.DY = d.y; C.DZ = d.z; C.NOD = nod;
        C.BX = 2.0f * o.x; C.BY = 2.0f * o.y; C.BZ = 2.0f * o.z;
        C.NOO = oo * 7.62939453125e-6f - oo;               // the ray's share of the margin: 2^-17 o.o
        float bestT = tMax;
        int bestId = -1;
        for (int base = 0; base < simdCount; base += 64)
        {
            unsigned long long cand = sweep_chunk64(SmemPairs{sphP}, base, simdCount - base < 64 ? simdCount - base : 64, C);
            // pass 2 on the untouched {s, r^2} array in the reference form (Maths.cpp:97-102), two candidates per trip
            while (cand)
            {
                const int ja = __clzll((long long)cand);
                cand &= ~(0x8000000000000000ull >> ja);
                const bool hasB = cand != 0ull;
                const int jb = hasB ? __clzll((long long)cand) : ja;
                cand &= ~(0x8000000000000000ull >> jb);
                Q4 sa, sb;
                asm("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(sa.x), "=f"(sa.y), "=f"(sa.z), "=f"(sa.w) : "r"(sph + (uint32_t)(base + ja) * 16u));
                asm("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(sb.x), "=f"(sb.y), "=f"(sb.z), "=f"(sb.w) : "r"(sph + (uint32_t)(base + jb) * 16u));
                float nba, nbb;
                const float da = sphere_discr<false>(sa, o, d, nba), db = sphere_discr<false>(sb, o, d, nbb);
                const float sqa = M<false>::sqrt_(fmaxf(da, 0.0f)), sqb = M<false>::sqrt_(fmaxf(db, 0.0f));
                float ta = nba - sqa, tb = nbb - sqb;
                if (ta <= tMin) ta = nba + sqa;
                if (tb <= tMin) tb = nbb + sqb;
                if (da > 0.0f && ta > tMin && ta < bestT) { bestT = ta; bestId = base + ja; }
                if (hasB && db > 0.0f && tb > tMin && tb < bestT) { bestT = tb; bestId = base + jb; }
            }
        }
        tOut = bestT;
        return bestId;
    }
};

// Pair array for FastHitterK2C straight from the staged {s, r^2} array (which stays as it is): -K_i plus the sphere's share
// of the margin, 2^-17 |s_i|^2, in double precision; padded "impossible" spheres get -1e30 (never candidates).
__device__ __forceinline__ void build_sph_pairs_from_r2(const SceneView& sc, const float4* sph, float4* pairs)
{
    for (int p = threadIdx.x; 2 * p < sc.simdCount; p += blockDim.x)
    {
        const float4 a = sph[2 * p], b = sph[2 * p + 1];
        const double Sa = (double)a.x * a.x + (double)a.y * a.y + (double)a.z * a.z, Sb = (double)b.x * b.x + (double)b.y * b.y + (double)b.z * b.z;
        const double m = 7.62939453125e-6;      // 2^-17
        // round the constant UP (towards the permissive side): the margin must not shrink by the rounding of -K
        const float na = __double2float_ru(Sa * m - (Sa - (double)a.w)), nbv = __double2float_ru(Sb * m - (Sb - (double)b.w));
        pairs[2 * p] = make_float4(a.x, b.x, a.y, b.y);
        pairs[2 * p + 1] = make_float4(a.z, b.z, 2 * p < sc.count ? na : -1.0e30f, 2 * p + 1 < sc.count ? nbv : -1.0e30f);
    }
}

// Pair array for FastHitterK2 from the {s, K} array build_sphK() left in place: pair p = spheres 2p, 2p+1 as
// {x0, x1, y0, y1} {z0, z1, -K0, -K1}.
__device__ __forceinline__ void build_sph_pairs(const SceneView& sc, const float4* sphK, float4* pairs)
{
    for (int p = threadIdx.x; 2 * p < sc.simdCount; p += blockDim.x)
    {
        const float4 a = sphK[2 * p], b = sphK[2 * p + 1];
        pairs[2 * p] = make_float4(a.x, b.x, a.y, b.y);
        pairs[2 * p + 1] = make_float4(a.z, b.z, -a.w, -b.w);
    }
}

// Dynamic shared memory of the fast kernels: [staged blob | pad to 128 B | pair array (KFORM 2/3) | per-warp buffers].
// A launch with nothing behind the blob requests the blob itself, unpadded. roundPairs pads the pair array to 128 B
// before the buffers: the slab queue does, variants 5 and 8 (no buffers) and the fit rules of fast_queue_kform and the
// queue's CTA size do not. The difference is deliberate and kept: it sets how much shared memory those launches
// request, and with it their occupancy and grid.
struct FastSmem
{
    uint32_t pairs;     // offset of the pair array
    uint32_t buffers;   // offset of the per-warp buffers (queue: camera rays; wavefront: the path pool)
    uint32_t bytes;     // dynamic shared memory of the launch
};
__host__ __device__ inline FastSmem fast_smem(uint32_t stagedBytes, uint32_t pairBytes = 0, uint32_t bufferBytes = 0,
                                              bool roundPairs = false)
{
    FastSmem s;
    s.pairs = (stagedBytes + 127u) & ~127u;
    s.buffers = s.pairs + (roundPairs ? (pairBytes + 127u) & ~127u : pairBytes);
    s.bytes = pairBytes + bufferBytes != 0 ? s.buffers + bufferBytes : stagedBytes;
    return s;
}

// Sweep setup of the kernels that pick a sweep form KFORM, run after stage_blob/make_view; returns that form's hitter.
//   0  reference form on the staged {s, r^2} array (SerialHitter)
//   1  expanded form: {s, r^2} rewritten to {s, K} in place (FastHitterK)
//   2  expanded form on the pair array, built from {s, K} (FastHitterK2)
//   3  conservative pair array built from {s, r^2}, which stays for the reference-form pass 2 (FastHitterK2C)
//   4  form 2 with the pair array in the kernel parameter pp (FastHitterKC; at most kParamPairSpheres padded spheres),
//      no pair array in shared memory; pass 2 on {s, K} as in form 2
//   5  form 4 with the half-precision pass 1 on pp->h (FastHitterKH). Not an instance of its own: the form-4 kernels
//      sweep with FastHitterK45, which takes form 4's or form 5's complete sweep per call from pp->half
// The sweep's loads are plain (schedulable) asm: their addresses are made opaque AFTER the barrier so that none of them
// can be hoisted above the rewrite of the sphere array or the construction of the pair array.
template <int KFORM>
__device__ __forceinline__ auto prepare_sweep(const SceneView& sc, unsigned char* smem, const SceneBlobLayout& L, uint32_t stagedBytes,
                                              const ParamPairs* pp = nullptr)
{
    float4* sph = reinterpret_cast<float4*>(smem + L.offSph);
    float4* pairs = reinterpret_cast<float4*>(smem + fast_smem(stagedBytes).pairs);
    if constexpr (KFORM == 1 || KFORM == 2 || KFORM == 4) build_sphK(sc, sph);
    __syncthreads();
    if constexpr (KFORM == 0) return SerialHitter<false>();
    else if constexpr (KFORM == 1)
    {
        FastHitterK h; h.sphK = sc.sphShared; h.simdCount = sc.simdCount;
        asm volatile("" : "+r"(h.sphK));
        return h;
    }
    else if constexpr (KFORM == 2)
    {
        build_sph_pairs(sc, sph, pairs);
        __syncthreads();
        FastHitterK2 h; h.sphK = sc.sphShared; h.pairs.sphP = smem_u32(pairs); h.simdCount = sc.simdCount;
        asm volatile("" : "+r"(h.sphK), "+r"(h.pairs.sphP));
        return h;
    }
    else if constexpr (KFORM == 4)
    {
        FastHitterK45 h; h.fp32.sphK = sc.sphShared; h.fp32.pairs.pp = pp; h.fp32.simdCount = sc.simdCount; h.pp = pp;
        asm volatile("" : "+r"(h.fp32.sphK));
        return h;
    }
    else
    {
        build_sph_pairs_from_r2(sc, sph, pairs);
        __syncthreads();
        FastHitterK2C h; h.sph = sc.sphShared; h.sphP = smem_u32(pairs); h.simdCount = sc.simdCount;
        asm volatile("" : "+r"(h.sph), "+r"(h.sphP));
        return h;
    }
}

// Light-sampling mode of path_step, fixed at compile time per kernel instance:
//   kLsOn       explicit light sampling (DO_LIGHT_SAMPLING 1); the scene flag is not looked at
//   kLsOff      DO_LIGHT_SAMPLING 0: a Lambert vertex bounces at once and adds its emission; no shadow rays, so the
//               light-sampling block and the QPath fields it keeps (nextDir, thrAlb, nl, pend) are dead code
//   kLsRuntime  either, from the scene flag (warp-uniform): the kernels that have no kLsOff twin
enum { kLsOn = 0, kLsOff = 1, kLsRuntime = 2 };

// The first light from index j on that a Lambert vertex on sphere `mid` samples: a light never samples itself (Test.cpp:100).
__device__ __forceinline__ int next_light(const SceneView& sc, int j, int mid)
{
    while (j < sc.nLights && sc.lights[j].id == mid) ++j;
    return j;
}

// The shadow ray from o towards light Lr (Test.cpp:104-131, the facing normal nl already resolved): a direction l drawn
// uniformly in the cone the light subtends, and the returned weight m * omega / pi. The ray adds thrAlb * E_light * weight
// when it reaches its light.
// The cone from o that light Lr subtends: its unit axis sw, and the cosine of its half-angle as the return value (not
// above 0 where o lies inside or on the light, d <= r).
__device__ __forceinline__ float light_cone_cos(const LightRec& Lr, V3 o, V3& sw)
{
    V3 scn = v3(Lr.cx, Lr.cy, Lr.cz);
    V3 pc = scn - o;
    float d2 = dot(pc, pc);
    float inv = __frsqrt_rn(d2);          // d2 is a squared distance between distinct spheres: never denormal
    sw = pc * inv;
    return M<false>::sqrt_(1.0f - Lr.radius * Lr.radius * inv * inv);
}

// The branch-free orthonormal basis (su, sv) around the unit vector w of Duff et al. 2017 (sample_light_cone's cone,
// hg_sample's scattering cone).
__device__ __forceinline__ void duff_basis(V3 w, V3& su, V3& sv)
{
    const float sgn = copysignf(1.0f, w.z);
    const float oa = __fdividef(-1.0f, sgn + w.z);       // |sgn + w.z| in [1, 2]: MUFU.RCP + FMUL instead of the IEEE sequence
    const float ob = w.x * w.y * oa;
    su = v3(1.0f + sgn * w.x * w.x * oa, sgn * ob, -sgn * w.x);
    sv = v3(ob, sgn + w.y * w.y * oa, -w.y);
}

// TEX with fogG (a fog scatter vertex, lambert_next): the weight is omega x the fog's phase function at cos = l . nl (nl
// holds the incoming direction there; fogG points at the fog's {g, ...}) instead.
template <bool TEX = false>
__device__ __forceinline__ float sample_light_cone(const LightRec Lr, V3 o, V3 nl, uint32_t& rng, V3& l, const Q4* fogG = nullptr)
{
    V3 sw;
    const float cosAMax = light_cone_cos(Lr, o, sw);
    // any orthonormal (su, sv) around sw gives the same cone-sample distribution (phi is uniform): use the
    // branch-free basis of Duff et al. 2017 instead of normalize(cross(up, sw)), cross(sw, su) (Test.cpp:108-109)
    V3 su, sv;
    duff_basis(sw, su, sv);
    float eps1 = RandomFloat01(rng), eps2 = RandomFloat01(rng);
    float cosA = 1.0f - eps1 + eps1 * cosAMax;
    float sinA = M<false>::sqrt_(1.0f - cosA * cosA);
    float phi = 2.0f * TPT_PI * eps2;
    float sp, cp;
    __sincosf(phi, &sp, &cp);
    l = su * (cp * sinA) + sv * (sp * sinA) + sw * cosA;
    float omega = 2.0f * TPT_PI * (1.0f - cosAMax);
    if constexpr (TEX)
        if (fogG) return omega * hg_phase(dot(l, nl), fogG->x);
    float dl = dot(l, nl);
    float m = (0.0f < dl) ? dl : 0.0f;
    return m * omega * (1.0f / TPT_PI);
}

// ---- homogeneous media inside glass spheres (tpt_set_media, kSceneMedia; DESIGN §3.14)
// A Henyey-Greenstein direction around the unit direction d with asymmetry g (g > 0 forward) from the draws xi1 (cos theta)
// and xi2 (phi).
__device__ __forceinline__ V3 hg_sample(V3 d, float g, float xi1, float xi2)
{
    float cosT = 1.0f - 2.0f * xi1;
    if (fabsf(g) >= 1e-3f)
    {
        const float s = __fdividef(1.0f - g * g, 1.0f - g + 2.0f * g * xi1);
        cosT = fminf(fmaxf(__fdividef(1.0f + g * g - s * s, 2.0f * g), -1.0f), 1.0f);
    }
    const float sinT = M<false>::sqrt_(fmaxf(1.0f - cosT * cosT, 0.0f));
    float sp, cp;
    __sincosf(2.0f * TPT_PI * xi2, &sp, &cp);
    V3 su, sv;
    duff_basis(d, su, sv);
    return su * (sinT * cp) + sv * (sinT * sp) + d * cosT;
}

// exp(-sigma t) per channel, at most 1 (the factor only ever lowers the throughput).
__device__ __forceinline__ V3 transmittance(const Q4& m, float t)
{
    return v3(fminf(__expf(-m.x * t), 1.0f), fminf(__expf(-m.y * t), 1.0f), fminf(__expf(-m.z * t), 1.0f));
}

// The medium of sphere `mid` on a path segment of length t that ended on the inside face of that glass sphere: with
// sigma_s > 0 one free-flight distance t_s = -ln(1 - u) / sigma_s is drawn. Returns true when the path scattered before t
// (the hit is not shaded): past the call's depth cap (sc.maxDepth) it ends with nothing added (*finished), otherwise the
// throughput takes exp(-sigma_a t_s) and the path goes on from the scatter point along an HG direction (two more draws)
// as a path ray whose next hit adds its emission. Otherwise the throughput takes exp(-sigma_a t) and the caller shades the hit.
// Media entry [count] and the entries of spheres without a medium are zero: no draw, and a factor of exactly 1.
__device__ __forceinline__ bool medium_step(const SceneView& sc, QPath& st, int mid, float t, bool& finished)
{
    const Q4 m = sc.media[mid];
    if (m.w > 0.0f)
    {
        const float ts = __fdividef(-__logf(1.0f - RandomFloat01(st.rng)), m.w);
        if (ts < t)
        {
            if (st.depth >= sc.maxDepth) { finished = true; return true; }
            const float g = reinterpret_cast<const float*>(sc.media + sc.count + 1)[mid];
            st.thr = st.thr * transmittance(m, ts);
            st.o = st.o + st.d * ts;
            const float xi1 = RandomFloat01(st.rng);
            const float xi2 = RandomFloat01(st.rng);
            st.d = hg_sample(st.d, g, xi1, xi2);
            st.doMaterialE = true;
            ++st.depth;
            return true;
        }
    }
    st.thr = st.thr * transmittance(m, t);
    return false;
}

// ---- fog between the spheres (tpt_set_fog, kSceneFog; DESIGN §3.16)
// QPath::mid of a fog scatter vertex on its way through lambert_next. A Lambert vertex's mid is its sphere (0..count) or,
// from tpt_trace_irradiance, the caller's id, which begin_vertex keeps at -1 or above in the instances that trace fog: no
// light is excluded (next_light), and the mark cannot be a caller's.
constexpr int kMidFog = -2;
// QPath::kind of the path ray that leaves a fog scatter vertex. It and the vertex's cone rays start at distance 0 rather
// than TPT_MIN_T: the scatter point lies in air, but it may lie within TPT_MIN_T of a surface, which such a ray would
// skip (into glass at an angle past the critical one, where total internal reflection then keeps the path until the
// cap). path_step sets it back to 0 once the ray is traced.
constexpr int kKindFogPath = INT_MAX;

// The fog length L of the segment o + s d, s in [0, t], and where it starts, max(t_in, 0), in tin (fog_chord).
__device__ __forceinline__ float fog_length(const SceneView& sc, V3 o, V3 d, float t, float& tin)
{
    const Q4 b = sc.fog[0];
    return fog_chord(o.x, o.y, o.z, d.x, d.y, d.z, t, b.x, b.y, b.z, b.w, &tin);
}

// A shadow ray's factor over its segment of length t in air: exp(-(sigma_a + sigma_s) L) per channel, no draw.
__device__ __forceinline__ V3 fog_transmittance(const SceneView& sc, V3 o, V3 d, float t)
{
    float tin;
    const float L = fog_length(sc, o, d, t, tin);
    const Q4 m = sc.fog[1];
    return transmittance(Q4{m.x + m.w, m.y + m.w, m.z + m.w, 0.0f}, L);
}

// The fog on a path ray's segment of length t in air (it ended on the outside face of a sphere, or left the scene with
// t = TPT_MAX_T): with a fog length L > 0 and sigma_s > 0 one free-flight distance t_s = -ln(1 - u) / sigma_s is drawn
// along the fog part. Returns true when the path scattered at o + d (max(t_in, 0) + t_s), t_s < L (the hit or miss is
// not shaded): past the call's depth cap it ends with nothing added (*finished); otherwise the throughput takes
// exp(-sigma_a t_s) and two more draws give a Henyey-Greenstein direction. Without light sampling the path goes on along
// it as a path ray whose next hit adds its emission (depth + 1). With it, the vertex is set up like a Lambert vertex for
// lambert_next (wantLight): nextDir the HG direction, thrAlb the throughput, nl the incoming direction, mid kMidFog and
// doMaterialE false (no environment sample); lambert_next samples every light and then bounces (depth + 1). Otherwise
// the throughput takes exp(-sigma_a L) and the caller shades the hit or the miss.
template <int LS>
__device__ __forceinline__ bool fog_step(const SceneView& sc, QPath& st, float t, bool& finished, bool& wantLight)
{
    float tin;
    const float L = fog_length(sc, st.o, st.d, t, tin);
    if (!(L > 0.0f)) return false;
    const Q4 m = sc.fog[1];
    if (m.w > 0.0f)
    {
        const float ts = __fdividef(-__logf(1.0f - RandomFloat01(st.rng)), m.w);
        if (ts < L)
        {
            if (st.depth >= sc.maxDepth) { finished = true; return true; }
            st.thr = st.thr * transmittance(m, ts);
            st.o = st.o + st.d * (tin + ts);
            const float xi1 = RandomFloat01(st.rng);
            const float xi2 = RandomFloat01(st.rng);
            const V3 dir = hg_sample(st.d, sc.fog[2].x, xi1, xi2);
            if (LS == kLsOff)
            {
                st.d = dir;
                st.doMaterialE = true;
                st.kind = kKindFogPath;
                ++st.depth;
            }
            else
            {
                st.nextDir = dir;
                st.thrAlb = st.thr;
                st.nl = st.d;
                st.mid = kMidFog;
                st.doMaterialE = false;
                wantLight = true;
            }
            return true;
        }
    }
    st.thr = st.thr * transmittance(m, L);
    return false;
}

// ---- "max_depth" past the reference's cap (kSceneDepth; DESIGN §3.15)
// Russian roulette at a path ray's hit once the path is at depth TPT_MAX_DEPTH or deeper, in calls whose cap is larger:
// one draw u, and with q = min(1, max channel of the throughput) the path ends with nothing added when u >= q (returns
// true); otherwise its throughput is divided by q, which keeps the estimator of the capped path unbiased.
__device__ __forceinline__ bool roulette(QPath& st)
{
    const float u = RandomFloat01(st.rng);
    const float q = fminf(fmaxf(fmaxf(st.thr.x, st.thr.y), st.thr.z), 1.0f);
    if (!(u < q)) return true;
    if (q < 1.0f) st.thr = st.thr * __fdividef(1.0f, q);   // q >= u >= 0 and q > 0 here
    return false;
}

// Metal bounce direction (Test.cpp:137-150); the path goes on when dot(result, normal) > 0. With roughness == 0 the
// unit-sphere sample has zero weight, so the fast mode skips drawing it (the exact mode must draw it: it advances the
// shared RNG stream).
__device__ __forceinline__ V3 metal_dir(V3 d, V3 normal, float roughness, uint32_t& rng)
{
    V3 refl = reflect(d, normal);
    if (roughness != 0.0f) refl = refl + roughness * fast_in_unit_sphere(rng);
    return M<false>::normalize(refl);
}

// Bilinear lookup of the W x H lat-long image of RGBA texels at `tex` (global memory) in the direction d
// (include/tpt_b200.h pins the mapping): phi = atan2(d.x, -d.z), theta = acos(d.y); continuous texel coordinates
// u = (phi + pi) / 2pi * W, v = theta / pi * H, texel (i, j) centred at (i + 1/2, j + 1/2), row 0 at +y; columns wrapping,
// rows clamped. Every blend is a + f * (b - a), so a constant image returns its constant bit for bit. Four 128-bit
// read-only loads; RGB: twelve 32-bit ones of R, G and B only, at 32-bit texel offsets (fewer registers live: the texture
// instances stay at 80 without spilling). The environment map (env_radiance) and the sphere textures (sphere_texture)
// both read through it.
// CELL: also the sampling probability P of the cell [i, i+1) x [j, j+1) that holds (u + 1/2, v + 1/2), from the alpha of
// whichever of the four texels that is (tpt_env_tables.h).
template <bool CELL = false, bool RGB = false>
__device__ __forceinline__ V3 latlong_lookup(const float4* tex, int W, int H, V3 d, float* cellP = nullptr)
{
    constexpr float kPi = 3.14159265358979f;
    const float phi = atan2f(d.x, -d.z);
    const float theta = acosf(fminf(fmaxf(d.y, -1.0f), 1.0f));
    const float u = (phi + kPi) * (0.5f / kPi) * (float)W - 0.5f;
    const float v = theta * (1.0f / kPi) * (float)H - 0.5f;
    const float fu = floorf(u), fv = floorf(v);
    const float tu = u - fu, tv = v - fv;
    int x0 = (int)fu, y0 = (int)fv;                  // x0 in [-1, W - 1] up to rounding, y0 in [-1, H - 1]
    x0 = x0 < 0 ? x0 + W : (x0 >= W ? x0 - W : x0);
    x0 = min(max(x0, 0), W - 1);                     // a non-finite d converts to 0: any texel, never out of bounds
    const int x1 = x0 + 1 == W ? 0 : x0 + 1;
    const int y1 = min(max(y0 + 1, 0), H - 1);
    y0 = min(max(y0, 0), H - 1);
    auto lerp = [](float p, float q, float f) { return p + f * (q - p); };
    if constexpr (RGB)
    {
        auto ld = [&](int x, int y) {
            const float* f = reinterpret_cast<const float*>(tex + (uint32_t)(y * W + x));
            return v3(__ldg(f), __ldg(f + 1), __ldg(f + 2));
        };
        const V3 a = ld(x0, y0), b = ld(x1, y0), c = ld(x0, y1), e = ld(x1, y1);
        if constexpr (CELL) *cellP = __ldg(reinterpret_cast<const float*>(tex + (uint32_t)((tv < 0.5f ? y0 : y1) * W + (tu < 0.5f ? x0 : x1))) + 3);
        const V3 top = v3(lerp(a.x, b.x, tu), lerp(a.y, b.y, tu), lerp(a.z, b.z, tu));
        const V3 bot = v3(lerp(c.x, e.x, tu), lerp(c.y, e.y, tu), lerp(c.z, e.z, tu));
        return v3(lerp(top.x, bot.x, tv), lerp(top.y, bot.y, tv), lerp(top.z, bot.z, tv));
    }
    const float4* row0 = tex + (size_t)y0 * W;
    const float4* row1 = tex + (size_t)y1 * W;
    const float4 a = __ldg(row0 + x0), b = __ldg(row0 + x1), c = __ldg(row1 + x0), e = __ldg(row1 + x1);
    if constexpr (CELL) *cellP = tv < 0.5f ? (tu < 0.5f ? a.w : b.w) : (tu < 0.5f ? c.w : e.w);
    const V3 top = v3(lerp(a.x, b.x, tu), lerp(a.y, b.y, tu), lerp(a.z, b.z, tu));
    const V3 bot = v3(lerp(c.x, e.x, tu), lerp(c.y, e.y, tu), lerp(c.z, e.z, tu));
    return v3(lerp(top.x, bot.x, tv), lerp(top.y, bot.y, tv), lerp(top.z, bot.z, tv));
}

// Radiance of tpt_set_environment's lat-long map in the unit direction d (row 0 at the zenith).
template <bool CELL = false>
__device__ __forceinline__ V3 env_radiance(const SceneView& sc, V3 d, float* cellP = nullptr)
{
    const float4* env = reinterpret_cast<const float4*>(((uint64_t)sc.envHi << 32) | sc.envLo);
    return latlong_lookup<CELL>(env, sc.envW, sc.envH, d, cellP);
}

// The layer of sphere `id` in the texture set ts (sc.tex: tpt_set_textures' albedo; sc.emit: tpt_set_emission_textures'
// emission; the caller checks the set's flag), or -1 for a sphere without one (-1 in the table, or an id at or past
// ts.spheres, which begin_call keeps at most the scene's count: padding spheres have none).
__device__ __forceinline__ int sphere_layer(const TexSet& ts, int id)
{
    if (id >= ts.spheres) return -1;
    return __ldg(reinterpret_cast<const int*>(((uint64_t)ts.tabHi << 32) | ts.tabLo) + id);
}

// The W x H texels of layer `layer` of ts.
__device__ __forceinline__ const float4* texture_layer(const TexSet& ts, int layer)
{
    return reinterpret_cast<const float4*>(((uint64_t)ts.texHi << 32) | ts.texLo) + (uint32_t)(layer * ts.W * ts.H);
}

// base x the lookup of layer `layer` (>= 0) of ts at the shading normal n ((pos - centre) / r): the texture's product
// comes first, so a constant layer c gives base x c rounded once. Draws no random numbers. CELL: also the alpha of the
// cell that holds n's (u, v) into *cellP (latlong_lookup).
template <bool CELL = false>
__device__ __forceinline__ V3 sphere_texture_layer(const TexSet& ts, int layer, V3 base, V3 n, float* cellP = nullptr)
{
    return base * latlong_lookup<CELL, true>(texture_layer(ts, layer), ts.W, ts.H, n, cellP);
}

// The textured value of a hit on sphere `id` with shading normal n: base (the material's albedo or emission) x the
// lookup of the sphere's layer in ts at n, or base itself for a sphere without a layer (sphere_layer's test, as early
// returns: the AOV kernel's code stays what it was before emission textures).
__device__ __forceinline__ V3 sphere_texture(const TexSet& ts, int id, V3 base, V3 n)
{
    if (id >= ts.spheres) return base;
    const int layer = __ldg(reinterpret_cast<const int*>(((uint64_t)ts.tabHi << 32) | ts.tabLo) + id);
    if (layer < 0) return base;
    return sphere_texture_layer(ts, layer, base, n);
}

// What a fast path sees when it leaves the scene: the caller's environment while one is set, else the reference sky
// (sky() stays the exact and reference-GPU kernels' own, untouched).
__device__ __forceinline__ V3 fast_sky(V3 d, const SceneView& sc)
{
    return (sc.flags & kSceneEnvironment) ? env_radiance(sc, d) : sky(d, sc);
}

// ---- environment sampling ("environment_sampling", kSceneEnvSampling; tpt_env_tables.h pins tables, draws, density)
constexpr float kEnvPdfScale = 1.0f / (2.0f * TPT_PI * TPT_PI);      // pdf_e = P * W * H / (2 pi^2 sin theta)
constexpr int kKindEnv = -1;                                         // QPath::kind of an environment sample's shadow ray

// Power-heuristic weight of a bounce against the environment sampler, pdf_b^2 / (pdf_b^2 + pdf_e^2); 1 where the sampler
// has no density (pdf_e zero or not a number: P = 0 at a pole).
__device__ __forceinline__ float env_bounce_weight(float pb, float pe)
{
    const float b2 = pb * pb, e2 = pe * pe;
    return e2 > 0.0f ? b2 / (b2 + e2) : 1.0f;
}

// One draw from the tables of a W x H lat-long image (the environment map or an emission layer): tex, its texels with
// each cell's probability P in their alpha; rows, its H row entries followed by its W * H column entries
// (tpt_env_tables.h). Six draws (row, row alias test, column, column alias test, in-cell u and v offsets); returns the
// unit direction of the drawn (u, v) by the inverse of latlong_lookup's mapping, with P and s = sin theta. The tables
// are read through the read-only path.
__device__ __forceinline__ V3 latlong_sample(const float4* tex, const float2* rows, uint32_t W, uint32_t H, uint32_t& rng,
                                             float& P, float& s)
{
    const float2* cols = rows + H;
    uint32_t j = __umulhi((XorShift32(rng) & 0xFFFFFFu) << 8, H);          // (k * H) >> 24
    const float2 er = __ldg(rows + j);
    if (!(RandomFloat01(rng) < er.x)) j = (uint32_t)__float_as_int(er.y);
    const float2* crow = cols + (size_t)j * W;
    uint32_t i = __umulhi((XorShift32(rng) & 0xFFFFFFu) << 8, W);
    const float2 ec = __ldg(crow + i);
    if (!(RandomFloat01(rng) < ec.x)) i = (uint32_t)__float_as_int(ec.y);
    P = __ldg(&tex[(size_t)j * W + i].w);
    const float u = (float)i + RandomFloat01(rng);
    const float v = (float)j + RandomFloat01(rng);
    float sp, cp, c;
    __sincosf(__fdividef(u, (float)W) * (2.0f * TPT_PI) - TPT_PI, &sp, &cp);
    __sincosf(__fdividef(v, (float)H) * TPT_PI, &s, &c);
    return v3(s * sp, c, -s * cp);
}

// One environment sample at a Lambert vertex whose bounce is cosine-distributed about nl: latlong_sample's direction
// into l, and true when its shadow ray is traced (c = l.nl > 0 and sin theta > 0), with pend = (c / pi) pdf_e /
// (pdf_e^2 + pdf_b^2), pdf_b = c / pi: the ray adds thrAlb * L(l) * pend when it leaves the scene.
__device__ __forceinline__ bool sample_env(const SceneView& sc, V3 nl, uint32_t& rng, V3& l, float& pend)
{
    const uint32_t W = (uint32_t)sc.envW, H = (uint32_t)sc.envH;
    const float4* tex = reinterpret_cast<const float4*>(((uint64_t)sc.envHi << 32) | sc.envLo);
    float P, s;
    l = latlong_sample(tex, reinterpret_cast<const float2*>(tex + (size_t)W * H), W, H, rng, P, s);
    const float fW = (float)W, fH = (float)H;
    const float cn = dot(l, nl);
    if (!(cn > 0.0f && s > 0.0f)) return false;
    const float pe = P * (fW * fH * kEnvPdfScale) / s;
    const float pb = cn * (1.0f / TPT_PI);
    pend = pb * pe / (pe * pe + pb * pb);
    return true;
}

// The miss of a path in the sampling instances: fast_sky's radiance, and for the bounce of a Lambert vertex that took an
// environment sample (doMaterialE false, pend = the bounce's pdf_b >= 0) that radiance times env_bounce_weight. Camera
// rays, Metal and glass bounces (doMaterialE true) and vertices without a sample (pend -1) keep full weight.
__device__ __forceinline__ V3 fast_sky_mis(const SceneView& sc, const QPath& st)
{
    if (!(sc.flags & kSceneEnvSampling)) return fast_sky(st.d, sc);
    float P;
    const V3 L = env_radiance<true>(sc, st.d, &P);
    if (st.doMaterialE || !(st.pend >= 0.0f)) return L;
    const float s = M<false>::sqrt_(fmaxf(fmaf(-st.d.y, st.d.y, 1.0f), 0.0f));
    const float pe = P * ((float)sc.envW * (float)sc.envH * kEnvPdfScale) / s;
    return L * env_bounce_weight(st.pend, pe);
}

// ---- emission texture sampling ("emission_texture_sampling", kSceneEmitSampling; tpt_env_tables.h pins the tables)
// At a light-sampled Lambert vertex o, a light with a sampleable emission layer gets, after its cone sample, one texture
// sample: latlong_sample's draw from its layer's tables gives the unit normal n and the point x = c + r n, of solid-angle
// density at o
//   pt(x) = P W H / (2 pi^2 sin theta) / r^2 * |x - o|^2 / cos_x,   cos_x = n . normalize(o - x),
// against the cone's pc = 1 / omega. Both rays are weighted with the power heuristic, written with q = pt omega = pt / pc
// (so that omega 0, P 0 and an overflowing pt stay finite): the cone's w_c = pc^2 / (pc^2 + pt^2) = 1 / (1 + q^2), the
// texture sample's pend_t = (m / pi) pt / (pt^2 + pc^2) = (m / pi) omega / (q + 1 / q).
constexpr int kKindEmit = -2;                // QPath::kind of light j's texture-sample shadow ray: kKindEmit - j

// The sampling tables of emission layer `layer` (>= 0): its rows, then its columns; null when the layer has none (all
// of its weights are zero: the sentinel alias kEmitNoTables in its first row).
__device__ __forceinline__ const float2* emit_tables(const TexSet& ts, int layer)
{
    const float2* t = reinterpret_cast<const float2*>(reinterpret_cast<const int*>(((uint64_t)ts.tabHi << 32) | ts.tabLo) +
                                                      ts.tabWords) + (size_t)layer * ((size_t)ts.H + (size_t)ts.W * ts.H);
    return __float_as_int(__ldg(t).y) < 0 ? nullptr : t;
}

// q = pt(x) omega for a point x on light Lr with unit normal n, sin theta s and cell probability P, seen from o at
// squared distance d2 with cos_x = cx.
__device__ __forceinline__ float emit_q(const TexSet& ts, const LightRec& Lr, float P, float s, float d2, float cx, float omega)
{
    return __fdividef(P * ((float)ts.W * (float)ts.H * kEnvPdfScale) * d2 * omega, s * (Lr.radius * Lr.radius) * cx);
}

// The cone weight w_c of a cone ray from o that met light Lr (emission layer `layer`) at x with normal n, where the
// lookup read cell probability P: 1 for a light without tables and for o inside or on the light (no texture sample).
__device__ __forceinline__ float emit_cone_weight(const SceneView& sc, const LightRec& Lr, int layer, V3 o, V3 x, V3 n, float P)
{
    V3 sw;
    const float cosAMax = light_cone_cos(Lr, o, sw);
    if (!(cosAMax > 0.0f) || !emit_tables(sc.emit, layer)) return 1.0f;
    const V3 ox = o - x;
    const float d2 = dot(ox, ox);
    const float s = M<false>::sqrt_(fmaxf(fmaf(-n.y, n.y, 1.0f), 0.0f));
    const float q = emit_q(sc.emit, Lr, P, s, d2, dot(n, ox) * __frsqrt_rn(d2), 2.0f * TPT_PI * (1.0f - cosAMax));
    return q > 0.0f ? __fdividef(1.0f, fmaf(q, q, 1.0f)) : 1.0f;
}

// The texture sample of light Lr at the vertex st.o (facing normal st.nl), after its cone sample: nothing, and no draws,
// for a light without a sampleable layer or a vertex inside or on it; otherwise the six draws, and true when its shadow
// ray is traced (x faces o, m = l . nl > 0 and sin theta > 0), with the direction in st.d and pend_t in st.pend.
__device__ __forceinline__ bool sample_emit(const SceneView& sc, const LightRec& Lr, QPath& st)
{
    const int layer = sphere_layer(sc.emit, Lr.id);
    if (layer < 0) return false;
    const float2* tabs = emit_tables(sc.emit, layer);
    V3 sw;
    const float cosAMax = light_cone_cos(Lr, st.o, sw);
    if (!tabs || !(cosAMax > 0.0f)) return false;
    float P, s;
    const V3 n = latlong_sample(texture_layer(sc.emit, layer), tabs, (uint32_t)sc.emit.W, (uint32_t)sc.emit.H, st.rng, P, s);
    const V3 ox = st.o - (v3(Lr.cx, Lr.cy, Lr.cz) + n * Lr.radius);
    const float d2 = dot(ox, ox), inv = __frsqrt_rn(d2);
    const float cx = dot(n, ox) * inv;
    st.d = neg(ox) * inv;
    const float m = dot(st.d, st.nl);
    if (!(cx > 0.0f && m > 0.0f && s > 0.0f)) return false;
    const float omega = 2.0f * TPT_PI * (1.0f - cosAMax);
    const float q = emit_q(sc.emit, Lr, P, s, d2, cx, omega);
    st.pend = m * (1.0f / TPT_PI) * __fdividef(omega, q + __fdividef(1.0f, q));
    return true;
}

// The rest of a Lambert vertex after its shadow ray towards light lightFrom - 1 (or, lightFrom = 0, after the vertex's
// own shading): the next light the vertex samples, its cone and shadow ray, or, when none is left, the bounce along
// st.nextDir with throughput st.thrAlb. Without light sampling (kLsOff) there are no lights to sample: the bounce.
// ENVM 2 with kSceneEnvSampling: after the lights (lightFrom <= nLights), one environment sample at a vertex hit from
// outside (st.doMaterialE, path_step) and its shadow ray, which comes back with lightFrom = nLights + 1; then the
// bounce, which keeps its pdf_b in pend for its miss (fast_sky_mis), or -1 where the vertex took no sample.
// TEX with kSceneEmitSampling: after the cone ray of light coneOf (>= 0), that light's texture sample (sample_emit) and its
// shadow ray, which comes back with lightFrom = coneOf + 1 and coneOf -1.
// TEX at a fog scatter vertex (mid kMidFog, fog_step): every light's cone weighted by the phase function, no texture or
// environment sample, then the bounce.
template <int LS, int ENVM = 1, bool TEX = false>
__device__ __forceinline__ void lambert_next(const SceneView& sc, QPath& st, int lightFrom, int coneOf = -1)
{
    if constexpr (TEX)
        if (coneOf >= 0 && (sc.flags & kSceneEmitSampling) && st.mid != kMidFog && sample_emit(sc, sc.lights[coneOf], st))
        {
            st.kind = kKindEmit - coneOf;
            return;
        }
    const int j = LS == kLsOff ? sc.nLights : next_light(sc, lightFrom, st.mid);
    if (j < sc.nLights)
    {
        if constexpr (TEX)
            st.pend = sample_light_cone<true>(sc.lights[j], st.o, st.nl, st.rng, st.d, st.mid == kMidFog ? sc.fog + 2 : nullptr);
        else
            st.pend = sample_light_cone(sc.lights[j], st.o, st.nl, st.rng, st.d);
        st.kind = 1 + j;
    }
    else
    {
        bool envSampled = false;
        if constexpr (ENVM == 2)
        {
            envSampled = (sc.flags & kSceneEnvSampling) && st.doMaterialE;
            if (envSampled && lightFrom <= sc.nLights && sample_env(sc, st.nl, st.rng, st.d, st.pend))
            {
                st.kind = kKindEnv;
                return;
            }
        }
        st.d = st.nextDir;
        st.thr = st.thrAlb;
        if constexpr (TEX) st.kind = st.mid == kMidFog ? kKindFogPath : 0;
        else st.kind = 0;
        if constexpr (ENVM == 2) st.pend = envSampled ? fmaxf(dot(st.nextDir, st.nl), 0.0f) * (1.0f / TPT_PI) : -1.0f;
        st.doMaterialE = LS == kLsRuntime && emission_after_lambert(sc);
        ++st.depth;
    }
}

// One iteration of the per-lane path state machine every fast kernel shades with: intersect the lane's current ray
// (path or shadow) against all spheres, then shade. Returns true when the lane's path has ended (st.col is final).
// ENVM, the environment mode: 0 the miss sees the reference sky only (the slab queue's 64-register 8-CTA instances, which
// a lookup made spill; pick_queue does not choose them while an environment is set); 1 fast_sky; 2 fast_sky plus, where
// the call's kSceneEnvSampling is set, environment sampling at light-sampled Lambert vertices (the slab queue's 6-CTA and
// 768-thread light-sampling instances).
// NEXT false: stop before lambert_next, for a caller that runs it later (the block wavefront). A Lambert vertex just shaded
// and a returning shadow ray then leave the light to go on from in st.kind.
// TEX: where the call's kSceneTextures is set, Lambert and Metal hits take the textured albedo for the material's albedo,
// and where its kSceneEmissionTextures is set, every hit takes the textured emission for the material's emission and a
// light's shadow ray that reaches it the light's emission x its layer's lookup at the normal where the ray meets it (the
// slab queue's instances with ENVM 2 and their light-sampling-off twins; pick_queue runs them while either is set), and
// where its kSceneMedia is set, a path ray that ends on the inside face of a glass sphere runs medium_step first. TEX also
// takes the call's depth cap (sc.maxDepth, "max_depth") for the reference's, with roulette past it where it is larger.
// Where its kSceneFog is set, a path ray in air (a miss, or a hit on an outside face) runs fog_step first, and a shadow
// ray in air takes the fog's transmittance (fog_transmittance).
template <int LS, int ENVM = 1, bool NEXT = true, bool TEX = false, class Hitter>
__device__ __forceinline__ bool path_step(const SceneView& sc, QPath& st, unsigned& rc, const Hitter& hitter)
{
    // ---- intersect
    float t = TPT_MAX_T;
    int id = -1;
    // TEX: the rays that leave a fog scatter point (its path ray, and its cone rays: kind > 0 at mid kMidFog) start at 0
    float tMin = TPT_MIN_T;
    if constexpr (TEX)
        if (st.kind == kKindFogPath || (st.kind > 0 && st.mid == kMidFog)) tMin = 0.0f;
    if (st.active) { id = hitter.hit(sc, st.o, st.d, tMin, TPT_MAX_T, t); ++rc; }

    // ---- shade
    bool wantLight = false;
    int lightFrom = 0;
    int coneOf = -1;          // TEX: the light whose cone ray just returned
    bool finished = false;
    if (st.active)
    {
        if (LS == kLsOff || st.kind == 0 || (TEX && st.kind == kKindFogPath))
        {
            if constexpr (TEX) st.kind = 0;
            // a miss runs in air to TPT_MAX_T: the fog may scatter the path before it leaves
            bool fogged = false;
            if constexpr (TEX)
                if (id < 0 && (sc.flags & kSceneFog)) fogged = fog_step<LS>(sc, st, TPT_MAX_T, finished, wantLight);
            if (fogged) {}
            else if (id < 0)
            {
                if constexpr (ENVM == 2) st.col = st.col + st.thr * fast_sky_mis(sc, st);
                else if constexpr (ENVM == 1) st.col = st.col + st.thr * fast_sky(st.d, sc);
                else st.col = st.col + st.thr * sky(st.d, sc);
                finished = true;
            }
            else
            {
                Q4 s = ld_sph(sc, id);
                V3 pos = st.o + st.d * t;
                V3 normal = (pos - v3(s.x, s.y, s.z)) * sc.invRadius[id];
                const int mid = id < sc.count ? id : sc.count;
                Mat mat = load_mat(sc, mid);
                // the compiler turns a three-way test of mat.type into a jump table (LDC from the constant bank + BRX: two
                // long-latency steps in front of every shading branch); keeping the second test opaque keeps it two branches
                int mtype = mat.type;
                // Lambert and Metal use the albedo (glass does not): with textures, the textured one
                if constexpr (TEX)
                {
                    if ((sc.flags & kSceneTextures) && mtype != kDielectric) mat.albedo = sphere_texture(sc.tex, id, mat.albedo, normal);
                    // every emission this hit adds below is mat.emissive: with emission textures, the textured one
                    if (sc.flags & kSceneEmissionTextures) mat.emissive = sphere_texture(sc.emit, id, mat.emissive, normal);
                }
                // the hit is not shaded when, past the reference's depth in a call whose "max_depth" is larger, Russian
                // roulette ends the path first (roulette), or when the path segment ran inside a glass sphere with a
                // medium and scattered inside it (medium_step; otherwise the medium absorbs along it), or ran in air and
                // scattered in the fog (fog_step; otherwise the fog absorbs along it)
                bool unshaded = false;
                if constexpr (TEX)
                {
                    if (sc.maxDepth > TPT_MAX_DEPTH && st.depth >= TPT_MAX_DEPTH && roulette(st)) unshaded = finished = true;
                    else if ((sc.flags & kSceneMedia) && mtype == kDielectric && dot(st.d, normal) > 0.0f)
                        unshaded = medium_step(sc, st, mid, t, finished);
                    else if ((sc.flags & kSceneFog) && !(dot(st.d, normal) > 0.0f))
                        unshaded = fog_step<LS>(sc, st, t, finished, wantLight);
                }
                // the depth cap: the reference's in every instance but TEX's, which take the call's
                const int maxDepth = TEX ? sc.maxDepth : TPT_MAX_DEPTH;
                if (unshaded) {}
                else if (st.depth >= maxDepth) { st.col = st.col + st.thr * mat.emissive; finished = true; }
                else if (LS == kLsOff && mtype == kLambert)
                {
                    // Test.cpp:86-92 without the light loop; the emission is always added (Test.cpp:209-215 compiled out)
                    st.col = st.col + st.thr * mat.emissive;
                    V3 target = normal + RandomUnitVector<false>(st.rng);
                    st.thr = st.thr * mat.albedo;
                    st.o = pos; st.d = M<false>::normalize(target); ++st.depth;
                }
                else if (mtype == kLambert)
                {
                    if (st.doMaterialE) st.col = st.col + st.thr * mat.emissive;
                    V3 target = normal + RandomUnitVector<false>(st.rng);
                    st.nextDir = M<false>::normalize(target);
                    st.thrAlb = st.thr * mat.albedo;
                    st.nl = dot(normal, st.d) < 0.0f ? normal : neg(normal);
                    // until the bounce, doMaterialE says whether the vertex takes an environment sample: only when hit from
                    // outside, where the bounce's axis (normal) is nl
                    if constexpr (ENVM == 2) st.doMaterialE = dot(normal, st.d) < 0.0f;
                    st.mid = mid;
                    st.o = pos;
                    wantLight = true; lightFrom = 0;
                }
                else if (opaque_int(mtype) == kMetal)
                {
                    V3 outDir = metal_dir(st.d, normal, mat.roughness, st.rng);
                    if (dot(outDir, normal) > 0.0f)
                    {
                        if (LS == kLsOff || st.doMaterialE) st.col = st.col + st.thr * mat.emissive;
                        st.doMaterialE = true;
                        st.thr = st.thr * mat.albedo;
                        st.o = pos; st.d = outDir; ++st.depth;
                    }
                    else { st.col = st.col + st.thr * mat.emissive; finished = true; }
                }
                else
                {
                    V3 att, outDir;
                    bool ok = scatter_specular<false>(mat, st.d, pos, normal, st.rng, att, outDir);
                    if (!ok) { st.col = st.col + st.thr * mat.emissive; finished = true; }
                    else
                    {
                        if (LS == kLsOff || st.doMaterialE) st.col = st.col + st.thr * mat.emissive;
                        st.doMaterialE = true;
                        st.thr = st.thr * att;
                        st.o = pos; st.d = outDir; ++st.depth;
                    }
                }
            }
        }
        else if (ENVM == 2 && st.kind == kKindEnv)
        {
            // the environment sample's shadow ray (sample_env); after it, the bounce
            if (id < 0)
            {
                V3 e = env_radiance(sc, st.d);
                if constexpr (TEX)
                    if (sc.flags & kSceneFog) e = e * fog_transmittance(sc, st.o, st.d, TPT_MAX_T);
                st.col = st.col + (st.thrAlb * e) * st.pend;
            }
            wantLight = true; lightFrom = sc.nLights + 1;
        }
        else
        {
            // a light's shadow ray: its cone's (kind 1 + j) or, with TEX, its texture sample's (kind kKindEmit - j)
            const bool texRay = TEX && st.kind < kKindEnv;
            const int j = texRay ? kKindEmit - st.kind : st.kind - 1;
            const LightRec& Lj = sc.lights[j];
            if (id == Lj.id)
            {
                V3 e = v3(Lj.ex, Lj.ey, Lj.ez);
                float pend = st.pend;
                // an emission-textured light: its layer's lookup at the normal of the point where the shadow ray meets it,
                // and with kSceneEmitSampling a cone ray's power-heuristic weight against the light's texture sample
                if constexpr (TEX)
                    if (sc.flags & kSceneEmissionTextures)
                    {
                        const int layer = sphere_layer(sc.emit, id);
                        if (layer >= 0)
                        {
                            const V3 x = st.o + st.d * t;
                            const V3 n = (x - v3(Lj.cx, Lj.cy, Lj.cz)) * sc.invRadius[id];
                            if (!texRay && (sc.flags & kSceneEmitSampling) && st.mid != kMidFog)
                            {
                                float P;
                                e = sphere_texture_layer<true>(sc.emit, layer, e, n, &P);
                                pend *= emit_cone_weight(sc, Lj, layer, st.o, x, n, P);
                            }
                            else
                                e = sphere_texture_layer(sc.emit, layer, e, n);
                        }
                    }
                // a shadow ray that meets its light's outside face ran in air: the fog's transmittance along it
                if constexpr (TEX)
                    if ((sc.flags & kSceneFog) && !(dot(st.d, st.o + st.d * t - v3(Lj.cx, Lj.cy, Lj.cz)) > 0.0f))
                        e = e * fog_transmittance(sc, st.o, st.d, t);
                st.col = st.col + (st.thrAlb * e) * pend;
            }
            wantLight = true; lightFrom = j + 1;
            if (!texRay) coneOf = j;
        }
    }
    if (NEXT && LS != kLsOff && wantLight) lambert_next<LS, ENVM, TEX>(sc, st, lightFrom, coneOf);
    return finished;
}

// tpt_trace_irradiance: the lane's fresh path (begin_path from a point entry {p, n}: st.o = p, st.d = n) becomes a white
// Lambert vertex at p whose facing normal is n, as if a camera ray had just hit it: the bounce direction drawn first, then
// lambert_next picks the first light (or the bounce). No emission of its own (doMaterialE is not looked at before the
// next hit); depth 0, so the path keeps a camera path's budget. `mid`: the sphere the point lies on, or -1.
template <int LS, int ENVM = 1, bool TEX = false>
__device__ __forceinline__ void begin_vertex(const SceneView& sc, QPath& st, int mid)
{
    st.nl = st.d;
    st.nextDir = M<false>::normalize(st.d + RandomUnitVector<false>(st.rng));
    st.thrAlb = v3(1, 1, 1);
    st.mid = TEX ? max(mid, -1) : mid;     // (TEX: a negative id never matches a light, and kMidFog marks fog vertices)
    lambert_next<LS, ENVM, TEX>(sc, st, 0);     // (begin_path left doMaterialE true: the point takes an environment sample)
}

// The sphere id of point entry `tag` (tpt_trace_irradiance, tpt_trace_samples): ids are per input, so an entry of a list
// reads its input's. -1 without ids.
__device__ __forceinline__ int point_id(const int* ids, const int* entries, uint32_t tag)
{
    return ids ? __ldg(ids + (entries ? (uint32_t)__ldg(entries + tag) : tag)) : -1;
}

// ---- variant 0 ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kFastThreads)
k_fast_mega(DrawParams p, const unsigned char* __restrict__ blob, SceneBlobLayout L, int count, int nLights, uint32_t stagedBytes)
{
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ uint64_t bar;
    __shared__ float sW[kMaxFramesPerDraw];
    __shared__ float sWPrev;
    stage_blob(smem, blob, stagedBytes, &bar);
    if (threadIdx.x == 0) { float wp; blend_weights(p, sW, wp); sWPrev = wp; }
    __syncthreads();
    SceneView sc = make_view(smem, blob, L, stagedBytes, count, nLights);

    // 16x16 pixel block, each warp an 8x4 patch
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tilesX = (p.width + 15) / 16;
    const int tx = blockIdx.x % tilesX, ty = blockIdx.x / tilesX;
    const int x = tx * 16 + (warp & 1) * 8 + (lane & 7);
    const int ri = ty * 16 + (warp >> 1) * 4 + (lane >> 3);
    unsigned rc = 0;
    if (x < p.width && ri < p.numRows)
    {
        const int y = region_pixel(p, ri, x).y;
        SerialHitter<false> hitter;
        V3 acc = v3(0, 0, 0);
        const float invSpp = 1.0f / (float)p.spp;
        for (int fi = 0; fi < p.numFrames; ++fi)
        {
            // one stream per pixel and frame, carried across the pixel's samples
            uint32_t state = pixel_seed((uint32_t)(y * p.width + x), (uint32_t)(p.frame0 + fi));
            V3 col = v3(0, 0, 0);
            for (int s = 0; s < p.spp; ++s)
            {
                QPath st;
                const Ray r = fast_camera_ray(p, x, y, state);
                begin_path(st, r, state);
                while (!path_step<kLsRuntime>(sc, st, rc, hitter)) {}
                state = st.rng;
                col = col + st.col;
            }
            acc = acc + col * (invSpp * sW[fi]);
        }
        float* px = p.image + region_pixel(p, ri, x).off * 4;
        st_stream_f4(px, blend_prev(p, px, sWPrev, acc.x, acc.y, acc.z));
    }
    flush_ray_count(p.rayCounter, rc, lane);
}

// ---- variant 1 ------------------------------------------------------------------------------------------------
template <int MINB>
__global__ void __launch_bounds__(kFastThreads, MINB)
k_fast_persistent(DrawParams p, const unsigned char* __restrict__ blob, SceneBlobLayout L, int count, int nLights,
                  uint32_t stagedBytes, int numTiles)
{
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ uint64_t bar;
    __shared__ float sW[kMaxFramesPerDraw];
    __shared__ float sWPrev;
    __shared__ float sAcc[kTilePix * 3];
    __shared__ int sTile;
    __shared__ int sTask;
    stage_blob(smem, blob, stagedBytes, &bar);
    if (threadIdx.x == 0) { float wp; blend_weights(p, sW, wp); sWPrev = wp; }
    for (int i = threadIdx.x; i < kTilePix * 3; i += kFastThreads) sAcc[i] = 0.0f;
    SceneView sc = make_view(smem, blob, L, stagedBytes, count, nLights);
    const int lane = threadIdx.x & 31;
    const long long regionPix = (long long)p.numRows * p.width;
    const int S = p.spp * p.numFrames;          // samples per pixel in this draw
    const float invSpp = 1.0f / (float)p.spp;
    SerialHitter<false> hitter;
    unsigned rc = 0;

    for (;;)
    {
        __syncthreads(); // sAcc zeroed / previous tile written
        if (threadIdx.x == 0) { sTile = (int)atomicAdd(p.workCounter, 1u); sTask = 0; }
        __syncthreads();
        const int tile = sTile;
        if (tile >= numTiles) break;
        const long long pix0 = (long long)tile * kTilePix;
        const int tilePix = (int)(regionPix - pix0 < kTilePix ? regionPix - pix0 : kTilePix);
        const int tileTasks = tilePix * S;

        QPath st;
        st.active = false;
        for (;;)
        {
            // ---- regeneration: lanes without a path take the next (pixel, sample) of the tile
            unsigned need = __ballot_sync(0xffffffffu, !st.active);
            if (need)
            {
                int base = 0;
                const int leader = __ffs(need) - 1;
                if (lane == leader) base = atomicAdd(&sTask, __popc(need));
                base = __shfl_sync(0xffffffffu, base, leader);
                if (!st.active)
                {
                    const int task = base + __popc(need & ((1u << lane) - 1u));
                    if (task < tileTasks)
                    {
                        // samples of one pixel sit in adjacent lanes: coherent primary rays
                        const int pixIn = task / S, sIdx = task % S;
                        const int fi = sIdx / p.spp;
                        const RegionPixel q = region_pixel(p, pix0 + pixIn);
                        uint32_t rng = pixel_seed((uint32_t)(q.y * p.width + q.x) * (uint32_t)p.spp + (uint32_t)(sIdx % p.spp),
                                                  (uint32_t)(p.frame0 + fi));
                        const Ray r = fast_camera_ray(p, q.x, q.y, rng);
                        begin_path(st, r, rng);
                        st.pixOff = (uint32_t)pixIn;        // pixel index inside the tile
                        st.weight = invSpp * sW[fi];
                    }
                }
            }
            if (!__any_sync(0xffffffffu, st.active)) break;

            if (path_step<kLsRuntime>(sc, st, rc, hitter))
            {
                atomicAdd(&sAcc[st.pixOff * 3 + 0], st.col.x * st.weight);
                atomicAdd(&sAcc[st.pixOff * 3 + 1], st.col.y * st.weight);
                atomicAdd(&sAcc[st.pixOff * 3 + 2], st.col.z * st.weight);
                st.active = false;
            }
        }

        // ---- tile done
        __syncthreads();
        write_tile(p, sAcc, pix0, tilePix, sWPrev, kFastThreads);
    }
    flush_ray_count(p.rayCounter, rc, lane);
}

// Diagnostic build (-DTPT_TRACE_WARPS=1, tools/warp_trace.py): every warp of k_fast_queue records global-timer stamps (entry,
// first slab, queue exhausted, exit), its trip counts and the lane-slots it used after the queue ran dry: the kernel's
// end effects (fill, drain, stragglers) measured instead of guessed. Not compiled into the shipped library.
#ifndef TPT_TRACE_WARPS
#define TPT_TRACE_WARPS 0
#endif
#if TPT_TRACE_WARPS
__device__ unsigned long long* g_warpTrace = nullptr;
__device__ __forceinline__ unsigned long long gtimer() { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); return t; }
#endif

// KFORM: the sweep form (prepare_sweep). THREADS: 128 (6 CTAs/SM) for scenes whose staged geometry is small; one big CTA
// per SM when the sphere arrays fill most of an SM's shared memory.
// Dynamic shared memory (FastSmem): [staged blob][pair array (KFORM 2/3)][per-warp camera-ray buffers, 2 KB per warp at raysOffset].
// The body is shared by k_fast_queue (light sampling) and k_fast_queue_nolight (DO_LIGHT_SAMPLING 0) below.
// SRC: the ray source. kSrcCamera: camera rays of the image region. kSrcRays (k_fast_rays): the caller's p.numRays rays
// (load_slab_rays), a slab being 64 consecutive rays x one sample index, finished paths adding col / spp to p.image[ray];
// with p.pointStart (tpt_trace_irradiance) the entries are surface points, each sample starting as a Lambert vertex.
// With p.sums (tpt_trace_samples) they add (v, 1) and, with p.sq4, (v^2, 0) per sample instead, and with p.entries the
// slab's entries are list positions whose inputs load_slab_rays gathers.
// kSrcPixels (k_fast_samples): the draw's camera rays for the p.numRays entries of a pixel list (generate_list_rays), a
// slab being 64 consecutive entries x one sample index, finished paths adding (col, 1) to p.image[entry] and, with
// MOMENTS, (col^2, 0) to p.sq4[entry].
enum QueueSource { kSrcCamera = 0, kSrcRays = 1, kSrcPixels = 2 };
template <int THREADS, int KFORM, int LS, int SRC = kSrcCamera, bool MOMENTS = false, int ENVM = 1, bool TEX = false>
__device__ __forceinline__ void
fast_queue_body(DrawParams p, const unsigned char* __restrict__ blob, SceneBlobLayout L, int count, int nLights,
                uint32_t stagedBytes, uint32_t numSlabs, uint32_t S, unsigned int* __restrict__ bandDone, uint32_t mtilesPerBand,
                uint32_t raysOffset, const ParamPairs& pp)
{
    // a pixel list with an index outside the image, or an entry list with an index outside the inputs, traces nothing
    // (the call reports the index)
    if constexpr (SRC == kSrcPixels)
        if (p.pixels && *p.badPixel != ~0ull) return;
    if constexpr (SRC == kSrcRays)
        if (p.entries && *p.badPixel != ~0ull) return;
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ uint64_t bar;
    __shared__ float sW[kMaxFramesPerDraw];
    // camera rays of the warp's current slab, generated 4 per lane in one convergent burst when the slab is fetched:
    // {origin.xyz, rng state} {direction.xyz, pixel offset}; regeneration then only pops an entry.
    float4 (*sRays)[kSlabPix][2] = reinterpret_cast<float4 (*)[kSlabPix][2]>(smem + raysOffset);
#if TPT_TRACE_WARPS
    const unsigned long long trEntry = gtimer();
    unsigned long long trReady = 0, trDry = 0;
    unsigned trTrips = 0, trDryTrips = 0, trDryLanes = 0;
#endif
    stage_blob(smem, blob, stagedBytes, &bar);
    if (threadIdx.x == 0) { float wp; blend_weights(p, sW, wp); }
    // the 128-thread instances are only launched for scenes whose whole blob is staged (launch_fast): their view points into
    // shared memory for every section, so materials, lights and 1/r load with LDS instead of generic LD
    SceneView sc = make_view<THREADS == 128>(smem, blob, L, stagedBytes, count, nLights);
    const auto hitter = prepare_sweep<KFORM>(sc, smem, L, stagedBytes, &pp);
    const int lane = threadIdx.x & 31;
    const uint32_t regionPix = SRC != kSrcCamera ? p.numRays : (uint32_t)((long long)p.numRows * p.width);
    const float invSpp = 1.0f / (float)p.spp;

    unsigned rc = 0;

    // warp-uniform slab cursor
    uint32_t slabCur = 0, slabEnd = 0;
    float slabW = 0.0f;
    bool exhausted = false;
    // progress reporting for host-buffer draws (bandDone != nullptr): slabs are dealt in pixel order, so the image
    // completes band by band; every lane counts the paths it finished per band and publishes the count (after a
    // __threadfence so its reductions are visible first) when it moves on to the next band. The host's copy stream
    // waits on these counters (cuStreamWaitValue32) and starts the D2H of a band while later bands are still traced.
    // (Measured: whichever band is dealt first completes at ~50 % of the kernel, not at 1/bands — warps progress
    // unevenly and a few keep their first slab for a long time — so about half of the copy overlaps; dealing slabs from
    // both ends of the image by hardware warp slot, and cheap-rows-first ordering, did not change that.)
    uint32_t slabBand = 0;
    int curBand = -1;
    uint32_t doneCnt = 0, myBand = 0;
    // tpt_trace_irradiance (p.pointStart, launch-uniform): a lane that takes a point entry starts it as a Lambert vertex
    // (begin_vertex) inside the deal in the 128-thread instances, and right after the deal in the 768-thread ones. Both
    // places were measured (H100 SXM, 700 W; trace_rays, whose paths never take the branch): inside the deal the
    // 768-thread form-3 instance sweeps the 4096-sphere stress scene 4.5 % slower than without the feature, after the deal
    // it runs as before (+0.5 %), while for the 128-thread instances the deal is the place that costs nothing.
    constexpr bool kStartInDeal = THREADS != TPT_BIG_THREADS;
    const bool pointStart = SRC == kSrcRays && p.pointStart;
    const int* pointIds = p.pointIds;
    const int* entries = p.entries;
    bool fresh = false;       // the lane has just been dealt an entry (the 768-thread instances' start after the deal)

    QPath st;
    st.active = false;
    for (;;)
    {
        // a slab from the global counter: its rays into the warp's buffer, tag = image float4 offset (camera rays) or entry.
        // (Defined inside the loop: defined above it, the 768-thread KFORM 0 k_fast_samples instances took one more register.)
        auto refill = [&](const DrawParams& p) {
            uint32_t slab = 0;
            if (lane == 0) slab = atomicAdd(p.workCounter, 1u);
            slab = __shfl_sync(0xffffffffu, slab, 0);
            if (slab >= numSlabs) return kDealExhausted;
            uint32_t mtile = slab / S;
            const uint32_t s = slab - mtile * S;
            // progress mode: walk the image from its LAST macro-tile to its first. Row 0 is the bottom of the image
            // (ground, light sampling: the expensive pixels); starting with the cheap upper rows makes pixels
            // complete early at a high rate, so most of the D2H runs under the expensive rows' tracing.
            if (bandDone) mtile = (numSlabs / S) - 1u - mtile;
            const uint32_t pix0 = mtile * kSlabPix;
            slabEnd = regionPix - pix0 < (uint32_t)kSlabPix ? regionPix - pix0 : (uint32_t)kSlabPix;
            slabCur = 0;
            const int ri0 = (int)(pix0 / (uint32_t)p.width), x0 = (int)(pix0 - (uint32_t)ri0 * (uint32_t)p.width);
            const uint32_t fi = s / (uint32_t)p.spp;
            const uint32_t sample = s - fi * (uint32_t)p.spp, frame = (uint32_t)p.frame0 + fi;
            // tpt_trace_samples: a sample's value is col x weight, weight 1 (rays) or pi (points, set at the start)
            slabW = SRC == kSrcRays && p.sums ? 1.0f : invSpp * sW[fi];
            slabBand = bandDone ? mtile / mtilesPerBand : 0u;
            __syncwarp();       // every lane has popped what it needed from the previous slab
            if constexpr (SRC == kSrcRays) slabEnd = load_slab_rays(p, sRays[threadIdx.x >> 5], lane, slabEnd, pix0, sample, frame);
            else if constexpr (SRC == kSrcPixels) generate_list_rays(p, sRays[threadIdx.x >> 5], lane, slabEnd, pix0, sample, frame);
            else generate_slab_rays(p, sRays[threadIdx.x >> 5], lane, slabEnd, x0, ri0, sample, frame, -1);
            __syncwarp();
            return kDealRefilled;
        };
        deal_paths(p, st, sRays[threadIdx.x >> 5], slabCur, slabEnd, exhausted, lane, refill, [&](uint32_t tag) {
            st.pixOff = tag; st.weight = slabW; myBand = slabBand;
            // tpt_trace_irradiance: the entry is a point {p, n}; E = pi x the white Lambert vertex's radiance
            if constexpr (SRC == kSrcRays && kStartInDeal)
                if (pointStart)
                {
                    begin_vertex<LS, ENVM, TEX>(sc, st, point_id(pointIds, entries, tag));
                    st.weight *= TPT_PI;
                }
            if constexpr (SRC == kSrcRays && !kStartInDeal) fresh = true;
        });
        if constexpr (SRC == kSrcRays && !kStartInDeal)
            if (pointStart && fresh)
            {
                begin_vertex<LS, ENVM, TEX>(sc, st, point_id(pointIds, entries, st.pixOff));
                st.weight *= TPT_PI;
                fresh = false;
            }
        if (!__any_sync(0xffffffffu, st.active)) break;
#if TPT_TRACE_WARPS
        if (!trReady) trReady = gtimer();
        ++trTrips;
        if (exhausted) { if (!trDry) trDry = gtimer(); ++trDryTrips; trDryLanes += (unsigned)__popc(__ballot_sync(0xffffffffu, st.active)); }
#endif

        if (path_step<LS, ENVM, true, TEX>(sc, st, rc, hitter))
        {
            if constexpr (SRC == kSrcPixels)
            {
                red_add_f4(p.image + (size_t)st.pixOff * 4, st.col.x, st.col.y, st.col.z, 1.0f);
                if constexpr (MOMENTS)
                    red_add_f4(p.sq4 + (size_t)st.pixOff * 4, st.col.x * st.col.x, st.col.y * st.col.y, st.col.z * st.col.z);
            }
            else
            {
                // the mean's share col / spp, or with p.sums (tpt_trace_samples) the sample v and its count
                const V3 v = st.col * st.weight;
                red_add_f4(p.image + (size_t)st.pixOff * 4, v.x, v.y, v.z, SRC == kSrcRays && p.sums ? 1.0f : 0.0f);
                if constexpr (SRC == kSrcRays)
                    if (p.sq4) red_add_f4(p.sq4 + (size_t)st.pixOff * 4, v.x * v.x, v.y * v.y, v.z * v.z);
            }
            st.active = false;
            if (bandDone)
            {
                if ((int)myBand != curBand)
                {
                    if (doneCnt) { __threadfence(); atomicAdd(bandDone + curBand, doneCnt); }
                    curBand = (int)myBand; doneCnt = 0;
                }
                ++doneCnt;
            }
        }
    }
    if (bandDone && doneCnt) { __threadfence(); atomicAdd(bandDone + curBand, doneCnt); }
    flush_ray_count(p.rayCounter, rc, lane);
#if TPT_TRACE_WARPS
    if (lane == 0 && g_warpTrace)
    {
        unsigned smid; asm volatile("mov.u32 %0, %smid;" : "=r"(smid));
        unsigned long long* t = g_warpTrace + ((size_t)blockIdx.x * (THREADS / 32) + (threadIdx.x >> 5)) * 8;
        t[0] = trEntry; t[1] = trReady; t[2] = trDry; t[3] = gtimer(); t[4] = trTrips; t[5] = trDryTrips; t[6] = trDryLanes; t[7] = smid;
    }
#endif
}

// path_step's environment mode of a light-sampling slab-queue instance with MINB CTAs per SM and sweep form KFORM: the
// reference-form (KFORM 0) 6-CTA and 768-thread instances sample the environment (pick_queue runs them while it is
// sampled), the other 6-CTA, 768-thread and 7-CTA ones only look it up, the 8-CTA ones have no lookup. Measured on an
// H100 (700 W): the sampling code in the packed-sweep instance bench.py runs (k_fast_queue<128, 6, 4>) cost its
// map-less 720p draw 20 % (23 200 -> 18 400 Mray/s) at the same 80 registers and no stack, so it is kept out of the
// instances the default sweep forms run.
__host__ __device__ constexpr int env_mode(int minb, int kform) { return minb == 8 ? 0 : minb == 7 || kform != 0 ? 1 : 2; }
// path_step's TEX of a slab-queue instance, light sampling on or off: the same reference-form 6-CTA and 768-thread
// instances look up textures (pick_queue runs them while textures are set), so no instance a default call runs carries
// the lookup.
__host__ __device__ constexpr bool tex_mode(int minb, int kform) { return env_mode(minb, kform) == 2; }

template <int THREADS, int MINB, int KFORM>
__global__ void __launch_bounds__(THREADS, MINB)
k_fast_queue(DrawParams p, const unsigned char* __restrict__ blob, SceneBlobLayout L, int count, int nLights,
             uint32_t stagedBytes, uint32_t numSlabs, uint32_t S, unsigned int* __restrict__ bandDone, uint32_t mtilesPerBand,
             uint32_t raysOffset, const __grid_constant__ ParamPairs pp)
{
    fast_queue_body<THREADS, KFORM, kLsOn, kSrcCamera, false, env_mode(MINB, KFORM), tex_mode(MINB, KFORM)>(p, blob, L, count, nLights, stagedBytes, numSlabs, S, bandDone, mtilesPerBand, raysOffset, pp);
}

// DO_LIGHT_SAMPLING 0 (scene flag kSceneNoLightSampling): the same kernel without the light-sampling half of the state
// machine. Same launch shapes and instances as k_fast_queue (launch_queue_t picks one or the other).
template <int THREADS, int MINB, int KFORM>
__global__ void __launch_bounds__(THREADS, MINB)
k_fast_queue_nolight(DrawParams p, const unsigned char* __restrict__ blob, SceneBlobLayout L, int count, int nLights,
                     uint32_t stagedBytes, uint32_t numSlabs, uint32_t S, unsigned int* __restrict__ bandDone, uint32_t mtilesPerBand,
                     uint32_t raysOffset, const __grid_constant__ ParamPairs pp)
{
    fast_queue_body<THREADS, KFORM, kLsOff, kSrcCamera, false, MINB != 8 ? 1 : 0, tex_mode(MINB, KFORM)>(p, blob, L, count, nLights, stagedBytes, numSlabs, S, bandDone, mtilesPerBand, raysOffset, pp);
}

// tpt_trace_rays: the slab queue on caller rays (RAYS = true), with the same launch shapes as k_fast_queue and the
// DO_LIGHT_SAMPLING 0 twin. Only the instances pick_queue<true> can choose are instantiated.
template <int THREADS, int MINB, int KFORM>
__global__ void __launch_bounds__(THREADS, MINB)
k_fast_rays(DrawParams p, const unsigned char* __restrict__ blob, SceneBlobLayout L, int count, int nLights,
            uint32_t stagedBytes, uint32_t numSlabs, uint32_t S, unsigned int* __restrict__ bandDone, uint32_t mtilesPerBand,
            uint32_t raysOffset, const __grid_constant__ ParamPairs pp)
{
    fast_queue_body<THREADS, KFORM, kLsOn, kSrcRays, false, env_mode(MINB, KFORM), tex_mode(MINB, KFORM)>(p, blob, L, count, nLights, stagedBytes, numSlabs, S, bandDone, mtilesPerBand, raysOffset, pp);
}

template <int THREADS, int MINB, int KFORM>
__global__ void __launch_bounds__(THREADS, MINB)
k_fast_rays_nolight(DrawParams p, const unsigned char* __restrict__ blob, SceneBlobLayout L, int count, int nLights,
                    uint32_t stagedBytes, uint32_t numSlabs, uint32_t S, unsigned int* __restrict__ bandDone, uint32_t mtilesPerBand,
                    uint32_t raysOffset, const __grid_constant__ ParamPairs pp)
{
    fast_queue_body<THREADS, KFORM, kLsOff, kSrcRays, false, MINB != 8 ? 1 : 0, tex_mode(MINB, KFORM)>(p, blob, L, count, nLights, stagedBytes, numSlabs, S, bandDone, mtilesPerBand, raysOffset, pp);
}

// tpt_draw_samples: the slab queue on a pixel list (SRC = kSrcPixels), per-entry sums and, with MOMENTS, sums of squares.
// Same launch shapes and instances as k_fast_rays.
template <int THREADS, int MINB, int KFORM, bool MOMENTS>
__global__ void __launch_bounds__(THREADS, MINB)
k_fast_samples(DrawParams p, const unsigned char* __restrict__ blob, SceneBlobLayout L, int count, int nLights,
               uint32_t stagedBytes, uint32_t numSlabs, uint32_t S, unsigned int* __restrict__ bandDone, uint32_t mtilesPerBand,
               uint32_t raysOffset, const __grid_constant__ ParamPairs pp)
{
    fast_queue_body<THREADS, KFORM, kLsOn, kSrcPixels, MOMENTS, env_mode(MINB, KFORM), tex_mode(MINB, KFORM)>(p, blob, L, count, nLights, stagedBytes, numSlabs, S, bandDone,
                                                                 mtilesPerBand, raysOffset, pp);
}

template <int THREADS, int MINB, int KFORM, bool MOMENTS>
__global__ void __launch_bounds__(THREADS, MINB)
k_fast_samples_nolight(DrawParams p, const unsigned char* __restrict__ blob, SceneBlobLayout L, int count, int nLights,
                       uint32_t stagedBytes, uint32_t numSlabs, uint32_t S, unsigned int* __restrict__ bandDone,
                       uint32_t mtilesPerBand, uint32_t raysOffset, const __grid_constant__ ParamPairs pp)
{
    fast_queue_body<THREADS, KFORM, kLsOff, kSrcPixels, MOMENTS, MINB != 8 ? 1 : 0, tex_mode(MINB, KFORM)>(p, blob, L, count, nLights, stagedBytes, numSlabs, S, bandDone,
                                                                  mtilesPerBand, raysOffset, pp);
}

// The index check of tpt_draw_samples' pixel list and tpt_trace_samples' entry list: the smallest (entry << 32 | index) of the entries whose index lies outside [0, numPix)
// into *bad, which stays ~0 when there is none.
__global__ void k_check_pixels(const int* __restrict__ pixels, long long n, long long numPix, unsigned long long* bad)
{
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    {
        const int v = __ldg(pixels + i);
        if (v < 0 || v >= numPix) atomicMin(bad, ((unsigned long long)i << 32) | (uint32_t)v);
    }
}

// ---- variant 8 ------------------------------------------------------------------------------------------------
// "warp-owned pixel groups": the warp-level dealing and path state machine of variant 3, but the unit a warp pulls from
// the global counter is a GROUP of kGroupPix consecutive pixels with ALL their samples of this draw. The group's radiance
// is accumulated in the warp's own shared-memory slot; when its last path ends, 16 lanes write the 16 finished float4
// pixels with ONE coalesced 128-bit store each (256 contiguous bytes) — straight into the caller's buffer: local HBM,
// a peer GPU's HBM over NVLink (multi-GPU write-out), or page-locked HOST memory over PCIe (host-buffer draws finish
// with the kernel: no staging image, no device-to-host copy). No prepare kernel, no L2 reductions, no block barriers
// after the prologue. Because of ray regeneration a warp has paths of several groups in flight: kGroupOpen slots per
// warp; a new group is only opened in a slot whose previous group has been written out.
constexpr int kGroupPix = 16;
constexpr int kGroupOpen = 8;

// Camera rays of one chunk of a group: `ns` sample indices [s0, s0+ns) x npix pixels, entry q = sl*npix + px, into the warp's
// shared buffer: {origin.xyz, rng} {direction.xyz, px | slot << 4 | frame-in-draw << 8}.
__device__ __forceinline__ void generate_group_rays(const DrawParams& p, float4 (*rays)[2], int lane, uint32_t npix, uint32_t ns,
                                                    uint32_t pix0, uint32_t s0, uint32_t slot)
{
    for (uint32_t q = (uint32_t)lane; q < npix * ns; q += 32)
    {
        const uint32_t sl = npix == (uint32_t)kGroupPix ? q >> 4 : q / npix;
        const uint32_t px = q - sl * npix;
        const RegionPixel g = region_pixel(p, pix0 + px);
        const uint32_t s = s0 + sl, fi = s / (uint32_t)p.spp, ss = s - fi * (uint32_t)p.spp;
        uint32_t rng = pixel_seed((uint32_t)(g.y * p.width + g.x) * (uint32_t)p.spp + ss, (uint32_t)p.frame0 + fi);
        Ray r = fast_camera_ray(p, g.x, g.y, rng);
        rays[q][0] = make_float4(r.orig.x, r.orig.y, r.orig.z, __uint_as_float(rng));
        rays[q][1] = make_float4(r.dir.x, r.dir.y, r.dir.z, __uint_as_float(px | (slot << 4) | (fi << 8)));
    }
}

// The body is shared by k_fast_group (light sampling) and k_fast_group_nolight (DO_LIGHT_SAMPLING 0) below.
template <int KFORM, bool ALLS, int LS>
__device__ __forceinline__ void
fast_group_body(DrawParams p, const unsigned char* __restrict__ blob, SceneBlobLayout L, int count, int nLights,
                uint32_t stagedBytes, uint32_t numGroups, uint32_t S, float wPrev)
{
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ uint64_t bar;
    __shared__ float sW[kMaxFramesPerDraw];
    __shared__ float4 sRays[kQueueThreads / 32][kSlabPix][2];
    __shared__ float4 sAcc[kQueueThreads / 32][kGroupOpen][kGroupPix];
    __shared__ int sRemain[kQueueThreads / 32][kGroupOpen];
    __shared__ uint32_t sGrpPix0[kQueueThreads / 32][kGroupOpen];
    stage_blob(smem, blob, stagedBytes, &bar);
    if (threadIdx.x == 0) { float wp; blend_weights(p, sW, wp); }
    for (int i = threadIdx.x; i < (kQueueThreads / 32) * kGroupOpen * kGroupPix; i += kQueueThreads) (&sAcc[0][0][0])[i] = make_float4(0, 0, 0, 0);
    if (threadIdx.x < (kQueueThreads / 32) * kGroupOpen) (&sRemain[0][0])[threadIdx.x] = 0;
    SceneView sc = make_view<ALLS>(smem, blob, L, stagedBytes, count, nLights);     // ALLS: whole blob staged -> LDS for every section
    const auto hitter = prepare_sweep<KFORM>(sc, smem, L, stagedBytes);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t regionPix = (uint32_t)((long long)p.numRows * p.width);
    const float invSpp = 1.0f / (float)p.spp;
    unsigned rc = 0;

    // warp-uniform cursors: current chunk of rays in sRays, current group
    uint32_t chunkCur = 0, chunkEnd = 0;
    uint32_t sNext = S;                     // next sample index of the current group to generate (== S: group exhausted)
    uint32_t grpPix0 = 0, grpNpix = 0, curSlot = 0, groupsOpened = 0;
    bool exhausted = false;

    // the next chunk of up to 4 sample indices of the current group, opening a new group when it has none left
    auto refill = [&](const DrawParams& p) {
        if (sNext >= S)
        {
            const uint32_t slot = groupsOpened % (uint32_t)kGroupOpen;
            if (sRemain[warp][slot] != 0) return kDealBlocked;     // that slot's group still has paths in flight: trace them first
            uint32_t g = 0;
            if (lane == 0) g = atomicAdd(p.workCounter, 1u);
            g = __shfl_sync(0xffffffffu, g, 0);
            if (g >= numGroups) return kDealExhausted;
            grpPix0 = g * (uint32_t)kGroupPix;
            grpNpix = regionPix - grpPix0 < (uint32_t)kGroupPix ? regionPix - grpPix0 : (uint32_t)kGroupPix;
            curSlot = slot; ++groupsOpened; sNext = 0;
            if (lane == 0) { sRemain[warp][slot] = (int)(grpNpix * S); sGrpPix0[warp][slot] = grpPix0; }
        }
        const uint32_t ns = S - sNext < 4u ? S - sNext : 4u;
        __syncwarp();       // every lane has popped what it needed from the previous chunk
        generate_group_rays(p, sRays[warp], lane, grpNpix, ns, grpPix0, sNext, curSlot);
        __syncwarp();
        chunkCur = 0; chunkEnd = grpNpix * ns; sNext += ns;
        return kDealRefilled;
    };

    QPath st;
    st.active = false;
    for (;;)
    {
        deal_paths(p, st, sRays[warp], chunkCur, chunkEnd, exhausted, lane, refill, [&](uint32_t tag) {
            st.pixOff = tag & 0xffu;                         // px | slot << 4
            st.weight = invSpp * sW[tag >> 8];
        });
        if (!__any_sync(0xffffffffu, st.active)) break;

        bool lastOfGroup = false;
        if (path_step<LS>(sc, st, rc, hitter))
        {
            float* a = reinterpret_cast<float*>(&sAcc[warp][st.pixOff >> 4][st.pixOff & 15u]);
            atomicAdd(a + 0, st.col.x * st.weight);
            atomicAdd(a + 1, st.col.y * st.weight);
            atomicAdd(a + 2, st.col.z * st.weight);
            st.active = false;
            lastOfGroup = atomicSub(&sRemain[warp][st.pixOff >> 4], 1) == 1;
        }
        // ---- a group completed: 16 lanes write its 16 pixels, one coalesced 128-bit store each
        unsigned trig = __ballot_sync(0xffffffffu, lastOfGroup);
        while (trig)
        {
            const int src = __ffs(trig) - 1;
            trig &= trig - 1;
            const uint32_t slot = __shfl_sync(0xffffffffu, st.pixOff >> 4, src);
            const uint32_t pix0 = sGrpPix0[warp][slot];
            const uint32_t npix = regionPix - pix0 < (uint32_t)kGroupPix ? regionPix - pix0 : (uint32_t)kGroupPix;
            if ((uint32_t)lane < npix)
            {
                float* px = p.image + region_pixel(p, pix0 + (uint32_t)lane).off * 4;
                const float4 a = sAcc[warp][slot][lane];
                st_stream_f4(px, blend_prev(p, px, wPrev, a.x, a.y, a.z));
                sAcc[warp][slot][lane] = make_float4(0, 0, 0, 0);
            }
            __syncwarp();
        }
    }
    flush_ray_count(p.rayCounter, rc, lane);
}

template <int MINB, int KFORM, bool ALLS>
__global__ void __launch_bounds__(kQueueThreads, MINB)
k_fast_group(DrawParams p, const unsigned char* __restrict__ blob, SceneBlobLayout L, int count, int nLights,
             uint32_t stagedBytes, uint32_t numGroups, uint32_t S, float wPrev)
{
    fast_group_body<KFORM, ALLS, kLsOn>(p, blob, L, count, nLights, stagedBytes, numGroups, S, wPrev);
}

// DO_LIGHT_SAMPLING 0 twin of k_fast_group (see k_fast_queue_nolight).
template <int MINB, int KFORM, bool ALLS>
__global__ void __launch_bounds__(kQueueThreads, MINB)
k_fast_group_nolight(DrawParams p, const unsigned char* __restrict__ blob, SceneBlobLayout L, int count, int nLights,
                     uint32_t stagedBytes, uint32_t numGroups, uint32_t S, float wPrev)
{
    fast_group_body<KFORM, ALLS, kLsOff>(p, blob, L, count, nLights, stagedBytes, numGroups, S, wPrev);
}

// ---- variant 5------------------------------------------------------------------------------------------------
// "tile queue": the warp-level slab dealing and path state machine of variant 3, but a CTA owns a tile of kTileQPix
// pixels for ALL its samples: radiance is accumulated in shared memory and the finished tile is written ONCE with
// coalesced 128-bit stores (st.global.L1::no_allocate.v4, + 128-bit loads of `prev` when it has weight). The store
// target may be another GPU's memory (CUDA IPC mapping): this is the fused render + gather of the multi-GPU path —
// pixels leave over NVLink tile by tile while the other tiles are still being traced. One block barrier per tile; with
// S = spp x frames >= 16 the per-tile tail is < 1 %, at S = 4 variant 3 is the better choice.
constexpr int kTileQPix = 1024;

template <int MINB, int KFORM>
__global__ void __launch_bounds__(kQueueThreads, MINB)
k_fast_tileq(DrawParams p, const unsigned char* __restrict__ blob, SceneBlobLayout L, int count, int nLights,
             uint32_t stagedBytes, uint32_t numTiles, uint32_t S, float wPrev, uint32_t tileQPix)
{
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ uint64_t bar;
    __shared__ float sW[kMaxFramesPerDraw];
    __shared__ float sAcc[kTileQPix * 3];
    __shared__ float4 sRays[kQueueThreads / 32][kSlabPix][2];   // see k_fast_queue
    __shared__ uint32_t sTile, sSlab;
    stage_blob(smem, blob, stagedBytes, &bar);
    if (threadIdx.x == 0) { float wp; blend_weights(p, sW, wp); }
    for (int i = threadIdx.x; i < kTileQPix * 3; i += kQueueThreads) sAcc[i] = 0.0f;
    SceneView sc = make_view(smem, blob, L, stagedBytes, count, nLights);
    const auto hitter = prepare_sweep<KFORM>(sc, smem, L, stagedBytes);
    const int lane = threadIdx.x & 31;
    const uint32_t regionPix = (uint32_t)((long long)p.numRows * p.width);
    const float invSpp = 1.0f / (float)p.spp;
    unsigned rc = 0;

    for (;;)
    {
        __syncthreads();
        if (threadIdx.x == 0) { sTile = atomicAdd(p.workCounter, 1u); sSlab = 0; }
        __syncthreads();
        const uint32_t tile = sTile;
        if (tile >= numTiles) break;
        const uint32_t tilePix0 = tile * tileQPix;
        const uint32_t tilePix = regionPix - tilePix0 < tileQPix ? regionPix - tilePix0 : tileQPix;
        const uint32_t slabsPerSample = (tilePix + kSlabPix - 1) / kSlabPix;
        const uint32_t tileSlabs = slabsPerSample * S;

        uint32_t slabCur = 0, slabEnd = 0;
        float slabW = 0.0f;
        bool exhausted = false;
        // a slab of the tile from the CTA's counter, tag = pixel index inside the tile
        auto refill = [&](const DrawParams& p) {
            uint32_t slab = 0;
            if (lane == 0) slab = atomicAdd(&sSlab, 1u);
            slab = __shfl_sync(0xffffffffu, slab, 0);
            if (slab >= tileSlabs) return kDealExhausted;
            const uint32_t s = slab / slabsPerSample, g = slab - s * slabsPerSample;   // sample-major inside the tile
            const uint32_t q0 = g * kSlabPix;
            slabEnd = tilePix - q0 < (uint32_t)kSlabPix ? tilePix - q0 : (uint32_t)kSlabPix;
            slabCur = 0;
            const uint32_t pix0 = tilePix0 + q0;
            const int ri0 = (int)(pix0 / (uint32_t)p.width), x0 = (int)(pix0 - (uint32_t)ri0 * (uint32_t)p.width);
            const uint32_t fi = s / (uint32_t)p.spp;
            slabW = invSpp * sW[fi];
            __syncwarp();
            generate_slab_rays(p, sRays[threadIdx.x >> 5], lane, slabEnd, x0, ri0, s - fi * (uint32_t)p.spp, (uint32_t)p.frame0 + fi, (int)q0);
            __syncwarp();
            return kDealRefilled;
        };
        QPath st;
        st.active = false;
        for (;;)
        {
            deal_paths(p, st, sRays[threadIdx.x >> 5], slabCur, slabEnd, exhausted, lane, refill,
                       [&](uint32_t tag) { st.pixOff = tag; st.weight = slabW; });
            if (!__any_sync(0xffffffffu, st.active)) break;
            if (path_step<kLsRuntime>(sc, st, rc, hitter))
            {
                atomicAdd(&sAcc[st.pixOff * 3 + 0], st.col.x * st.weight);
                atomicAdd(&sAcc[st.pixOff * 3 + 1], st.col.y * st.weight);
                atomicAdd(&sAcc[st.pixOff * 3 + 2], st.col.z * st.weight);
                st.active = false;
            }
        }

        // ---- tile finished (the stores may go to a peer GPU's memory)
        __syncthreads();
        write_tile(p, sAcc, tilePix0, tilePix, wPrev, (uint32_t)kQueueThreads);
    }
    flush_ray_count(p.rayCounter, rc, lane);
}

// ---- variant 6 ------------------------------------------------------------------------------------------------
// "block wavefront": the persistent design of the north star taken literally. A CTA keeps kWaveSlots path slots in
// SHARED memory (a QPath and the hit of its last sweep, 8 float4 per slot) and runs every iteration in four phases
// separated by block barriers:
//   sweep     thread i regenerates slot i if it is free (next path of the CTA's chunk) and intersects slot i's
//             ray (path or shadow) against all spheres -> every lane has a ray, no divergence outside pass 2;
//   sort      the slot is classified {miss, lambert, metal, dielectric, shadow-return, terminal} and appended to
//             that type's index list with warp __ballot_sync + prefix popcount (one shared atomic per warp per type);
//   scatter   the lists are cut into 32-entry chunks and dealt to the warps: every warp runs path_step on the stored
//             hits of ONE type, so it takes one branch of Scatter() (Test.cpp:83-193) without divergence; Lambert
//             vertices and returning shadow rays append themselves to the light list;
//   light     lambert_next for every slot on the light list: its next shadow ray or its bounce (explicit light
//             sampling, Test.cpp:96-133).
// So the shading is path_step's, with its lambert_next in a phase of its own: inlined into the scatter phase, where the
// slot's QPath and the chunk walk are live, it made the 64-register instance spill. Radiance leaves through the same
// 128-bit vector reductions as variant 3.
constexpr int kWaveThreads = 256;
constexpr int kWaveSlots = 256;        // one slot per thread
constexpr int kWaveFields = 8;
constexpr int kWaveChunk = 4096;       // paths taken from the global counter at a time
// A slot's fields: the path's {o, rng} {d, state word} {thr, pend} {col, -}; its Lambert vertex's {nextDir, mid}
// {thrAlb, -} {nl, -}; and {t, id} of the hit its last sweep found, with the path's {pixOff, weight}, which regeneration
// writes and a finished path reads.
enum { WF_O = 0, WF_D, WF_THR, WF_COL, WF_NEXT, WF_THRALB, WF_NL, WF_HIT };
enum { WT_MISS = 0, WT_LAMBERT, WT_METAL, WT_DIEL, WT_SHADOW, WT_TERMINAL, WT_COUNT };
// a slot's state word (WF_D.w): bits 0-15 kind (0 path ray, 1 + j shadow ray of light j, kKindFree), bits 16-23 depth,
// bit 24 doMaterialE. The launcher refuses nLights >= kKindFree.
constexpr int kKindFree = 0xffff;
constexpr unsigned kWavePath = 1u << WF_O | 1u << WF_D | 1u << WF_THR | 1u << WF_COL;
constexpr unsigned kWaveVertex = 1u << WF_NEXT | 1u << WF_THRALB | 1u << WF_NL;

// The QPath fields held by the slot's fields in `fields` (bit f: field f); the others are left undefined. Each phase loads
// only what it reads and stores only what it writes: a field loaded and stored back unchanged stays live in a register
// through the shading, and k_fast_wave<4> has none to spare.
__device__ __forceinline__ QPath wave_load(const float4* pool, int slot, unsigned fields)
{
    const float4* f = pool + slot;
    QPath st;
    st.active = true;
    if (fields & 1u << WF_O) { const float4 v = f[WF_O * kWaveSlots]; st.o = v3(v.x, v.y, v.z); st.rng = __float_as_uint(v.w); }
    if (fields & 1u << WF_D)
    {
        const float4 v = f[WF_D * kWaveSlots];
        const int w = __float_as_int(v.w);
        st.d = v3(v.x, v.y, v.z);
        st.kind = w & 0xffff; st.depth = (w >> 16) & 0xff; st.doMaterialE = (w >> 24) & 1;
    }
    if (fields & 1u << WF_THR) { const float4 v = f[WF_THR * kWaveSlots]; st.thr = v3(v.x, v.y, v.z); st.pend = v.w; }
    if (fields & 1u << WF_COL) { const float4 v = f[WF_COL * kWaveSlots]; st.col = v3(v.x, v.y, v.z); }
    if (fields & 1u << WF_NEXT) { const float4 v = f[WF_NEXT * kWaveSlots]; st.nextDir = v3(v.x, v.y, v.z); st.mid = __float_as_int(v.w); }
    if (fields & 1u << WF_THRALB) { const float4 v = f[WF_THRALB * kWaveSlots]; st.thrAlb = v3(v.x, v.y, v.z); }
    if (fields & 1u << WF_NL) { const float4 v = f[WF_NL * kWaveSlots]; st.nl = v3(v.x, v.y, v.z); }
    return st;
}
__device__ __forceinline__ void wave_store(float4* pool, int slot, const QPath& st, unsigned fields)
{
    float4* f = pool + slot;
    if (fields & 1u << WF_O) f[WF_O * kWaveSlots] = make_float4(st.o.x, st.o.y, st.o.z, __uint_as_float(st.rng));
    if (fields & 1u << WF_D)
        f[WF_D * kWaveSlots] = make_float4(st.d.x, st.d.y, st.d.z, __int_as_float(st.kind | st.depth << 16 | (int)st.doMaterialE << 24));
    if (fields & 1u << WF_THR) f[WF_THR * kWaveSlots] = make_float4(st.thr.x, st.thr.y, st.thr.z, st.pend);
    if (fields & 1u << WF_COL) f[WF_COL * kWaveSlots] = make_float4(st.col.x, st.col.y, st.col.z, 0.0f);
    if (fields & 1u << WF_NEXT) f[WF_NEXT * kWaveSlots] = make_float4(st.nextDir.x, st.nextDir.y, st.nextDir.z, __int_as_float(st.mid));
    if (fields & 1u << WF_THRALB) f[WF_THRALB * kWaveSlots] = make_float4(st.thrAlb.x, st.thrAlb.y, st.thrAlb.z, 0.0f);
    if (fields & 1u << WF_NL) f[WF_NL * kWaveSlots] = make_float4(st.nl.x, st.nl.y, st.nl.z, 0.0f);
}
__device__ __forceinline__ void wave_free(float4* pool, int slot) { pool[WF_D * kWaveSlots + slot].w = __int_as_float(kKindFree); }

// The hitter of the scatter phase: the hit the sweep phase stored for the slot.
struct StoredHit
{
    int id;
    float t;
    __device__ __forceinline__ int hit(const SceneView&, V3, V3, float, float, float& tOut) const { tOut = t; return id; }
};

struct WaveArgs
{
    uint32_t totalPaths, S;
    FastDiv divS, divW, divSpp;
};

template <int MINB>
__global__ void __launch_bounds__(kWaveThreads, MINB)
k_fast_wave(DrawParams p, const unsigned char* __restrict__ blob, SceneBlobLayout L, int count, int nLights,
            uint32_t stagedBytes, uint32_t poolOffset, WaveArgs wa)
{
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ uint64_t bar;
    __shared__ float sW[kMaxFramesPerDraw];
    __shared__ uint16_t sList[WT_COUNT][kWaveSlots];
    __shared__ uint16_t sLight[kWaveSlots];
    __shared__ int sCount[WT_COUNT];
    __shared__ int sLightCount;
    __shared__ uint32_t sNextPath, sEndPath;
    __shared__ int sExhausted, sLive;
    stage_blob(smem, blob, stagedBytes, &bar);
    float4* pool = reinterpret_cast<float4*>(smem + poolOffset);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const unsigned ltMask = (1u << lane) - 1u;
    if (tid == 0)
    {
        float wp; blend_weights(p, sW, wp);
        for (int fi = 0; fi < p.numFrames; ++fi) sW[fi] *= 1.0f / (float)p.spp;     // the weight of one path of frame fi
        sNextPath = 0; sEndPath = 0; sExhausted = 0; sLive = 0; sLightCount = 0;
        for (int t = 0; t < WT_COUNT; ++t) sCount[t] = 0;
    }
    wave_free(pool, tid);
    SceneView sc = make_view(smem, blob, L, stagedBytes, count, nLights);
    SerialHitter<false> hitter;
    unsigned rc = 0;
    __syncthreads();

    for (;;)
    {
        // ---- list reset + chunk refill (thread 0 only, between the previous iteration's last barrier and this one)
        if (tid == 0)
        {
            sLightCount = 0;
            for (int t = 0; t < WT_COUNT; ++t) sCount[t] = 0;
            if (!sExhausted && sNextPath >= sEndPath)
            {
                const uint32_t base = atomicAdd(p.workCounter, (unsigned)kWaveChunk);
                if (base >= wa.totalPaths) sExhausted = 1;
                else { sNextPath = base; sEndPath = base + kWaveChunk < wa.totalPaths ? base + kWaveChunk : wa.totalPaths; }
            }
        }
        __syncthreads();

        // ---- phase 1: regenerate own slot if free, then sweep
        int type = -1;
        {
            QPath st = wave_load(pool, tid, 1u << WF_O | 1u << WF_D);
            const unsigned need = __ballot_sync(0xffffffffu, st.kind == kKindFree);
            if (need)
            {
                uint32_t base = 0;
                if (lane == 0) base = atomicAdd(&sNextPath, (uint32_t)__popc(need));
                base = __shfl_sync(0xffffffffu, base, 0);
                const uint32_t idx = base + (uint32_t)__popc(need & ltMask);
                if (st.kind == kKindFree && idx < sEndPath)
                {
                    const uint32_t slab = idx >> 7, q = idx & 127u;
                    const uint32_t mtile = fdiv(slab, wa.divS), s = slab - mtile * wa.S;
                    uint32_t pix = mtile * 128u + q;
                    const uint32_t regionPix = (uint32_t)p.numRows * (uint32_t)p.width;
                    if (pix < regionPix)
                    {
                        const uint32_t ri = fdiv(pix, wa.divW), x = pix - ri * (uint32_t)p.width;
                        const uint32_t fi = fdiv(s, wa.divSpp), ss = s - fi * (uint32_t)p.spp;
                        const int y = p.row0 + (int)ri * p.rowStep;
                        uint32_t rng = pixel_seed((uint32_t)(y * p.width + (int)x) * (uint32_t)p.spp + ss, (uint32_t)p.frame0 + fi);
                        const Ray r = fast_camera_ray(p, (int)x, y, rng);
                        st = QPath{};
                        begin_path(st, r, rng);
                        wave_store(pool, tid, st, kWavePath);
                        float4& h = pool[WF_HIT * kWaveSlots + tid];
                        h.z = __uint_as_float((uint32_t)((p.packed ? (int)ri : y) * p.width + (int)x));    // pixOff
                        h.w = sW[fi];                                                                       // weight
                    }
                }
            }
            if (st.kind != kKindFree)
            {
                float t;
                const int id = hitter.hit(sc, st.o, st.d, TPT_MIN_T, TPT_MAX_T, t);
                pool[WF_HIT * kWaveSlots + tid].x = t;
                pool[WF_HIT * kWaveSlots + tid].y = __int_as_float(id);
                if (st.kind != 0) type = WT_SHADOW;
                else if (id < 0) type = WT_MISS;
                else
                {
                    const int mtype = f_as_i(sc.matA[id < sc.count ? id : sc.count].w);
                    type = st.depth >= TPT_MAX_DEPTH ? WT_TERMINAL : (mtype == kLambert ? WT_LAMBERT : (mtype == kMetal ? WT_METAL : WT_DIEL));
                }
            }
        }
        // ---- phase 2: sort slots by type (ballot + prefix)
#pragma unroll
        for (int T = 0; T < WT_COUNT; ++T)
        {
            const unsigned m = __ballot_sync(0xffffffffu, type == T);
            if (m)
            {
                int base = 0;
                if (lane == 0) base = atomicAdd(&sCount[T], __popc(m));
                base = __shfl_sync(0xffffffffu, base, 0);
                if (type == T) sList[T][base + __popc(m & ltMask)] = (uint16_t)tid;
            }
        }
        __syncthreads();
        const int live = sCount[0] + sCount[1] + sCount[2] + sCount[3] + sCount[4] + sCount[5];
        if (live == 0 && sExhausted) break;

        // ---- phase 3: path_step per type, 32-entry chunks dealt to the warps (path_step counts the ray the sweep traced)
        {
            int chunk = warp;               // chunk ids over the concatenation of the type lists
            int T = 0, first = 0;           // `first` = chunk id of type T's first chunk
            for (;;)
            {
                while (T < WT_COUNT && chunk >= first + ((sCount[T] + 31) >> 5)) { first += (sCount[T] + 31) >> 5; ++T; }
                if (T >= WT_COUNT) break;
                const int k = ((chunk - first) << 5) + lane;
                const bool on = k < sCount[T];
                const int slot = on ? sList[T][k] : 0;
                const bool wantLight = on && (T == WT_LAMBERT || T == WT_SHADOW);     // they go on in phase 4
                if (on)
                {
                    QPath st = wave_load(pool, slot, kWavePath | (T == WT_SHADOW ? 1u << WF_THRALB : 0u));
                    const float4* h = pool + WF_HIT * kWaveSlots + slot;
                    if (path_step<kLsRuntime, 1, false>(sc, st, rc, StoredHit{__float_as_int(h->y), h->x}))
                    {
                        const uint32_t pixOff = __float_as_uint(h->z);
                        const float w = h->w;
                        red_add_f4(p.image + (size_t)pixOff * 4, st.col.x * w, st.col.y * w, st.col.z * w);
                        wave_free(pool, slot);
                    }
                    else wave_store(pool, slot, st, kWavePath | (T == WT_LAMBERT ? kWaveVertex : 0u));
                }
                const unsigned lm = __ballot_sync(0xffffffffu, wantLight);
                if (lm)
                {
                    int base = 0;
                    if (lane == 0) base = atomicAdd(&sLightCount, __popc(lm));
                    base = __shfl_sync(0xffffffffu, base, 0);
                    if (wantLight) sLight[base + __popc(lm & ltMask)] = (uint16_t)slot;
                }
                chunk += kWaveThreads / 32;
            }
        }
        __syncthreads();

        // ---- phase 4: lambert_next for Lambert vertices / returning shadow rays (Test.cpp:96-133)
        {
            const int nL = sLightCount;
            for (int k = tid; k < ((nL + 31) & ~31); k += kWaveThreads)
            {
                if (k < nL)
                {
                    const int slot = sLight[k];
                    QPath st = wave_load(pool, slot, kWavePath & ~(1u << WF_COL) | kWaveVertex);
                    lambert_next<kLsRuntime>(sc, st, st.kind);
                    wave_store(pool, slot, st, kWavePath & ~(1u << WF_COL));
                }
            }
        }
        __syncthreads();
    }
    flush_ray_count(p.rayCounter, rc, lane);
}

} // namespace tpt
#include "tpt_refgpu.cuh"
namespace tpt {

// ---- sweep form (KFORM, see prepare_sweep) per kernel family -------------------------------------------------------
// Inputs: sc.kformMode, the fast_kform option (0 reference form, 1 expanded form, 2 pair array where it fits), and
// sc.kformOk, the scene passes the expanded form's accuracy gate (tpt_set_scene; never with fast_kform 0).
// The families differ on purpose:
//   slab queue (variants 3/4/9, and tpt_draw's automatic variant): the pair array where the blob, the pairs and 24
//     camera-ray buffers fit in 200 KB, else form 1; pick_queue turns form 2 into form 4 (pair array in the kernel
//     parameter) for scenes of at most 64 padded spheres when fast_kform is 2 or 4; the form-4 instances run form 5 (the
//     half-precision pass 1) when fast_kform is 2 and build_half_pairs accepted the scene. A scene that fails the gate runs the
//     conservative form 3 when fast_kform is 2 or 3 and the pairs fit, else form 0.
//   group and tile queue (variants 8 and 5): the pair array up to 1024 spheres, else form 1. No form 3: a scene that
//     fails the gate runs form 0.
//   reference-GPU native instance: form 2 under the group rule but only when fast_kform is 2, else its own
//     reference-form setup (RgSetupPlain); never form 1 or 3.
static uint32_t simd_count(const SceneDev& sc) { return (uint32_t)((sc.count + 3) / 4 * 4); }
// bytes of the pair array a sweep form keeps in shared memory (forms 2 and 3; form 4 has it in the kernel parameter)
static uint32_t smem_pair_bytes(const SceneDev& sc, int kform) { return kform == 2 || kform == 3 ? simd_count(sc) * 16 : 0; }

int fast_queue_kform(const SceneDev& sc)
{
    const bool pairsFit = fast_smem(sc.stagedBytes, simd_count(sc) * 16, 24 * 2048).bytes <= 200 * 1024;
    if (sc.kformMode == 0) return 0;
    if (sc.kformOk) return (sc.kformMode == 1 || !pairsFit) ? 1 : 2;
    return (sc.kformMode >= 2 && pairsFit) ? 3 : 0;
}
static int fast_group_kform(const SceneDev& sc)
{
    return !sc.kformOk ? 0 : (sc.kformMode == 1 || simd_count(sc) > 1024 ? 1 : 2);
}
static int refgpu_fast_kform(const SceneDev& sc)
{
    return sc.kformOk && sc.kformMode >= 2 && simd_count(sc) <= 1024 ? 2 : 0;
}

// Runtime sweep form -> kernel instance: f(std::integral_constant<int, kform>) for kform in [1, KMAX], f(<0>) otherwise.
template <int KMAX, class F>
static auto for_kform(int kform, F f)
{
    if constexpr (KMAX == 0) return f(std::integral_constant<int, 0>());
    else return kform == KMAX ? f(std::integral_constant<int, KMAX>()) : for_kform<KMAX - 1>(kform, f);
}
// the light-sampling instance, or its DO_LIGHT_SAMPLING 0 twin where the scene turns light sampling off
template <class Kernel>
static Kernel light_twin(const SceneDev& sc, Kernel on, Kernel off) { return (sc.layout.flags & kSceneNoLightSampling) ? off : on; }

// The reference-GPU-compatible mode's native instance sweeps like the fast mode: expanded form on the pair array.
struct RgSetupK2
{
    using Hitter = FastHitterK2;
    static constexpr int kMinBlocks = 6;
    static size_t dyn_smem(const SceneDev& sc) { return fast_smem(sc.stagedBytes, simd_count(sc) * 16).bytes; }
    static __device__ __forceinline__ Hitter prepare(SceneView& sc, unsigned char* smem, const SceneBlobLayout& L, uint32_t stagedBytes)
    {
        return prepare_sweep<2>(sc, smem, L, stagedBytes);   // padded spheres get K = 1e30: never candidates (ComputeShader.hlsl:134)
    }
};

cudaError_t launch_refgpu_fast(const DrawParams& p, const SceneDev& sc, int numSMs, cudaStream_t stream)
{
    if (refgpu_fast_kform(sc) == 2) return launch_refgpu_t<false, RgSetupK2>(p, sc, numSMs, stream);
    return launch_refgpu_t<false>(p, sc, numSMs, stream);
}

float prev_weight(int frame0, int numFrames, unsigned flags)
{
    float w = 1.0f;
    for (int f = 0; f < numFrames; ++f) w *= lerp_fac(frame0 + f, flags);
    return w;
}

using QueueKernel = decltype(&k_fast_queue<128, TPT_QUEUE_MINB, 0>);
// SRC: the camera-ray family (k_fast_queue), tpt_trace_rays' (k_fast_rays) or tpt_draw_samples' (k_fast_samples, MOMENTS
// selecting the instance that also adds squares)
template <int SRC, bool MOMENTS, int THREADS, int MINB, int KFORM>
static QueueKernel queue_instance(const SceneDev& sc)
{
    if constexpr (SRC == kSrcRays) return light_twin(sc, k_fast_rays<THREADS, MINB, KFORM>, k_fast_rays_nolight<THREADS, MINB, KFORM>);
    else if constexpr (SRC == kSrcPixels)
        return light_twin(sc, k_fast_samples<THREADS, MINB, KFORM, MOMENTS>, k_fast_samples_nolight<THREADS, MINB, KFORM, MOMENTS>);
    else return light_twin(sc, k_fast_queue<THREADS, MINB, KFORM>, k_fast_queue_nolight<THREADS, MINB, KFORM>);
}
template <int SRC, bool MOMENTS, int THREADS, int MINB>
static QueueKernel queue_kernel(const SceneDev& sc, int kform)
{
    return for_kform<3>(kform, [&](auto K) { return queue_instance<SRC, MOMENTS, THREADS, MINB, decltype(K)::value>(sc); });
}

struct QueuePick
{
    QueueKernel kern;
    int threads, kform;
};
// The slab-queue instance for `samples` samples of each of `regionPix` pixels, rays or list entries (variants 3/4/9;
// tpt_trace_rays and tpt_draw_samples take variant 3's choice). Small scenes: 128-thread CTAs, 6 (variant 4: 7, at 72 registers) per SM; scenes whose arrays
// fill most of an SM's shared memory: ONE 768-thread CTA per SM (24 warps share one copy of the geometry instead of 2 CTAs
// x 4 warps with a copy each). Long launches (many slabs per warp) run 8 CTAs of 64 registers per SM instead of 6 of 80
// (the same rule for form 4: at 720p x 4 spp its 8-CTA instance is 3 % slower than the 6-CTA one);
// short ones keep 6, where a warp only gets ~12 slabs and the drain of the last ones weighs more with more warps. Variant
// 9 forces the 8-CTA instance (A/B runs). While an environment is set the 6-CTA instances run instead (the 8-CTA ones
// have no lookup).
template <int SRC, bool MOMENTS = false>
static QueuePick pick_queue(const SceneDev& sc, int variant, long long regionPix, long long samples, int numSMs)
{
    QueuePick q;
    q.kform = fast_queue_kform(sc);
    // the environment-sampling, texture and media instances sweep in the reference form (env_mode, tex_mode)
    const bool refInstances = (sc.layout.flags & kSceneRefForm) != 0;
    if (refInstances) q.kform = 0;
    // the pair array of a scene of at most 64 padded spheres goes in the kernel parameter (form 4), except for variant 4,
    // with "fast_kform" 3 and for tpt_draw_samples' pixel lists (not measured with form 4; they keep form 2). The same
    // instances run form 5 (the half-precision pass 1) when the parameter says so (sc.pairs.half, begin_call).
    if (q.kform == 2 && (sc.kformMode == 2 || sc.kformMode == 4) && simd_count(sc) <= (uint32_t)kParamPairSpheres &&
        SRC != kSrcPixels && !(SRC == kSrcCamera && variant == 4))
        q.kform = 4;
    const bool big = fast_smem(sc.stagedBytes, smem_pair_bytes(sc, q.kform), 4 * 2048).bytes > 36 * 1024 ||
                     sc.stagedBytes != sc.layout.totalBytes;
    const long long slabsPerWarp = ((regionPix + kSlabPix - 1) / kSlabPix) * samples / ((long long)numSMs * 32);
    // the 8-CTA instances have no environment lookup (at 64 registers it made them spill) and no texture lookup: with
    // either set, the 6-CTA ones run
    const bool eight = !(sc.layout.flags & (kSceneEnvironment | kSceneAnyTextures)) && (variant == 9 || (variant == 3 && slabsPerWarp >= 48));
    q.threads = big ? TPT_BIG_THREADS : 128;
    if (big) q.kern = queue_kernel<SRC, MOMENTS, TPT_BIG_THREADS, 1>(sc, q.kform);
    else if (q.kform == 4)
    {
        if constexpr (SRC != kSrcPixels)
            q.kern = eight ? queue_instance<SRC, MOMENTS, 128, 8, 4>(sc) : queue_instance<SRC, MOMENTS, 128, 6, 4>(sc);
    }
    else if (q.kform == 2 && eight) q.kern = queue_instance<SRC, MOMENTS, 128, 8, 2>(sc);
    else if (SRC == kSrcCamera && variant == 4) q.kern = queue_kernel<kSrcCamera, false, 128, 7>(sc, q.kform);
    else q.kern = queue_kernel<SRC, MOMENTS, 128, TPT_QUEUE_MINB>(sc, q.kform);
    return q;
}

// regionPix: pixels of the draw's region, tpt_trace_rays' ray count or the length of tpt_draw_samples' or
// tpt_trace_samples' list. The accumulation buffer is prepared first: a draw's region blended by the weight of `prev`
// (k_prepare_image), caller rays' float4 outputs zeroed; tpt_draw_samples and tpt_trace_samples (p.sums) add to the
// caller's sums as they are.
template <int SRC>
static cudaError_t launch_queue(const QueuePick& q, long long regionPix, const DrawParams& p, const SceneDev& sc, int numSMs,
                                cudaStream_t stream, unsigned int* bandDone, int numBands, unsigned int* bandExpected)
{
    const QueueKernel kern = q.kern;
    const int threads = q.threads;
    const FastSmem lay = fast_smem(sc.stagedBytes, smem_pair_bytes(sc, q.kform), (uint32_t)(threads / 32) * kSlabPix * 32, true);
    const uint32_t S = (uint32_t)(p.spp * p.numFrames);
    const long long slabs = ((regionPix + kSlabPix - 1) / kSlabPix) * S;
    if (slabs > 0x7fffffffLL) return cudaErrorInvalidValue;
    long long grid = 0;
    cudaError_t e = persistent_grid(kern, threads, lay.bytes, numSMs, (slabs + threads / 32 - 1) / (threads / 32), p, stream, grid);
    if (e != cudaSuccess) return e;
    if constexpr (SRC == kSrcRays)
    {
        if (!p.sums) e = cudaMemsetAsync(p.image, 0, (size_t)regionPix * 16, stream);
    }
    else if constexpr (SRC == kSrcCamera)
    {
        note_launch();
        k_prepare_image<<<(unsigned)((regionPix + 255) / 256), 256, 0, stream>>>(p, prev_weight(p.frame0, p.numFrames, p.flags));
        e = cudaGetLastError();
    }
    if (e != cudaSuccess) return e;
    // optional progress bands (host-buffer draws): band b = macro-tiles [b*mpb, (b+1)*mpb)
    const uint32_t mtiles = (uint32_t)((regionPix + kSlabPix - 1) / kSlabPix);
    uint32_t mpb = 0;
    if (bandDone && numBands > 0)
    {
        mpb = (mtiles + (uint32_t)numBands - 1) / (uint32_t)numBands;
        for (int b = 0; b < numBands; ++b)
        {
            const long long p0 = (long long)b * mpb * kSlabPix, p1 = (long long)(b + 1) * mpb * kSlabPix;
            const long long px = (p1 < regionPix ? p1 : regionPix) - (p0 < regionPix ? p0 : regionPix);
            bandExpected[b] = (unsigned int)(px * S);
        }
    }
#if TPT_TRACE_WARPS
    static unsigned long long* dTrace = nullptr;
    const size_t traceWords = (size_t)grid * (threads / 32) * 8;
    if (getenv("TPT_TRACE_FILE"))
    {
        if (!dTrace) { cudaMalloc(&dTrace, (size_t)132 * 16 * 32 * 8 * 8); cudaMemcpyToSymbol(g_warpTrace, &dTrace, sizeof(dTrace)); }
        cudaMemsetAsync(dTrace, 0, traceWords * 8, stream);
    }
#endif
    e = launch_trace(kern, (unsigned)grid, threads, lay.bytes, stream, p, sc.blob, sc.layout, sc.count, sc.nLights, sc.stagedBytes,
                     (uint32_t)slabs, S, mpb ? bandDone : nullptr, mpb ? mpb : 1u, lay.buffers, sc.pairs);
#if TPT_TRACE_WARPS
    if (const char* tf = getenv("TPT_TRACE_FILE"))
    {
        cudaStreamSynchronize(stream);
        std::vector<unsigned long long> h(traceWords);
        cudaMemcpy(h.data(), dTrace, traceWords * 8, cudaMemcpyDeviceToHost);
        if (FILE* f = fopen(tf, "wb")) { fwrite(h.data(), 8, traceWords, f); fclose(f); }     // the last traced launch wins
    }
#endif
    return e;
}

// Diagnostic (tpt_debug_hit): the nearest-hit query of one sweep form on caller-supplied rays, staged exactly like
// k_fast_queue stages it. The parity tests compare forms ray by ray with it (ids and distance bits).
template <int KFORM>
__global__ void __launch_bounds__(256)
k_debug_hit(const unsigned char* __restrict__ blob, SceneBlobLayout L, int count, int nLights, uint32_t stagedBytes,
            const float* __restrict__ rays, int* __restrict__ outId, float* __restrict__ outT, long long n,
            const __grid_constant__ ParamPairs pp)
{
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ uint64_t bar;
    stage_blob(smem, blob, stagedBytes, &bar);
    SceneView sc = make_view(smem, blob, L, stagedBytes, count, nLights);
    const auto hitter = prepare_sweep<KFORM>(sc, smem, L, stagedBytes, &pp);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    {
        const V3 o{rays[6 * i], rays[6 * i + 1], rays[6 * i + 2]}, d{rays[6 * i + 3], rays[6 * i + 4], rays[6 * i + 5]};
        float t = TPT_MAX_T;
        outId[i] = hitter.hit(sc, o, d, TPT_MIN_T, TPT_MAX_T, t);
        outT[i] = t;
    }
}

cudaError_t launch_debug_hit(const SceneDev& sc, int kform, const float* dRays, int* dId, float* dT, long long n, int numSMs, cudaStream_t stream)
{
    auto kern = for_kform<4>(kform == 5 ? 4 : kform, [](auto K) { return k_debug_hit<decltype(K)::value>; });
    // the blob padded to 128 B even without a pair array: the end of the (possibly empty) pair array
    const size_t dyn = fast_smem(sc.stagedBytes, smem_pair_bytes(sc, kform)).buffers;
    if (dyn > 200 * 1024) return cudaErrorInvalidValue;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn);
    if (e != cudaSuccess) return e;
    ParamPairs pp = sc.pairs;
    pp.half = kform == 5;
    kern<<<numSMs, 256, dyn, stream>>>(sc.blob, sc.layout, sc.count, sc.nLights, sc.stagedBytes, dRays, dId, dT, n, pp);
    return cudaGetLastError();
}

// The index check of a caller list of n entries before the trace kernel that reads *badPixel: k_check_pixels against
// [0, limit).
cudaError_t launch_list_check(const int* list, long long n, long long limit, unsigned long long* badPixel, int numSMs,
                              cudaStream_t stream)
{
    cudaError_t e = cudaMemsetAsync(badPixel, 0xff, sizeof(unsigned long long), stream);
    if (e != cudaSuccess) return e;
    const long long blocks = (n + 255) / 256;
    note_launch();
    k_check_pixels<<<(unsigned)(blocks < 4LL * numSMs ? blocks : 4LL * numSMs), 256, 0, stream>>>(list, n, limit, badPixel);
    return cudaGetLastError();
}

cudaError_t launch_fast_rays(const DrawParams& p, const SceneDev& sc, long long numIn, unsigned long long* badPixel, int numSMs,
                             cudaStream_t stream)
{
    DrawParams q = p;
    if (p.entries)
    {
        if (cudaError_t e = launch_list_check(p.entries, p.numRays, numIn, badPixel, numSMs, stream)) return e;
        q.badPixel = badPixel;
    }
    const QueuePick k = pick_queue<kSrcRays>(sc, 3, p.numRays, p.spp, numSMs);
    return launch_queue<kSrcRays>(k, p.numRays, q, sc, numSMs, stream, nullptr, 0, nullptr);
}

cudaError_t launch_fast_samples(const DrawParams& p, const SceneDev& sc, unsigned long long* badPixel, int numSMs,
                                cudaStream_t stream)
{
    if (p.pixels)
        if (cudaError_t e = launch_list_check(p.pixels, p.numRays, (long long)p.width * p.height, badPixel, numSMs, stream))
            return e;
    DrawParams q = p;
    q.badPixel = badPixel;
    const QueuePick k = p.sq4 ? pick_queue<kSrcPixels, true>(sc, 3, p.numRays, p.spp, numSMs)
                              : pick_queue<kSrcPixels, false>(sc, 3, p.numRays, p.spp, numSMs);
    return launch_queue<kSrcPixels>(k, p.numRays, q, sc, numSMs, stream, nullptr, 0, nullptr);
}

// ---- first-hit AOVs (tpt_draw_aovs, tpt_trace_aovs) ----------------------------------------------------------------
// One nearest-hit sweep per sample and no shading: per pixel (or caller ray) albedo4 = (albedo.rgb, coverage) and
// normal4 = (normal.xyz, depth) of the primary hits, ids = the sphere id of sample 0. Persistent CTAs stage the scene as
// k_debug_hit does (blob + pair array, no ray buffers: every scene the slab queue stages fits); a warp pulls 32
// consecutive pixels or rays from the work counter and each lane owns one of them for all its samples, so every lane does
// exactly one sweep per sample and the warp stays converged. A pixel's result depends on its own samples only: the output
// is bitwise the same for any grid size or row sharding.
// RAYS = false: the draw's pixels y = row0 + i * rowStep; sample s of frame f uses the fast draw's camera ray
//   (pixel_seed((y * width + x) * spp + s, f), fast_camera_ray), frames blended like the image with prev * wPrev.
// RAYS = true: p.numRays caller rays {o.xyz, d.xyz}, loaded and normalised as load_slab_rays does; untraceable rays give
//   zeros and id -1 and are not counted.
constexpr int kAovThreads = 256, kAovMinBlocks = 3;     // <= 85 registers: three CTAs (24 warps) per SM for scenes that leave the shared memory to them

struct AovSample { V3 albedo, normal; float cov, t; };

template <class Hitter>
__device__ __forceinline__ int aov_sample(const SceneView& sc, const Hitter& hitter, V3 o, V3 d, AovSample& a)
{
    float t = TPT_MAX_T;
    const int id = hitter.hit(sc, o, d, TPT_MIN_T, TPT_MAX_T, t);
    if (id < 0) { a.albedo = v3(0, 0, 0); a.normal = v3(0, 0, 0); a.cov = 0.0f; a.t = 0.0f; return id; }
    const Q4 s = ld_sph(sc, id);
    const V3 pos = o + d * t;
    a.normal = (pos - v3(s.x, s.y, s.z)) * sc.invRadius[id];     // path_step's normal: not flipped, not renormalised
    const Q4 m = sc.matA[id < sc.count ? id : sc.count];         // a padded sphere (form 0) has the all-zero material
    a.albedo = v3(m.x, m.y, m.z);
    // the textured albedo for every material type (this kernel is not on a draw's path: a runtime branch is enough)
    if (sc.flags & kSceneTextures) a.albedo = sphere_texture(sc.tex, id, a.albedo, a.normal);
    a.cov = 1.0f; a.t = t;
    return id;
}

template <bool RAYS, int KFORM>
__global__ void __launch_bounds__(kAovThreads, kAovMinBlocks)
k_fast_aov(DrawParams p, const unsigned char* __restrict__ blob, SceneBlobLayout L, int count, int nLights, uint32_t stagedBytes,
           uint32_t numChunks, float wPrev, float* __restrict__ albedo4, float* __restrict__ normal4, int* __restrict__ ids)
{
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ uint64_t bar;
    __shared__ float sW[kMaxFramesPerDraw];
    stage_blob(smem, blob, stagedBytes, &bar);
    if (!RAYS && threadIdx.x == 0) { float wp; blend_weights(p, sW, wp); }
    SceneView sc = make_view(smem, blob, L, stagedBytes, count, nLights);
    const auto hitter = prepare_sweep<KFORM>(sc, smem, L, stagedBytes);     // (its barrier also publishes sW)
    const int lane = threadIdx.x & 31;
    const uint32_t n = RAYS ? p.numRays : (uint32_t)p.numRows * (uint32_t)p.width;
    const float invSpp = 1.0f / (float)p.spp;
    unsigned rc = 0;
    for (;;)
    {
        uint32_t chunk = 0;
        if (lane == 0) chunk = atomicAdd(p.workCounter, 1u);
        chunk = __shfl_sync(0xffffffffu, chunk, 0);
        if (chunk >= numChunks) break;
        const uint32_t i = chunk * 32u + (uint32_t)lane;
        if (i >= n) continue;
        AovSample acc{v3(0, 0, 0), v3(0, 0, 0), 0.0f, 0.0f};
        int id0 = -1;
        size_t off = i;
        if constexpr (RAYS)
        {
            const float* r = p.rays + (size_t)i * 6;
            const V3 o = v3(__ldg(r), __ldg(r + 1), __ldg(r + 2));
            const V3 d = M<false>::normalize(v3(__ldg(r + 3), __ldg(r + 4), __ldg(r + 5)));
            const bool ok = isfinite(o.x) && isfinite(o.y) && isfinite(o.z) && isfinite(d.x) && isfinite(d.y) && isfinite(d.z) &&
                            (d.x != 0.0f || d.y != 0.0f || d.z != 0.0f);
            if (ok) { id0 = aov_sample(sc, hitter, o, d, acc); ++rc; }
        }
        else
        {
            const RegionPixel q = region_pixel(p, i);
            const int x = q.x, y = q.y;
            for (int fi = 0; fi < p.numFrames; ++fi)
            {
                AovSample fs{v3(0, 0, 0), v3(0, 0, 0), 0.0f, 0.0f};
                for (int s = 0; s < p.spp; ++s)
                {
                    uint32_t rng = pixel_seed((uint32_t)(y * p.width + x) * (uint32_t)p.spp + (uint32_t)s, (uint32_t)(p.frame0 + fi));
                    const Ray r = fast_camera_ray(p, x, y, rng);
                    AovSample a;
                    const int id = aov_sample(sc, hitter, r.orig, r.dir, a);
                    if (fi == 0 && s == 0) id0 = id;
                    fs.albedo = fs.albedo + a.albedo; fs.normal = fs.normal + a.normal; fs.cov += a.cov; fs.t += a.t;
                }
                rc += (unsigned)p.spp;
                const float w = invSpp * sW[fi];
                acc.albedo = acc.albedo + fs.albedo * w; acc.normal = acc.normal + fs.normal * w;
                acc.cov += fs.cov * w; acc.t += fs.t * w;
            }
            off = q.off;
        }
        float4 va = make_float4(acc.albedo.x, acc.albedo.y, acc.albedo.z, acc.cov);
        float4 vn = make_float4(acc.normal.x, acc.normal.y, acc.normal.z, acc.t);
        // out = prev * wPrev + sum_f w_f mean_f, all four components; a zero weight does not read prev (NaN * 0)
        if (albedo4)
        {
            if (!RAYS && wPrev != 0.0f)
            {
                const float4 q = ld_stream_f4(albedo4 + off * 4);
                va = make_float4(fmaf(q.x, wPrev, va.x), fmaf(q.y, wPrev, va.y), fmaf(q.z, wPrev, va.z), fmaf(q.w, wPrev, va.w));
            }
            *reinterpret_cast<float4*>(albedo4 + off * 4) = va;
        }
        if (normal4)
        {
            if (!RAYS && wPrev != 0.0f)
            {
                const float4 q = ld_stream_f4(normal4 + off * 4);
                vn = make_float4(fmaf(q.x, wPrev, vn.x), fmaf(q.y, wPrev, vn.y), fmaf(q.z, wPrev, vn.z), fmaf(q.w, wPrev, vn.w));
            }
            *reinterpret_cast<float4*>(normal4 + off * 4) = vn;
        }
        if (ids) ids[off] = id0;
    }
    flush_ray_count(p.rayCounter, rc, lane);
}

cudaError_t launch_fast_aovs(const DrawParams& p, const SceneDev& sc, bool rays, float* albedo4, float* normal4, int* ids,
                             int numSMs, cudaStream_t stream)
{
    if (!rays && p.numFrames > kMaxFramesPerDraw) return cudaErrorInvalidValue;
    const int kform = fast_queue_kform(sc);
    auto kern = rays ? for_kform<3>(kform, [](auto K) { return k_fast_aov<true, decltype(K)::value>; })
                     : for_kform<3>(kform, [](auto K) { return k_fast_aov<false, decltype(K)::value>; });
    // [staged blob | pair array (forms 2/3)], nothing behind it
    const size_t dyn = fast_smem(sc.stagedBytes, smem_pair_bytes(sc, kform)).buffers;
    const long long n = rays ? (long long)p.numRays : (long long)p.numRows * p.width;
    const long long chunks = (n + 31) / 32;
    long long grid = 0;
    cudaError_t e = persistent_grid(kern, kAovThreads, dyn, numSMs, (chunks + kAovThreads / 32 - 1) / (kAovThreads / 32), p, stream, grid);
    if (e != cudaSuccess) return e;
    return launch_trace(kern, (unsigned)grid, kAovThreads, dyn, stream, p, sc.blob, sc.layout, sc.count, sc.nLights, sc.stagedBytes,
                        (uint32_t)chunks, rays ? 0.0f : prev_weight(p.frame0, p.numFrames, p.flags), albedo4, normal4, ids);
}

int fast_slab_pixels() { return kSlabPix; }

FastVariantInfo fast_variant_info(int variant)
{
    const bool queue = variant == 3 || variant == 4 || variant == 9;
    return {variant == 8, queue || (variant >= 5 && variant <= 7), queue, variant == 3 || variant == 9};
}

// The block wavefront (variants 6/7) indexes its paths in 31 bits, over whole 128-pixel slabs (tail pixels are skipped),
// and keeps 1 + the light index in 16 bits below kKindFree.
static long long wave_paths(long long regionPix, long long S) { return ((regionPix + 127) / 128) * 128 * S; }
static bool wave_fits(const SceneDev& sc, long long regionPix, long long S)
{
    return wave_paths(regionPix, S) <= 0x7fffffffLL && sc.nLights < kKindFree;
}

// The slab queue (3), always while the environment is sampled, textures are set or the scene has a medium (tpt_draw then
// never stores into mapped host memory),
// except: a draw into mapped host memory runs the group queue (8), which stores its finished pixels
// itself; and where the sweep dwarfs everything else (>= 1024 spheres) and the slab queue cannot run a packed-pair sweep
// (pair array does not fit, or "fast_kform" < 2), the block wavefront that sorts its paths by material before Scatter()
// is faster (4096 spheres, Mray/s: queue packed 443, wavefront 333, queue scalar 312).
int fast_auto_variant(const SceneDev& sc, long long regionPix, int spp, int numFrames, bool zeroCopy)
{
    if (sc.layout.flags & kSceneRefForm) return 3;   // the slab queue alone samples the environment, looks up textures and
                                                    // has media
    if (zeroCopy) return 8;
    const long long S = (long long)spp * (numFrames < kMaxFramesPerDraw ? numFrames : kMaxFramesPerDraw);   // first launch
    return sc.count >= 1024 && fast_queue_kform(sc) < 2 && wave_fits(sc, regionPix, S) ? 7 : 3;
}

cudaError_t launch_fast(const DrawParams& p, const SceneDev& sc, int variant, int numSMs, cudaStream_t stream,
                        unsigned int* bandDone, int numBands, unsigned int* bandExpected)
{
    if (p.numFrames > kMaxFramesPerDraw) return cudaErrorInvalidValue;
    const long long regionPix = (long long)p.numRows * p.width;
    const uint32_t S = (uint32_t)(p.spp * p.numFrames);
    long long grid = 0;
    cudaError_t e;
    if (variant == 0)
    {
        e = cudaFuncSetAttribute(k_fast_mega, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sc.stagedBytes);
        if (e != cudaSuccess) return e;
        const int tilesX = (p.width + 15) / 16, tilesY = (p.numRows + 15) / 16;
        return launch_trace(k_fast_mega, tilesX * tilesY, kFastThreads, sc.stagedBytes, stream, p, sc.blob, sc.layout, sc.count,
                            sc.nLights, sc.stagedBytes);
    }
    if (variant == 1 || variant == 2)
    {
        auto kern = variant == 1 ? k_fast_persistent<2> : k_fast_persistent<3>;
        const int numTiles = (int)((regionPix + kTilePix - 1) / kTilePix);
        e = persistent_grid(kern, kFastThreads, sc.stagedBytes, numSMs, numTiles, p, stream, grid);
        if (e != cudaSuccess) return e;
        return launch_trace(kern, (unsigned)grid, kFastThreads, sc.stagedBytes, stream, p, sc.blob, sc.layout, sc.count, sc.nLights,
                            sc.stagedBytes, numTiles);
    }
    if (variant == 3 || variant == 4 || variant == 9)
    {
        const QueuePick q = pick_queue<kSrcCamera>(sc, variant, regionPix, (long long)p.spp * p.numFrames, numSMs);
        return launch_queue<kSrcCamera>(q, regionPix, p, sc, numSMs, stream, bandDone, numBands, bandExpected);
    }
    if (variant == 8)
    {
        const int kform = fast_group_kform(sc);
        const bool alls = sc.stagedBytes == sc.layout.totalBytes;
        auto kern = for_kform<2>(kform, [&](auto K) {
            constexpr int k = decltype(K)::value;
            return alls ? light_twin(sc, k_fast_group<TPT_QUEUE_MINB, k, true>, k_fast_group_nolight<TPT_QUEUE_MINB, k, true>)
                        : light_twin(sc, k_fast_group<TPT_QUEUE_MINB, k, false>, k_fast_group_nolight<TPT_QUEUE_MINB, k, false>);
        });
        const size_t dyn = fast_smem(sc.stagedBytes, smem_pair_bytes(sc, kform)).bytes;
        const long long groups = (regionPix + kGroupPix - 1) / kGroupPix;
        if (groups > 0x7fffffffLL) return cudaErrorInvalidValue;
        e = persistent_grid(kern, kQueueThreads, dyn, numSMs, (groups + kQueueThreads / 32 - 1) / (kQueueThreads / 32), p, stream, grid);
        if (e != cudaSuccess) return e;
        return launch_trace(kern, (unsigned)grid, kQueueThreads, dyn, stream, p, sc.blob, sc.layout, sc.count, sc.nLights,
                            sc.stagedBytes, (uint32_t)groups, S, prev_weight(p.frame0, p.numFrames, p.flags));
    }
    if (variant == 6 || variant == 7)
    {
        if (!wave_fits(sc, regionPix, S)) return cudaErrorInvalidValue;
        auto kern = variant == 6 ? k_fast_wave<3> : k_fast_wave<4>;
        const FastSmem lay = fast_smem(sc.stagedBytes, 0, kWaveFields * kWaveSlots * 16);
        const long long total = wave_paths(regionPix, S);
        e = persistent_grid(kern, kWaveThreads, lay.bytes, numSMs, (total + kWaveChunk - 1) / kWaveChunk, p, stream, grid);
        if (e != cudaSuccess) return e;
        note_launch();
        k_prepare_image<<<(unsigned)((regionPix + 255) / 256), 256, 0, stream>>>(p, prev_weight(p.frame0, p.numFrames, p.flags));
        e = cudaGetLastError();
        if (e != cudaSuccess) return e;
        WaveArgs wa;
        wa.S = S;
        wa.totalPaths = (uint32_t)total;
        wa.divS = make_fastdiv(wa.S); wa.divW = make_fastdiv((uint32_t)p.width); wa.divSpp = make_fastdiv((uint32_t)p.spp);
        return launch_trace(kern, (unsigned)grid, kWaveThreads, lay.bytes, stream, p, sc.blob, sc.layout, sc.count, sc.nLights,
                            sc.stagedBytes, lay.buffers, wa);
    }
    if (variant == 5)
    {
        const int kform = fast_group_kform(sc);
        auto kern = for_kform<2>(kform, [](auto K) { return k_fast_tileq<6, decltype(K)::value>; });
        const size_t dyn = fast_smem(sc.stagedBytes, smem_pair_bytes(sc, kform)).bytes;
        // the tile size follows from the resident grid, which is clamped to the tiles afterwards
        e = persistent_grid(kern, kQueueThreads, dyn, numSMs, LLONG_MAX, p, stream, grid);
        if (e != cudaSuccess) return e;
        // tile size: >= ~8192 paths per tile keeps the per-tile barrier tail < 1-2 %; then shrink (down to one slab)
        // until there are >= 8 tiles per CTA so the end-of-kernel quantisation stays small on sharded images
        uint32_t tileQPix = (8192 / S + kSlabPix - 1) / kSlabPix * kSlabPix;
        if (tileQPix < (uint32_t)kSlabPix) tileQPix = kSlabPix;
        if (tileQPix > (uint32_t)kTileQPix) tileQPix = kTileQPix;
        while (tileQPix > (uint32_t)kSlabPix && (regionPix + tileQPix - 1) / tileQPix < 8 * grid && tileQPix * S > 2048) tileQPix -= kSlabPix;
        const long long tiles = (regionPix + tileQPix - 1) / tileQPix;
        if (grid > tiles) grid = tiles;
        return launch_trace(kern, (unsigned)grid, kQueueThreads, dyn, stream, p, sc.blob, sc.layout, sc.count, sc.nLights,
                            sc.stagedBytes, (uint32_t)tiles, S, prev_weight(p.frame0, p.numFrames, p.flags), tileQPix);
    }
    return cudaErrorInvalidValue;
}

} // namespace tpt
