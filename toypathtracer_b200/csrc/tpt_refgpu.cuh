// TPT_MODE_REFGPU: the estimator of the reference's own GPU back-ends (Cpp/Windows/ComputeShader.hlsl, the Metal port is
// the same), so that results and Mray/s can be compared like for like with the numbers the reference publishes for
// its D3D11/Metal paths (readme.md:64-77). It differs from the CPU path (SURVEY §8a "Divergences") in:
//   * one XorShift32 stream per PIXEL, seeded (x*1973 + y*9277 + frames*26699) | 1      ComputeShader.hlsl:380
//   * analytic disk / sphere samplers instead of rejection loops                        ComputeShader.hlsl:18-35
//   * schlick() saturates its argument                                                  ComputeShader.hlsl:73
//   * at most kMaxDepth = 10 path segments (the CPU path traces 11), no terminal emission  ComputeShader.hlsl:300
//   * colour accumulated front to back (col += curAtten * ..., curAtten *= attenuation) ComputeShader.hlsl:318-319
//   * plain ray-sphere loop: strict t < hitT, no SIMD padding                           ComputeShader.hlsl:130-158
//   * blend = lerp(col, prev, lerpFac), alpha written as 1                              ComputeShader.hlsl:391-392
// This is NOT a port of the shader's kernel structure (one thread per pixel in 8x8 groups, scene copied into
// groupshared by the threads): here the scene arrives by TMA bulk copy, the sweep is the two-pass candidate-mask
// sweep of tpt_integrator.cuh, and persistent CTAs pull pixel slabs from a queue with per-lane pixel regeneration.
//
// EXACT = true  (tpt_exact.cu, -fmad=false): every float op as the shader's source states it, IEEE sqrt/div, the
//               glibc-faithful sinf/cosf/powf — bit-equal to the CPU restatement oracle/refgpu_restate.cpp
//               (that oracle is "parity unpinned": no HLSL/Metal toolchain exists here to run the shader itself).
// EXACT = false (tpt_fast.cu): GPU-native arithmetic like the shader's own (FMA, MUFU sin/cos/rsq/lg2/ex2).
#pragma once
#include "tpt_integrator.cuh"
#include "tpt_device_utils.cuh"
#include "tpt_launch.h"

namespace tpt {

constexpr int kRgSlabPix = 64;
constexpr int kRgThreads = 128;

template <bool EXACT> struct RG
{
    // ComputeShader.hlsl:18-24
    static __device__ __forceinline__ V3 RandomInUnitDisk(uint32_t& state)
    {
        float a = RandomFloat01(state) * 2.0f * 3.1415926f;
        float ca, sa;
        sincos_(a, sa, ca);
        float m = M<EXACT>::sqrt_(RandomFloat01(state));
        return v3(ca * m, sa * m, 0.0f);
    }
    // ComputeShader.hlsl:25-35
    static __device__ __forceinline__ V3 RandomInUnitSphere(uint32_t& state)
    {
        float z = RandomFloat01(state) * 2.0f - 1.0f;
        float t = RandomFloat01(state) * 2.0f * 3.1415926f;
        float r = M<EXACT>::sqrt_(fmaxf(0.0f, 1.0f - z * z));
        float ct, st;
        sincos_(t, st, ct);
        float x = r * ct;
        float y = r * st;
        float m = cbrt_pow(RandomFloat01(state));
        return v3(x * m, y * m, z * m);
    }
    // ComputeShader.hlsl:36-44
    static __device__ __forceinline__ V3 RandomUnitVector(uint32_t& state)
    {
        float z = RandomFloat01(state) * 2.0f - 1.0f;
        float a = RandomFloat01(state) * 2.0f * 3.1415926f;
        float r = M<EXACT>::sqrt_(1.0f - z * z);
        float ca, sa;
        sincos_(a, sa, ca);
        return v3(r * ca, r * sa, z);
    }
    static __device__ __forceinline__ void sincos_(float a, float& s, float& c)
    {
        if (EXACT) { s = M<true>::sin_(a); c = M<true>::cos_(a); }
        else __sincosf(a, &s, &c);
    }
    // pow(x, 1.0 / 3.0), ComputeShader.hlsl:33
    static __device__ __forceinline__ float cbrt_pow(float x)
    {
        if (EXACT) return tptlibm::powf_glibc(x, 1.0f / 3.0f);
        return __powf(x, 1.0f / 3.0f);
    }
    // ComputeShader.hlsl:68-74
    static __device__ __forceinline__ float schlick(float cosine, float ri)
    {
        float r0 = M<EXACT>::div_(1.0f - ri, 1.0f + ri);
        r0 = r0 * r0;
        float x = 1.0f - cosine;
        x = fminf(fmaxf(x, 0.0f), 1.0f);     // saturate (NaN -> 0 like HLSL's saturate)
        return r0 + (1.0f - r0) * M<EXACT>::pow5_(x);
    }
    // ComputeShader.hlsl:121-126
    static __device__ __forceinline__ Ray GetRay(const Camera88& c, float s, float t, uint32_t& state)
    {
        V3 rd = c.lensRadius * RandomInUnitDisk(state);
        V3 offset = ld3(c.uu) * rd.x + ld3(c.vv) * rd.y;
        Ray r;
        r.orig = ld3(c.origin) + offset;
        r.dir = M<EXACT>::normalize(ld3(c.lowerLeftCorner) + s * ld3(c.horizontal) + t * ld3(c.vertical) - ld3(c.origin) - offset);
        return r;
    }
};

// One pixel's state in the persistent kernel: the shader's main() (ComputeShader.hlsl:353-395) as a resumable state
// machine, one sweep per step, so a lane whose pixel is done takes the next pixel of the warp's slab while the others
// keep tracing (ray regeneration at pixel granularity — the RNG stream is per pixel, its samples are serial).
struct RgPixel
{
    V3 o, d;
    V3 col, atten;            // Trace()'s col / curAtten (ComputeShader.hlsl:295-296)
    V3 sum;                   // sum over the pixel's samples so far
    // pending Lambert vertex while its shadow rays are in flight
    V3 pos, nl, albedo, nextDir, lightE, matE, contrib;
    uint32_t rng;
    int x, y;                 // pixel
    uint32_t pixOff;
    int s;                    // sample index
    int frame;                // frame index inside the draw
    int depth, kind, mid;     // kind 0: path ray, 1+j: shadow ray of light j
    bool doMaterialE, active;
};

template <bool EXACT>
__device__ __forceinline__ void rg_begin_sample(const DrawParams& p, RgPixel& st)
{
    float u = ((float)(uint32_t)st.x + RandomFloat01(st.rng)) * p.invWidth;     // ComputeShader.hlsl:383-384
    float v = ((float)(uint32_t)st.y + RandomFloat01(st.rng)) * p.invHeight;
    Ray r = RG<EXACT>::GetRay(p.cam, u, v, st.rng);
    st.o = r.orig; st.d = r.dir;
    st.col = v3(0, 0, 0); st.atten = v3(1, 1, 1);
    st.depth = 0; st.kind = 0; st.doMaterialE = true;
}

template <bool EXACT>
__device__ __forceinline__ void rg_begin_frame(const DrawParams& p, RgPixel& st)
{
    st.rng = ((uint32_t)st.x * 1973u + (uint32_t)st.y * 9277u + (uint32_t)(p.frame0 + st.frame) * 26699u) | 1u;   // :380
    st.s = 0; st.sum = v3(0, 0, 0);
    rg_begin_sample<EXACT>(p, st);
}

// One sweep + what follows it. Returns true when the pixel has finished ALL its frames of this draw.
template <bool EXACT, class Hitter>
__device__ __forceinline__ bool rg_step(const DrawParams& p, const SceneView& sc, RgPixel& st, unsigned& rc, const Hitter& hitter)
{
    float t = TPT_MAX_T;
    int id = -1;
    ++rc;
    id = hitter.hit(sc, st.o, st.d, TPT_MIN_T, TPT_MAX_T, t);
    bool sampleDone = false, wantLight = false;
    int lightFrom = 0;
    if (st.kind == 0)
    {
        if (id < 0)
        {
            float tt = 0.5f * (st.d.y + 1.0f);                                   // ComputeShader.hlsl:336-339
            V3 skyCol = sc.flags & kSceneMitsuba ? v3(0.15f, 0.21f, 0.3f)
                                                 : ((1.0f - tt) * v3(1.0f, 1.0f, 1.0f) + tt * v3(0.5f, 0.7f, 1.0f)) * 0.3f;
            st.col = st.col + st.atten * skyCol;
            sampleDone = true;
        }
        else
        {
            Q4 s = ld_sph(sc, id);
            V3 pos = st.o + st.d * t;
            V3 normal = (pos - v3(s.x, s.y, s.z)) * sc.invRadius[id];
            Mat mat = load_mat(sc, id);
            if (mat.type == kLambert)
            {
                V3 target = pos + normal + RG<EXACT>::RandomUnitVector(st.rng);   // ComputeShader.hlsl:189-191
                st.nextDir = M<EXACT>::normalize(target - pos);
                st.albedo = mat.albedo;
                st.nl = dot(normal, st.d) < 0.0f ? normal : neg(normal);
                st.pos = pos; st.mid = id; st.lightE = v3(0, 0, 0);
                st.matE = mat.emissive;                                           // parked until the vertex's lights are done
                wantLight = true; lightFrom = 0;
            }
            else
            {
                V3 attenuation, outDir;
                bool ok;
                if (mat.type == kMetal)                                           // ComputeShader.hlsl:234-244
                {
                    V3 refl = reflect(st.d, normal);
                    outDir = M<EXACT>::normalize(refl + mat.roughness * RG<EXACT>::RandomInUnitSphere(st.rng));
                    attenuation = mat.albedo;
                    ok = dot(outDir, normal) > 0.0f;
                }
                else if (mat.type == kDielectric)                                 // ComputeShader.hlsl:245-278
                {
                    V3 outwardN, refl = reflect(st.d, normal), refr = v3(0, 0, 0);
                    float nint, reflProb, cosine;
                    attenuation = v3(1, 1, 1);
                    float dn = dot(st.d, normal);
                    if (dn > 0.0f) { outwardN = neg(normal); nint = mat.ri; cosine = mat.ri * dn; }
                    else { outwardN = normal; nint = M<EXACT>::div_(1.0f, mat.ri); cosine = -dn; }
                    if (refract<EXACT>(st.d, outwardN, nint, refr)) reflProb = RG<EXACT>::schlick(cosine, mat.ri);
                    else reflProb = 1.0f;
                    outDir = RandomFloat01(st.rng) < reflProb ? M<EXACT>::normalize(refl) : M<EXACT>::normalize(refr);
                    ok = true;
                }
                else { attenuation = v3(1, 0, 1); outDir = v3(0, 0, 1); ok = false; }
                V3 matE = mat.emissive;
                if (ok)
                {
                    if (!st.doMaterialE) matE = v3(0, 0, 0);                      // ComputeShader.hlsl:314-316
                    st.doMaterialE = true;
                    st.col = st.col + st.atten * (matE + v3(0, 0, 0));
                    st.atten = st.atten * attenuation;
                    st.o = pos; st.d = outDir;
                    if (++st.depth >= TPT_MAX_DEPTH) sampleDone = true;           // loop bound, ComputeShader.hlsl:300
                }
                else { st.col = st.col + st.atten * matE; sampleDone = true; }    // ComputeShader.hlsl:323-326
            }
        }
    }
    else
    {
        const int j = st.kind - 1;
        if (id == sc.lights[j].id) st.lightE = st.lightE + st.contrib;               // ComputeShader.hlsl:226
        wantLight = true; lightFrom = j + 1;
    }
    if (wantLight)
    {
        int j = lightFrom;
        while (j < sc.nLights && sc.lights[j].id == st.mid) ++j;                  // ComputeShader.hlsl:198-199
        if (j < sc.nLights)
        {
            const LightRec L = sc.lights[j];
            V3 scn = v3(L.cx, L.cy, L.cz);
            V3 sw = M<EXACT>::normalize(scn - st.pos);
            V3 su = M<EXACT>::normalize(cross(fabsf(sw.x) > 0.01f ? v3(0, 1, 0) : v3(1, 0, 0), sw));
            V3 sv = cross(sw, su);
            V3 pc = st.pos - scn;
            float cosAMax = M<EXACT>::sqrt_(1.0f - M<EXACT>::div_(L.radius * L.radius, dot(pc, pc)));
            float eps1 = RandomFloat01(st.rng), eps2 = RandomFloat01(st.rng);
            float cosA = 1.0f - eps1 + eps1 * cosAMax;
            float sinA = M<EXACT>::sqrt_(1.0f - cosA * cosA);
            float phi = 2.0f * 3.1415926f * eps2;
            float sp, cp;
            RG<EXACT>::sincos_(phi, sp, cp);
            V3 l = su * cp * sinA + sv * sp * sinA + sw * cosA;                   // ComputeShader.hlsl:213 (left to right)
            float omega = 2.0f * 3.1415926f * (1.0f - cosAMax);
            float dl = dot(l, st.nl);
            float m = fmaxf(0.0f, dl);
            st.contrib = (st.albedo * v3(L.ex, L.ey, L.ez)) * M<EXACT>::div_(m * omega, 3.1415926f);   // :226
            st.o = st.pos; st.d = l; st.kind = 1 + j;
        }
        else
        {
            V3 matE = st.matE;
            if (!st.doMaterialE) matE = v3(0, 0, 0);
            st.doMaterialE = emission_after_lambert(sc);                          // Lambert (DO_LIGHT_SAMPLING 0: kept on)
            st.col = st.col + st.atten * (matE + st.lightE);                      // ComputeShader.hlsl:318-319
            st.atten = st.atten * st.albedo;
            st.o = st.pos; st.d = st.nextDir; st.kind = 0;
            if (++st.depth >= TPT_MAX_DEPTH) sampleDone = true;
        }
    }
    if (!sampleDone) return false;
    st.sum = st.sum + st.col;
    if (++st.s < p.spp) { rg_begin_sample<EXACT>(p, st); return false; }
    // pixel of this frame complete: col *= 1/spp; lerp(col, prev, lerpFac); alpha = 1   (ComputeShader.hlsl:387-392)
    V3 col = st.sum * M<EXACT>::div_(1.0f, (float)p.spp);
    const float lerpFac = lerp_fac(p.frame0 + st.frame, p.flags);
    float4* px = reinterpret_cast<float4*>(p.image) + st.pixOff;
    if (lerpFac != 0.0f)          // lerp(col, prev, 0) == col for every finite prev; a zero weight does not read the buffer
    {
        float4 prev = *px;
        col = v3(col.x + lerpFac * (prev.x - col.x), col.y + lerpFac * (prev.y - col.y), col.z + lerpFac * (prev.z - col.z));
    }
    *px = make_float4(col.x, col.y, col.z, 1.0f);
    if (++st.frame < p.numFrames) { rg_begin_frame<EXACT>(p, st); return false; }
    return true;
}

// How the kernel sweeps: the plain setup uses the two-pass reference-form sweep (strict or native arithmetic); tpt_fast.cu
// adds a setup with the expanded-form pair-array sweep for the native instance.
template <bool EXACT> struct RgSetupPlain
{
    using Hitter = SerialHitter<EXACT, false>;
    static constexpr int kMinBlocks = 1;
    static size_t dyn_smem(const SceneDev& sc) { return sc.stagedBytes; }
    static __device__ __forceinline__ Hitter prepare(SceneView& sc, unsigned char* smem, const SceneBlobLayout& L, uint32_t)
    {
        // the shader loops over sphereCount spheres only (ComputeShader.hlsl:134): the SIMD padding of the CPU path's SoA
        // ("impossible" spheres, Maths.h:381-387) must never be a candidate here -> r^2 = -1e30 makes discr hugely negative
        float4* sph = reinterpret_cast<float4*>(smem + L.offSph);
        for (int i = sc.count + (int)threadIdx.x; i < sc.simdCount; i += blockDim.x) sph[i].w = -1.0e30f;
        __syncthreads();
        asm volatile("" : "+r"(sc.sphShared));      // the sweep's asm loads must not be hoisted above the rewrite
        return Hitter();
    }
};

// Persistent CTAs; every warp pulls slabs of kRgSlabPix pixels from a global counter and deals them to its idle lanes.
template <bool EXACT, class Setup>
__global__ void __launch_bounds__(kRgThreads, Setup::kMinBlocks)
k_refgpu(DrawParams p, const unsigned char* __restrict__ blob, SceneBlobLayout L, int count, int nLights, uint32_t stagedBytes,
         uint32_t numSlabs)
{
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ uint64_t bar;
    stage_blob(smem, blob, stagedBytes, &bar);
    SceneView sc = make_view(smem, blob, L, stagedBytes, count, nLights);
    const typename Setup::Hitter hitter = Setup::prepare(sc, smem, L, stagedBytes);
    const int lane = threadIdx.x & 31;
    const unsigned ltMask = (1u << lane) - 1u;
    const uint32_t regionPix = (uint32_t)((long long)p.numRows * p.width);
    unsigned rc = 0;
    uint32_t slabCur = 0, slabEnd = 0, slabPix0 = 0;
    bool exhausted = false;
    RgPixel st;
    st.active = false;
    for (;;)
    {
        unsigned need = __ballot_sync(0xffffffffu, !st.active);
        while (need && !exhausted)
        {
            if (slabCur >= slabEnd)
            {
                uint32_t slab = 0;
                if (lane == 0) slab = atomicAdd(p.workCounter, 1u);
                slab = __shfl_sync(0xffffffffu, slab, 0);
                if (slab >= numSlabs) { exhausted = true; break; }
                slabPix0 = slab * (uint32_t)kRgSlabPix;
                slabEnd = regionPix - slabPix0 < (uint32_t)kRgSlabPix ? regionPix - slabPix0 : (uint32_t)kRgSlabPix;
                slabCur = 0;
            }
            const uint32_t avail = slabEnd - slabCur;
            const uint32_t rank = (uint32_t)__popc(need & ltMask);
            if (!st.active && rank < avail)
            {
                const uint32_t pix = slabPix0 + slabCur + rank;
                const int ri = (int)(pix / (uint32_t)p.width);
                st.x = (int)(pix - (uint32_t)ri * (uint32_t)p.width);
                st.y = p.row0 + ri * p.rowStep;
                st.pixOff = (uint32_t)((p.packed ? ri : st.y) * p.width + st.x);
                st.frame = 0;
                st.active = true;
                rg_begin_frame<EXACT>(p, st);
            }
            const uint32_t n = (uint32_t)__popc(need);
            slabCur += n < avail ? n : avail;
            need = __ballot_sync(0xffffffffu, !st.active);
        }
        if (!__any_sync(0xffffffffu, st.active)) break;
        if (st.active && rg_step<EXACT>(p, sc, st, rc, hitter)) st.active = false;
    }
    flush_ray_count(p.rayCounter, rc, lane);
}

template <bool EXACT, class Setup = RgSetupPlain<EXACT>>
static cudaError_t launch_refgpu_t(const DrawParams& p, const SceneDev& sc, int numSMs, cudaStream_t stream)
{
    auto kern = k_refgpu<EXACT, Setup>;
    const size_t dyn = Setup::dyn_smem(sc);
    const long long regionPix = (long long)p.numRows * p.width;
    const long long slabs = (regionPix + kRgSlabPix - 1) / kRgSlabPix;
    if (slabs > 0x7fffffffLL) return cudaErrorInvalidValue;
    long long grid = 0;
    cudaError_t e = persistent_grid(kern, kRgThreads, dyn, numSMs, (slabs + kRgThreads / 32 - 1) / (kRgThreads / 32), p, stream, grid);
    if (e != cudaSuccess) return e;
    return launch_trace(kern, (unsigned)grid, kRgThreads, dyn, stream, p, sc.blob, sc.layout, sc.count, sc.nLights, sc.stagedBytes,
                        (uint32_t)slabs);
}

} // namespace tpt
