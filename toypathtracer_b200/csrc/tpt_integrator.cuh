// The per-pixel hot loop of the reference (Camera::GetRay -> Trace -> HitWorld/HitSpheres -> Scatter),
// written once for both arithmetic modes:
//
//   EXACT = true   "replay": every float operation in the order the reference's C++ performs it, no FMA
//                  contraction (the translation unit is compiled with -fmad=false; host_sim with
//                  -ffp-contract=off), IEEE division/sqrt, glibc-faithful sinf/cosf/powf (tpt_libm.cuh), the
//                  reference's RNG stream (one XorShift32 chain per (frame,row), Test.cpp:280) and its
//                  back-to-front colour fold (Test.cpp:216). Output is bit-identical to the reference build.
//   EXACT = false  "fast": same estimator, same samplers, per-path RNG streams, FMA contraction and fast
//                  transcendental intrinsics allowed, colour folded front-to-back.
//
// Reference citations are to /root/reference/Cpp/Source/.
#pragma once
#include "tpt_libm.cuh"
#include "tpt_types.h"

#if defined(__CUDACC__)
#define TPT_D __device__ __forceinline__
#else
#define TPT_D inline
#endif

namespace tpt {

// Maths.h:9, Test.cpp:71-73
#define TPT_PI 3.1415926f
#define TPT_MIN_T 0.001f
#define TPT_MAX_T 1.0e7f
#define TPT_MAX_DEPTH 10
static_assert(TPT_MAX_DEPTH == kRefMaxDepth, "\"max_depth\" defaults to the reference's cap");

// ---- float3 (Maths.h:23-115 SSE semantics, scalar form proven bit-identical in SURVEY §9.2) ----------------
struct V3 { float x, y, z; };
TPT_HD V3 v3(float x, float y, float z) { V3 r; r.x = x; r.y = y; r.z = z; return r; }
TPT_HD V3 operator+(V3 a, V3 b) { return v3(a.x + b.x, a.y + b.y, a.z + b.z); }
TPT_HD V3 operator-(V3 a, V3 b) { return v3(a.x - b.x, a.y - b.y, a.z - b.z); }
TPT_HD V3 operator*(V3 a, V3 b) { return v3(a.x * b.x, a.y * b.y, a.z * b.z); }
TPT_HD V3 operator*(V3 a, float b) { return v3(a.x * b, a.y * b, a.z * b); }
TPT_HD V3 operator*(float a, V3 b) { return v3(a * b.x, a * b.y, a * b.z); }
// Maths.h:85: -a is (0 - a) in the SSE float3 (keeps +0 for +0)
TPT_HD V3 neg(V3 a) { return v3(0.0f - a.x, 0.0f - a.y, 0.0f - a.z); }
// Maths.h:114-115: (x + y) + z
TPT_HD float dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
// Maths.h:98-105
TPT_HD V3 cross(V3 a, V3 b) { return v3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
TPT_HD V3 ld3(const float* p) { return v3(p[0], p[1], p[2]); }

// The glibc restatements are a few hundred instructions each. They are called, not inlined: the exact kernels are
// latency-bound chains whose code has to stay inside the instruction cache (the split kernel ran at a 79 % i-cache hit
// rate with everything inlined), and a call costs a handful of cycles next to ~150 dependent double-precision operations.
#if defined(__CUDACC__)
#define TPT_OUTLINE static __host__ __device__ __noinline__
#else
#define TPT_OUTLINE static inline
#endif
TPT_OUTLINE float exact_sinf(float a) { float r; if (tptlibm::sinf_glibc(a, &r)) return r; return sinf(a); }
TPT_OUTLINE float exact_cosf(float a) { float r; if (tptlibm::cosf_glibc(a, &r)) return r; return cosf(a); }
TPT_OUTLINE float exact_pow5f(float x) { return tptlibm::powf_glibc(x, 5.0f); }
#if defined(__CUDA_ARCH__)
// IEEE sqrt / division expand to ~15 instructions + a slow-path call at every use: one shared copy each
TPT_OUTLINE float exact_sqrtf(float x) { return __fsqrt_rn(x); }
TPT_OUTLINE float exact_divf(float a, float b) { return __fdiv_rn(a, b); }
#endif

// EXACT: 0 = fast arithmetic, 1 = the reference's arithmetic, everything inlined (the latency-critical chains),
// 2 = the reference's arithmetic through the shared out-of-line copies above (the shade warps of the split kernel, whose
// code must stay small: same bits, a call instead of ~15-150 inlined instructions per use).
template <int EXACT> struct M
{
    // IEEE-exact in EXACT mode; approximate reciprocal / rsqrt forms allowed otherwise.
    static TPT_HD float sqrt_(float x)
    {
#if defined(__CUDA_ARCH__)
        if (EXACT == 2) return exact_sqrtf(x);
        if (EXACT) return __fsqrt_rn(x);
        float r;
        asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
        return r;
#else
        return sqrtf(x);
#endif
    }
    static TPT_HD float div_(float a, float b)
    {
#if defined(__CUDA_ARCH__)
        if (EXACT == 2) return exact_divf(a, b);
        return EXACT ? __fdiv_rn(a, b) : __fdividef(a, b);
#else
        return a / b;
#endif
    }
    static TPT_HD float sin_(float a)
    {
        if (EXACT == 2) return exact_sinf(a);
        if (EXACT) { float r; if (tptlibm::sinf_glibc(a, &r)) return r; return sinf(a); }
#if defined(__CUDA_ARCH__)
        return __sinf(a);
#else
        return sinf(a);
#endif
    }
    static TPT_HD float cos_(float a)
    {
        if (EXACT == 2) return exact_cosf(a);
        if (EXACT) { float r; if (tptlibm::cosf_glibc(a, &r)) return r; return cosf(a); }
#if defined(__CUDA_ARCH__)
        return __cosf(a);
#else
        return cosf(a);
#endif
    }
    // powf(x, 5) (Maths.h:331)
    static TPT_HD float pow5_(float x)
    {
        if (EXACT == 2) return exact_pow5f(x);
        if (EXACT) return tptlibm::powf_glibc(x, 5.0f);
        float x2 = x * x;
        return x2 * x2 * x;
    }
    // Maths.h:299-301: normalize(v) = v * (1.0f / sqrtf(dot(v,v)))
    static TPT_HD V3 normalize(V3 v)
    {
#if defined(__CUDA_ARCH__)
        if (!EXACT) return v * rsqrtf(dot(v, v));
#endif
        return v * div_(1.0f, sqrt_(dot(v, v)));
    }
};

// ---- RNG + samplers (Maths.cpp:5-47) ---------------------------------------------------------------------
TPT_HD uint32_t XorShift32(uint32_t& state)
{
    uint32_t x = state;
    x ^= x << 13;
    x ^= x >> 17;
    x ^= x << 15;
    state = x;
    return x;
}
// (x & 0xFFFFFF) / 16777216.0f is exact (24-bit integer times 2^-24)
TPT_HD float RandomFloat01(uint32_t& state) { return (float)(XorShift32(state) & 0xFFFFFF) * (1.0f / 16777216.0f); }

// Maths.cpp:20-28; g++ evaluates float3(R(), R(), 0) right to left (SURVEY §9.6): y = 1st draw, x = 2nd
TPT_HD V3 RandomInUnitDisk(uint32_t& state)
{
    V3 p;
    do
    {
        float y = RandomFloat01(state);
        float x = RandomFloat01(state);
        p = 2.0f * v3(x, y, 0.0f) - v3(1.0f, 1.0f, 0.0f);
    } while (dot(p, p) >= 1.0f);
    return p;
}
// Maths.cpp:30-37; z = 1st draw, y = 2nd, x = 3rd
TPT_HD V3 RandomInUnitSphere(uint32_t& state)
{
    V3 p;
    do
    {
        float z = RandomFloat01(state);
        float y = RandomFloat01(state);
        float x = RandomFloat01(state);
        p = 2.0f * v3(x, y, z) - v3(1.0f, 1.0f, 1.0f);
    } while (dot(p, p) >= 1.0f);
    return p;
}
// Maths.cpp:39-47
TPT_HD float u01(uint32_t x) { return (float)(x & 0xFFFFFF) * (1.0f / 16777216.0f); }   // RandomFloat01 of a raw draw
template <int EXACT> TPT_HD V3 RandomUnitVectorFromDraws(uint32_t x1, uint32_t x2);
template <int EXACT> TPT_HD V3 RandomUnitVector(uint32_t& state)
{
    const uint32_t x1 = XorShift32(state), x2 = XorShift32(state);
    return RandomUnitVectorFromDraws<EXACT>(x1, x2);
}
// Maths.cpp:39-47 on the two raw XorShift32 outputs it consumes (z first, then a)
template <int EXACT> TPT_HD V3 RandomUnitVectorFromDraws(uint32_t x1, uint32_t x2)
{
    float z = u01(x1) * 2.0f - 1.0f;
    float a = u01(x2) * 2.0f * TPT_PI;
    float r = M<EXACT>::sqrt_(1.0f - z * z);
#if defined(__CUDA_ARCH__)
    if (!EXACT)
    {
        float sa, ca;
        __sincosf(a, &sa, &ca);
        return v3(r * ca, r * sa, z);
    }
#endif
    float x = r * M<EXACT>::cos_(a);
    float y = r * M<EXACT>::sin_(a);
    return v3(x, y, z);
}

struct Ray { V3 orig, dir; };

// Maths.h:437-442
template <int EXACT> TPT_HD Ray GetRay(const Camera88& c, float s, float t, uint32_t& state)
{
    V3 rd = c.lensRadius * RandomInUnitDisk(state);
    V3 offset = ld3(c.uu) * rd.x + ld3(c.vv) * rd.y;
    Ray r;
    r.orig = ld3(c.origin) + offset;
    r.dir = M<EXACT>::normalize(ld3(c.lowerLeftCorner) + s * ld3(c.horizontal) + t * ld3(c.vertical) - ld3(c.origin) - offset);
    return r;
}

// ---- HitSpheres (Maths.cpp:50-203) ------------------------------------------------------------------------
// One sphere test, Maths.cpp:97-117 / 171-190. Candidate order is the SSE build's: smaller t wins; on an
// exact tie the lower SIMD lane (id & 3) wins, then the lower id (Maths.cpp:113-117 keeps the first hit per
// lane with a strict '<', Maths.cpp:126-152 picks the lowest lane among equal minima).
template <bool EXACT = true> TPT_HD bool hit_better(float t, int id, float bestT, int bestId)
{
    if (!EXACT) return t < bestT;          // ties have zero measure for independent random rays
    if (t < bestT) return true;
    if (t == bestT && bestId >= 0)
    {
        int l = id & 3, bl = bestId & 3;
        return l < bl || (l == bl && id < bestId);
    }
    return false;
}

template <int EXACT> TPT_HD void test_sphere(const Q4 s, int i, V3 o, V3 d, float tMin, float& bestT, int& bestId)
{
    float coX = s.x - o.x;
    float coY = s.y - o.y;
    float coZ = s.z - o.z;
    float nb = coX * d.x + coY * d.y + coZ * d.z;
    float c = coX * coX + coY * coY + coZ * coZ - s.w;
    float discr = nb * nb - c;
    if (discr > 0.0f)
    {
        float discrSq = M<EXACT>::sqrt_(discr);
        float t = nb - discrSq;
        if (t <= tMin) t = nb + discrSq;
        if (t > tMin && hit_better(t, i, bestT, bestId)) { bestT = t; bestId = i; }
    }
}

// sph[i] = {cx, cy, cz, r^2}. On the device the array always lives in shared memory (staged by TMA): read it
// with ld.shared.v4 (LDS.128; all lanes of a warp read the same address in the sweep -> broadcast).
TPT_HD Q4 ld_sph(const SceneView& sc, int i)
{
#if defined(__CUDA_ARCH__)
    Q4 r;
    asm("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "r"(sc.sphShared + (uint32_t)i * 16u));
    return r;
#else
    return sc.sph[i];
#endif
}

// Maths.cpp:97-102 / 171-176: the discriminant of one ray-sphere pair (shared by both passes below).
// `negc` receives r^2 - |co|^2 (fast form) or -(c) sign-equivalent information: negc < 0  <=>  c > 0 (ray origin
// outside the sphere).
template <bool EXACT> TPT_HD float sphere_discr(const Q4 s, V3 o, V3 d, float& nb, float& negc)
{
    float coX = s.x - o.x;
    float coY = s.y - o.y;
    float coZ = s.z - o.z;
#if defined(__CUDA_ARCH__)
    if (!EXACT)
    {
        // same polynomial, 10 instead of 11 FP32 issue slots: r^2 - |co|^2 folded into one FMA chain
        nb = fmaf(coX, d.x, fmaf(coY, d.y, coZ * d.z));
        negc = fmaf(-coX, coX, fmaf(-coY, coY, fmaf(-coZ, coZ, s.w)));
        return fmaf(nb, nb, negc);
    }
#endif
    nb = coX * d.x + coY * d.y + coZ * d.z;
    float c = coX * coX + coY * coY + coZ * coZ - s.w;
    negc = -c;
    return nb * nb - c;
}
template <bool EXACT> TPT_HD float sphere_discr(const Q4 s, V3 o, V3 d, float& nb)
{
    float negc;
    return sphere_discr<EXACT>(s, o, d, nb, negc);
}

// Every lane sweeps all spheres itself (lane = ray), in two passes per chunk of 32 spheres:
//   pass 1  branch-free, fully unrolled: discriminant of every sphere, sign collected in a 32-bit candidate mask
//           (10 FP32 ops + compare + predicated OR per sphere, independent across spheres);
//   pass 2  only the few spheres whose line the ray crosses (discr > 0): sqrt, root selection, nearest-hit
//           update. Each lane walks ITS OWN candidates, so a warp pays max-over-lanes candidates, not the union.
// Per sphere the arithmetic is exactly test_sphere()'s and the winner is chosen under the same total order, so
// the result is identical to the plain loop (and to Maths.cpp:165-202 + the SSE tie rule).
template <bool EXACT, bool SSETIE = EXACT> struct SerialHitter
{
    TPT_HD int hit(const SceneView& sc, V3 o, V3 d, float tMin, float tMax, float& tOut) const
    {
        float bestT = tMax;
        int bestId = -1;
        for (int base = 0; base < sc.simdCount; base += 32)
        {
            const int n = sc.simdCount - base < 32 ? sc.simdCount - base : 32;   // multiple of 4
#if defined(__CUDA_ARCH__)
            // sign bits of the discriminants, funnel-shifted into one word: after n spheres bit (n-1-k) holds
            // sign(discr_k). Candidates = sign clear (discr > 0, +0 or NaN); pass 2 re-checks discr > 0.
            uint32_t neg = 0;
#pragma unroll
            for (int k = 0; k < 32; k += 4)
            {
                if (k < n)
                {
#pragma unroll
                    for (int j = 0; j < 4; ++j)
                    {
                        // Reject in pass 1 when discr < 0, or when the sphere lies wholly behind the origin:
                        // nb < 0 (centre behind) and c > 0 (origin outside) => both roots <= 0 < tMin. With the
                        // rounded values: discr <= fl(nb^2), so sqrt(discr) <= |nb| and nb + sqrt(discr) <= 0 —
                        // the full test could never accept it, so skipping it changes nothing (exact mode too).
                        float nb, negc;
                        float discr = sphere_discr<EXACT>(ld_sph(sc, base + k + j), o, d, nb, negc);
                        uint32_t rej = __float_as_uint(discr) | (__float_as_uint(nb) & __float_as_uint(negc));
                        neg = __funnelshift_l(rej, neg, 1);
                    }
                }
            }
            uint32_t cand = ~neg & (n == 32 ? 0xffffffffu : ((1u << n) - 1u));
            while (cand)
            {
                const int bit = 31 - __clz((int)cand);     // highest bit first = lowest sphere index first
                cand &= ~(1u << bit);
                const int i = base + (n - 1 - bit);
#else
            uint32_t cand = 0;
            for (int k = 0; k < n; ++k)
            {
                float nb;
                if (sphere_discr<EXACT>(ld_sph(sc, base + k), o, d, nb) > 0.0f) cand |= 1u << k;
            }
            while (cand)
            {
                const int k = __builtin_ctz(cand);
                cand &= cand - 1;
                const int i = base + k;
#endif
                float nb;
                float discr = sphere_discr<EXACT>(ld_sph(sc, i), o, d, nb);
                if (discr > 0.0f)
                {
                    float discrSq = M<EXACT>::sqrt_(discr);
                    float t = nb - discrSq;
                    if (t <= tMin) t = nb + discrSq;
                    if (t > tMin && hit_better<SSETIE>(t, i, bestT, bestId)) { bestT = t; bestId = i; }
                }
            }
        }
        tOut = bestT;
        return bestId;
    }
};

#if defined(__CUDACC__)
// LANES lanes of a warp share one ray: lane `sub` sweeps spheres sub, sub+LANES, ... (a warp-wide SoA sweep
// from shared memory) and the nearest hit is reduced with shuffles under the same total order.
template <int EXACT, int LANES> struct GroupHitter
{
    unsigned mask;
    int sub;
    __device__ __forceinline__ int hit(const SceneView& sc, V3 o, V3 d, float tMin, float tMax, float& tOut) const
    {
        float bestT = tMax;
        int bestId = -1;
        for (int i = sub; i < sc.simdCount; i += LANES) test_sphere<EXACT>(ld_sph(sc, i), i, o, d, tMin, bestT, bestId);
        // Nearest hit over the LANES lanes under the total order (t, id & 3, id) with two hardware warp reductions
        // (REDUX) instead of log2(LANES) shuffle rounds: every candidate t is a positive float (t > tMin > 0, or tMax for
        // "no hit"), so its bit pattern orders like an unsigned integer; among the lanes that hold the minimum, the key
        // (id & 3) << 28 | id picks the SSE lane rule's winner (Maths.cpp:126-152).
        const unsigned tBits = __reduce_min_sync(mask, __float_as_uint(bestT));
        const unsigned key = (__float_as_uint(bestT) == tBits && bestId >= 0) ? (((unsigned)bestId & 3u) << 28) | (unsigned)bestId : 0xffffffffu;
        const unsigned win = __reduce_min_sync(mask, key);
        tOut = __uint_as_float(tBits);
        return win == 0xffffffffu ? -1 : (int)(win & 0x0fffffffu);
    }
};
template <int EXACT> struct GroupHitter<EXACT, 1> : SerialHitter<(EXACT != 0)> { unsigned mask; int sub; };

#endif

// ---- materials ---------------------------------------------------------------------------------------------
struct Mat { V3 albedo, emissive; float roughness, ri; int type; };
TPT_HD int f_as_i(float f) { return (int)tptlibm::f2u(f); }
TPT_HD Mat load_mat(const SceneView& sc, int id)
{
    Q4 a = sc.matA[id], b = sc.matB[id];
    Mat m;
    m.albedo = v3(a.x, a.y, a.z);
    m.type = f_as_i(a.w);
    m.emissive = v3(b.x, b.y, b.z);
    m.roughness = b.w;
    m.ri = sc.matRi[id];
    return m;
}

// Maths.h:310-313
TPT_HD V3 reflect(V3 v, V3 n) { return v - (2.0f * dot(v, n)) * n; }
// Maths.h:315-326
template <int EXACT> TPT_HD bool refract(V3 v, V3 n, float nint, V3& outRefracted)
{
    float dt = dot(v, n);
    float discr = 1.0f - nint * nint * (1.0f - dt * dt);
    if (discr > 0.0f)
    {
        outRefracted = nint * (v - n * dt) - n * M<EXACT>::sqrt_(discr);
        return true;
    }
    return false;
}
// Maths.h:327-332
template <int EXACT> TPT_HD float schlick(float cosine, float ri)
{
    float r0 = M<EXACT>::div_(1.0f - ri, 1.0f + ri);
    r0 = r0 * r0;
    return r0 + (1.0f - r0) * M<EXACT>::pow5_(1.0f - cosine);
}

// Explicit light sampling for one emissive sphere, Test.cpp:102-132. Returns the shadow-ray direction and the
// radiance it carries if the ray reaches the light (the caller shoots the ray).
template <int EXACT>
TPT_HD void sample_light(const LightRec& L, V3 pos, V3 normal, V3 rdir, V3 albedo, uint32_t& state, V3& l, V3& contrib)
{
    V3 sc = v3(L.cx, L.cy, L.cz);
    V3 sw = M<EXACT>::normalize(sc - pos);
    V3 su = M<EXACT>::normalize(cross(fabsf(sw.x) > 0.01f ? v3(0, 1, 0) : v3(1, 0, 0), sw));
    V3 sv = cross(sw, su);
    V3 pc = pos - sc;
    float cosAMax = M<EXACT>::sqrt_(1.0f - M<EXACT>::div_(L.radius * L.radius, dot(pc, pc)));
    float eps1 = RandomFloat01(state), eps2 = RandomFloat01(state);
    float cosA = 1.0f - eps1 + eps1 * cosAMax;
    float sinA = M<EXACT>::sqrt_(1.0f - cosA * cosA);
    float phi = 2.0f * TPT_PI * eps2;
    l = su * (M<EXACT>::cos_(phi) * sinA) + sv * (M<EXACT>::sin_(phi) * sinA) + sw * cosA;
    float omega = 2.0f * TPT_PI * (1.0f - cosAMax);
    V3 nl = dot(normal, rdir) < 0.0f ? normal : neg(normal);
    float d = dot(l, nl);
    float m = (0.0f < d) ? d : 0.0f;                      // std::max(0.0f, d), Test.cpp:131
    contrib = (albedo * v3(L.ex, L.ey, L.ez)) * M<EXACT>::div_(m * omega, TPT_PI);
}

// Test.cpp:83-193 for Metal and Dielectric (Lambert is handled by the callers because of its shadow rays).
// Returns false when the path ends (Metal scattering below the surface, unknown type).
template <int EXACT>
TPT_HD bool scatter_specular(const Mat& mat, V3 rdir, V3 pos, V3 normal, uint32_t& state, V3& attenuation, V3& outDir)
{
    if (mat.type == kMetal) // Test.cpp:137-150
    {
        V3 refl = reflect(rdir, normal);
        V3 rnd = RandomInUnitSphere(state);              // drawn even when roughness == 0
        outDir = M<EXACT>::normalize(refl + mat.roughness * rnd);
        attenuation = mat.albedo;
        return dot(outDir, normal) > 0.0f;
    }
    if (mat.type == kDielectric) // Test.cpp:151-186
    {
        V3 outwardN;
        V3 refl = reflect(rdir, normal);
        float nint;
        attenuation = v3(1, 1, 1);
        V3 refr = v3(0, 0, 0);
        float reflProb;
        float cosine;
        float dn = dot(rdir, normal);
        if (dn > 0.0f)
        {
            outwardN = neg(normal);
            nint = mat.ri;
            cosine = mat.ri * dn;
        }
        else
        {
            outwardN = normal;
            nint = M<EXACT>::div_(1.0f, mat.ri);
            cosine = -dn;
        }
        if (refract<EXACT>(rdir, outwardN, nint, refr)) reflProb = schlick<EXACT>(cosine, mat.ri);
        else reflProb = 1.0f;
        if (RandomFloat01(state) < reflProb) outDir = M<EXACT>::normalize(refl);
        else outDir = M<EXACT>::normalize(refr);
        return true;
    }
    attenuation = v3(1, 0, 1); // Test.cpp:187-191
    return false;
}

// Sky, Test.cpp:224-232 (DO_MITSUBA_COMPARE: constant environment, Test.cpp:226-227)
TPT_HD V3 sky(V3 dir, const SceneView& sc)
{
    if (sc.flags & kSceneMitsuba) return v3(0.15f, 0.21f, 0.3f);
    float t = 0.5f * (dir.y + 1.0f);
    return ((1.0f - t) * v3(1.0f, 1.0f, 1.0f) + t * v3(0.5f, 0.7f, 1.0f)) * 0.3f;
}

// doMaterialE after a Lambert vertex (Test.cpp:209-215): with light sampling the next hit's emission was already counted
// by the shadow rays and is suppressed; with DO_LIGHT_SAMPLING 0 that block is compiled out and every hit adds its
// emission. The light loops need no test of their own: with light sampling off the kernels get nLights = 0.
TPT_HD bool emission_after_lambert(const SceneView& sc) { return (sc.flags & kSceneNoLightSampling) != 0; }

// Test.cpp:195-234 (+ Scatter's Lambert branch, Test.cpp:86-136) for ONE camera ray, reference order.
// The recursion `matE + lightE + attenuation * Trace(...)` (Test.cpp:216) is unrolled with an explicit stack and
// folded back to front so the rounding sequence is the reference's.
template <class Hitter>
TPT_HD V3 trace_exact(const SceneView& sc, Ray r, uint32_t& state, unsigned& rayCount, const Hitter& hitter)
{
    V3 e[TPT_MAX_DEPTH + 1], a[TPT_MAX_DEPTH + 1];
    int n = 0;
    bool doMaterialE = true;
    V3 result;
    for (int depth = 0;; ++depth)
    {
        ++rayCount;
        float t;
        int id = hitter.hit(sc, r.orig, r.dir, TPT_MIN_T, TPT_MAX_T, t);
        if (id < 0) { result = sky(r.dir, sc); break; }
        // Maths.cpp:156-157 / 195-196
        Q4 s = ld_sph(sc, id);
        V3 pos = r.orig + r.dir * t;
        V3 normal = (pos - v3(s.x, s.y, s.z)) * sc.invRadius[id];
        // id >= count: a padded "impossible" sphere was hit; the reference reads s_SphereMats out of bounds
        // there (an all-zero Lambert in its build); entry [count] of the material arrays restates that.
        int mid = id < sc.count ? id : sc.count;
        Mat mat = load_mat(sc, mid);
        V3 matE = mat.emissive;
        if (depth >= TPT_MAX_DEPTH) { result = matE; break; }
        V3 attenuation, lightE = v3(0, 0, 0), outDir;
        if (mat.type == kLambert)
        {
            // Test.cpp:89-92
            V3 target = pos + normal + RandomUnitVector<true>(state);
            outDir = M<true>::normalize(target - pos);
            attenuation = mat.albedo;
            for (int j = 0; j < sc.nLights; ++j) // Test.cpp:96-133
            {
                const LightRec L = sc.lights[j];
                if (L.id == mid) continue; // Test.cpp:100
                V3 l, contrib;
                sample_light<true>(L, pos, normal, r.dir, mat.albedo, state, l, contrib);
                ++rayCount;
                float ts;
                int hid = hitter.hit(sc, pos, l, TPT_MIN_T, TPT_MAX_T, ts);
                if (hid == L.id) lightE = lightE + contrib;
            }
        }
        else if (!scatter_specular<true>(mat, r.dir, pos, normal, state, attenuation, outDir))
        {
            result = matE; // Test.cpp:218-221
            break;
        }
        if (!doMaterialE) matE = v3(0, 0, 0);   // Test.cpp:210
        doMaterialE = (mat.type != kLambert) || emission_after_lambert(sc);  // Test.cpp:214
        e[n] = matE + lightE;
        a[n] = attenuation;
        ++n;
        r.orig = pos;
        r.dir = outDir;
    }
    for (int k = n - 1; k >= 0; --k) result = e[k] + a[k] * result;
    return result;
}

// Test.cpp:272-276
TPT_HD float lerp_fac(int frameCount, unsigned flags)
{
    float lerpFac = M<true>::div_((float)frameCount, (float)(frameCount + 1));
    if (flags & 1u) lerpFac *= 0.9f;      // kFlagAnimate, DO_ANIMATE_SMOOTHING (Config.h:23)
    if (!(flags & 2u)) lerpFac = 0.0f;    // !kFlagProgressive
    return lerpFac;
}

// Test.cpp:280
TPT_HD uint32_t row_seed(int y, int frameCount) { return ((uint32_t)y * 9781u + (uint32_t)frameCount * 6271u) | 1u; }

// One pixel of the exact stream: Test.cpp:283-291 (col already multiplied by 1/spp).
template <class Hitter>
TPT_HD V3 pixel_exact(const SceneView& sc, const Camera88& cam, int x, int y, int spp, float invWidth, float invHeight,
                      uint32_t& state, unsigned& rayCount, const Hitter& hitter)
{
    V3 col = v3(0, 0, 0);
    for (int s = 0; s < spp; s++)
    {
        float u = ((float)x + RandomFloat01(state)) * invWidth;
        float v = ((float)(uint32_t)y + RandomFloat01(state)) * invHeight;
        Ray r = GetRay<true>(cam, u, v, state);
        col = col + trace_exact(sc, r, state, rayCount, hitter);
    }
    return col * M<true>::div_(1.0f, (float)spp);
}

} // namespace tpt

// ---- flat state machine of the exact path (one sphere sweep per step) ------------------------------------------------
// Same arithmetic and the same RNG draw order as pixel_exact()/trace_exact(), restructured so that a chain advances by
// exactly ONE HitSpheres sweep per step() call: with one thread per chain all lanes of a warp then meet at a single
// sweep call site every iteration (path rays and shadow rays alike) instead of diverging between the two call sites
// of the nested-loop form. Used when many (frame,row) chains are batched (tpt_exact.cu, LANES = 1).
namespace tpt {

struct XChain
{
    uint32_t rng;
    int x, s;                 // current pixel, sample index inside the pixel
    V3 pix;                   // sum over the pixel's samples so far (Test.cpp:283-289)
    V3 o, d;                  // ray of the next sweep
    int kind;                 // 0: path ray, 1+j: shadow ray towards light j
    int depth, n;             // Trace() recursion depth, number of stacked vertices
    bool doMaterialE;
    // the Lambert vertex whose lights are being sampled (Test.cpp:86-133)
    V3 pos, normal, rdir, albedo, outDir, lightE, matE, contrib;
    int mid, lightId;
    V3 e[TPT_MAX_DEPTH + 1], a[TPT_MAX_DEPTH + 1];
};

// Test.cpp:286-288: next camera ray of the chain
TPT_HD void xchain_begin_sample(XChain& c, const Camera88& cam, int y, float invWidth, float invHeight)
{
    float u = ((float)c.x + RandomFloat01(c.rng)) * invWidth;
    float v = ((float)(uint32_t)y + RandomFloat01(c.rng)) * invHeight;
    Ray r = GetRay<true>(cam, u, v, c.rng);
    c.o = r.orig; c.d = r.dir;
    c.kind = 0; c.depth = 0; c.n = 0; c.doMaterialE = true;
}

TPT_HD void xchain_begin(XChain& c, const Camera88& cam, int y, int frame, float invWidth, float invHeight)
{
    c.rng = row_seed(y, frame);
    c.x = 0; c.s = 0; c.pix = v3(0, 0, 0);
    xchain_begin_sample(c, cam, y, invWidth, invHeight);
}

// One sweep + the scatter logic that follows it. Returns true when pixel c.x has been completed: `pixelOut` then holds
// col * (1/spp) of that pixel (before the blend) and c.x has advanced; the caller stores it and stops at c.x == width.
template <class Hitter>
TPT_HD bool xchain_step(const SceneView& sc, const Camera88& cam, XChain& c, int y, int spp, int width, float invWidth,
                        float invHeight, unsigned& rayCount, const Hitter& hitter, V3& pixelOut)
{
    ++rayCount;
    float t;
    const int id = hitter.hit(sc, c.o, c.d, TPT_MIN_T, TPT_MAX_T, t);
    bool haveResult = false, nextLight = false;
    V3 result = v3(0, 0, 0);
    int j = 0;
    if (c.kind == 0)
    {
        if (id < 0) { result = sky(c.d, sc); haveResult = true; }
        else
        {
            Q4 s = ld_sph(sc, id);
            V3 pos = c.o + c.d * t;
            V3 normal = (pos - v3(s.x, s.y, s.z)) * sc.invRadius[id];
            const int mid = id < sc.count ? id : sc.count;
            Mat mat = load_mat(sc, mid);
            V3 matE = mat.emissive;
            if (c.depth >= TPT_MAX_DEPTH) { result = matE; haveResult = true; }
            else if (mat.type == kLambert)
            {
                V3 target = pos + normal + RandomUnitVector<true>(c.rng);
                c.outDir = M<true>::normalize(target - pos);
                c.albedo = mat.albedo;
                c.lightE = v3(0, 0, 0);
                c.pos = pos; c.normal = normal; c.rdir = c.d; c.matE = matE; c.mid = mid;
                nextLight = true; j = 0;
            }
            else
            {
                V3 attenuation, outDir;
                if (!scatter_specular<true>(mat, c.d, pos, normal, c.rng, attenuation, outDir)) { result = matE; haveResult = true; }
                else
                {
                    if (!c.doMaterialE) matE = v3(0, 0, 0);
                    c.doMaterialE = true;                       // mat.type != Lambert (Test.cpp:214)
                    c.e[c.n] = matE + v3(0, 0, 0);              // matE + lightE with Scatter's outLightE = 0 (Test.cpp:85)
                    c.a[c.n] = attenuation;
                    ++c.n;
                    c.o = pos; c.d = outDir; ++c.depth;
                }
            }
        }
    }
    else
    {
        if (id == c.lightId) c.lightE = c.lightE + c.contrib;
        nextLight = true; j = c.kind;                           // kind = 1 + (light just traced)
    }
    if (nextLight)
    {
        while (j < sc.nLights && sc.lights[j].id == c.mid) ++j; // Test.cpp:100
        if (j < sc.nLights)
        {
            const LightRec L = sc.lights[j];
            V3 l;
            sample_light<true>(L, c.pos, c.normal, c.rdir, c.albedo, c.rng, l, c.contrib);
            c.o = c.pos; c.d = l; c.kind = 1 + j; c.lightId = L.id;
        }
        else
        {
            V3 matE = c.matE;
            if (!c.doMaterialE) matE = v3(0, 0, 0);             // Test.cpp:210
            c.doMaterialE = emission_after_lambert(sc);         // Test.cpp:214 (Lambert)
            c.e[c.n] = matE + c.lightE;
            c.a[c.n] = c.albedo;
            ++c.n;
            c.o = c.pos; c.d = c.outDir; ++c.depth; c.kind = 0;
        }
    }
    if (!haveResult) return false;
    for (int k = c.n - 1; k >= 0; --k) result = c.e[k] + c.a[k] * result;   // Test.cpp:216, back to front
    c.pix = c.pix + result;
    bool pixelDone = false;
    if (++c.s == spp)
    {
        pixelOut = c.pix * M<true>::div_(1.0f, (float)spp);
        c.pix = v3(0, 0, 0); c.s = 0; ++c.x;
        pixelDone = true;
    }
    if (c.x < width) xchain_begin_sample(c, cam, y, invWidth, invHeight);
    return pixelDone;
}

} // namespace tpt

// ---- split form of the exact path: a PATH stream (geometry + RNG, no colour arithmetic) and a SHADE stream -----------------
// The serial dependency of the reference's per-row RNG chain (Test.cpp:280) runs through ray generation, the sphere sweep
// and the scatter DIRECTION only: which draws a sample consumes never depends on a colour, on a shadow ray's result or
// on the fold of Test.cpp:216. xpath_sample() therefore walks one camera sample with exactly the reference's RNG draw
// order and emits one event per path vertex; xshade_event() consumes the events later (on another warp, tpt_exact.cu
// k_trace_exact_split) and does everything the RNG chain does not wait for: explicit light sampling incl. the shadow
// rays (Test.cpp:96-133; its draws are taken from the state snapshot the event carries, the path stream only skips
// them), emission/attenuation bookkeeping (Test.cpp:207-221) and the back-to-front fold (Test.cpp:216). Same
// arithmetic, same order per quantity => the same bits as trace_exact().
namespace tpt {

enum { XE_LAMBERT = 0, XE_SPEC = 1, XE_END_SKY = 2, XE_END_MATE = 3 };

// One camera sample (Test.cpp:286-288 + Trace). emit(type, mid, a, b, c, rng):
//   XE_LAMBERT  a = pos, b = normal, c = incoming dir, rng = state BEFORE the light-sampling draws
//   XE_SPEC     Metal / Dielectric vertex that scattered (attenuation follows from the material)
//   XE_END_SKY  a = dir of the ray that missed everything           (sample ends)
//   XE_END_MATE depth limit or failed scatter: result = emissive    (sample ends, Test.cpp:218-221)
template <class Hitter, class Emit>
TPT_D void xpath_sample(const SceneView& sc, const Camera88& cam, int x, int y, float invWidth, float invHeight,
                        uint32_t& rng, unsigned& rayCount, const Hitter& hitter, Emit&& emit)
{
    float u = ((float)x + RandomFloat01(rng)) * invWidth;
    float v = ((float)(uint32_t)y + RandomFloat01(rng)) * invHeight;
    Ray r = GetRay<true>(cam, u, v, rng);
    const V3 zero = v3(0, 0, 0);
    for (int depth = 0;; ++depth)
    {
        ++rayCount;
        float t;
        const int id = hitter.hit(sc, r.orig, r.dir, TPT_MIN_T, TPT_MAX_T, t);
        if (id < 0) { emit(XE_END_SKY, 0, r.dir, zero, zero, 0u); return; }
        Q4 s = ld_sph(sc, id);
        V3 pos = r.orig + r.dir * t;
        V3 normal = (pos - v3(s.x, s.y, s.z)) * sc.invRadius[id];
        const int mid = id < sc.count ? id : sc.count;
        if (depth >= TPT_MAX_DEPTH) { emit(XE_END_MATE, mid, zero, zero, zero, 0u); return; }
        Mat mat = load_mat(sc, mid);
        if (mat.type == kLambert)
        {
            V3 target = pos + normal + RandomUnitVector<true>(rng);       // Test.cpp:89-92
            V3 outDir = M<true>::normalize(target - pos);
            const uint32_t rngLights = rng;
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
            for (int j = 0; j < sc.nLights; ++j)                          // Test.cpp:96-122: 2 draws + 1 ray per light
                if (sc.lights[j].id != mid) { XorShift32(rng); XorShift32(rng); ++rayCount; }
            emit(XE_LAMBERT, mid, pos, normal, r.dir, rngLights);
            r.orig = pos; r.dir = outDir;
        }
        else
        {
            V3 attenuation, outDir;
            if (!scatter_specular<true>(mat, r.dir, pos, normal, rng, attenuation, outDir)) { emit(XE_END_MATE, mid, zero, zero, zero, 0u); return; }
            emit(XE_SPEC, mid, zero, zero, zero, 0u);
            r.orig = pos; r.dir = outDir;
        }
    }
}

struct XShade
{
    V3 e[TPT_MAX_DEPTH + 1], a[TPT_MAX_DEPTH + 1];
    int n;
    bool doMaterialE;
};
TPT_HD void xshade_begin(XShade& sh) { sh.n = 0; sh.doMaterialE = true; }

// Consumes one event. lightFn(mid, pos, normal, rdir, albedo, rng) returns the Lambert vertex's lightE (Test.cpp:96-133).
// Returns true when the sample has ended: `result` is then Trace()'s return value for the camera ray.
template <class LightFn>
TPT_D bool xshade_event(const SceneView& sc, XShade& sh, int type, int mid, V3 a, V3 b, V3 c, uint32_t rng, LightFn&& lightFn, V3& result)
{
    if (type == XE_END_SKY) result = sky(a, sc);
    else
    {
        Mat mat = load_mat(sc, mid);
        V3 matE = mat.emissive;
        if (type == XE_END_MATE) result = matE;
        else
        {
            V3 lightE = v3(0, 0, 0), attenuation;
            if (type == XE_LAMBERT)
            {
                attenuation = mat.albedo;
                lightE = lightFn(mid, a, b, c, mat.albedo, rng);
            }
            else attenuation = mat.type == kMetal ? mat.albedo : v3(1, 1, 1);   // Test.cpp:149 / :158
            if (!sh.doMaterialE) matE = v3(0, 0, 0);      // Test.cpp:210
            sh.doMaterialE = (type != XE_LAMBERT) || emission_after_lambert(sc);   // Test.cpp:214
            sh.e[sh.n] = matE + lightE;
            sh.a[sh.n] = attenuation;
            ++sh.n;
            return false;
        }
    }
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
    for (int k = sh.n - 1; k >= 0; --k) result = sh.e[k] + sh.a[k] * result;   // Test.cpp:216, back to front
    return true;
}

// Reference-order light loop for one Lambert vertex with a hitter that traces one ray at a time (host simulation, and the
// semantics the device's grouped version must reproduce).
template <class Hitter>
TPT_D V3 xlights_serial(const SceneView& sc, const Hitter& hitter, int mid, V3 pos, V3 normal, V3 rdir, V3 albedo, uint32_t rng)
{
    V3 lightE = v3(0, 0, 0);
    for (int j = 0; j < sc.nLights; ++j)
    {
        const LightRec L = sc.lights[j];
        if (L.id == mid) continue;
        V3 l, contrib;
        sample_light<true>(L, pos, normal, rdir, albedo, rng, l, contrib);
        float ts;
        if (hitter.hit(sc, pos, l, TPT_MIN_T, TPT_MAX_T, ts) == L.id) lightE = lightE + contrib;
    }
    return lightE;
}

} // namespace tpt
