// Host-side packing of the reference's raw scene export (20 B spheres, 36 B materials, emissive id list)
// into the device blob described in tpt_types.h. Mirrors what UpdateTest does on the CPU path
// (Cpp/Source/Test.cpp:321-339: invRadius, SoA fill with r^2, emissive list) and SpheresSoA's padding to a
// multiple of 4 with "impossible" spheres (Cpp/Source/Maths.h:370-388).
#pragma once
#include "tpt_types.h"
#include "tpt_fog.h"
#include <vector>
#include <string.h>
#include <math.h>

namespace tpt {

#ifdef __CUDACC__
#define TPT_PACK_HD __host__ __device__
#else
#define TPT_PACK_HD
#endif

TPT_PACK_HD inline uint32_t align16(uint32_t x) { return (x + 15u) & ~15u; }

// The media section (tpt_set_media, kSceneMedia) of a blob of `count` spheres follows matRi: (count + 1) Q4
// {sigma_a.rgb, sigma_s}, then (count + 1) floats g, each part padded to 16 B; entry [count] is zero. Its offset, for the
// pack and for the kernels' views.
TPT_PACK_HD inline uint32_t media_offset(uint32_t offMatRi, int count) { return offMatRi + align16((uint32_t)(count + 1) * 4u); }
TPT_PACK_HD inline uint32_t media_bytes(int count) { return align16((uint32_t)(count + 1) * 16u) + align16((uint32_t)(count + 1) * 4u); }
// The fog section (tpt_set_fog, kSceneFog), kFogBytes, follows the media section where the blob has one, else matRi.
TPT_PACK_HD inline uint32_t fog_offset(uint32_t offMatRi, int count, uint32_t flags)
{
    return media_offset(offMatRi, count) + ((flags & kSceneMedia) ? media_bytes(count) : 0u);
}

inline SceneBlobLayout scene_blob_layout(int count, int nLights)
{
    int simdCount = (count + 3) / 4 * 4;
    SceneBlobLayout L;
    uint32_t off = 0;
    L.offSph = off;        off += align16((uint32_t)simdCount * 16u);
    L.offInvRadius = off;  off += align16((uint32_t)simdCount * 4u);
    L.offLights = off;     off += align16((uint32_t)(nLights > 0 ? nLights : 1) * (uint32_t)sizeof(LightRec));
    L.geomBytes = off;
    L.offMatA = off;       off += align16((uint32_t)(count + 1) * 16u);
    L.offMatB = off;       off += align16((uint32_t)(count + 1) * 16u);
    L.offMatRi = off;      off += align16((uint32_t)(count + 1) * 4u);
    L.totalBytes = off;
    L.flags = 0;
    L.envLo = L.envHi = 0;
    L.envW = L.envH = 0;
    L.tex = L.emit = TexSet{};
    return L;
}

// A medium record of tpt_set_media {sigma_a.r, sigma_a.g, sigma_a.b, sigma_s, g}: "no medium" when both sigmas are zero.
inline bool has_medium(const float* m5) { return m5[0] != 0.0f || m5[1] != 0.0f || m5[2] != 0.0f || m5[3] != 0.0f; }
// A fog record of tpt_set_fog {c.x, c.y, c.z, R, sigma_a.r, sigma_a.g, sigma_a.b, sigma_s, g}: "no fog" when its sigmas
// are all zero.
inline bool has_fog(const float* f9) { return f9 && has_medium(f9 + 4); }

// emissives == nullptr: derive the list like UpdateTest (Test.cpp:333-338).
// media5: mediaSpheres records of tpt_set_media (null: none). The blob gets the media section, and kSceneMedia, only when a
// sphere below `count` has a medium; otherwise its bytes are those of the scene without media.
// fog9: tpt_set_fog's record (null: none). The blob gets the fog section, and kSceneFog, only when it has a non-zero
// sigma; otherwise its bytes are those of the scene without fog.
inline void pack_scene_blob(const Sphere20* spheres, const Material36* mats, int count,
                            const int* emissives, int emissiveCount,
                            std::vector<unsigned char>& blob, SceneBlobLayout& L, int& nLights, uint32_t sceneFlags = 0,
                            const float* media5 = nullptr, int mediaSpheres = 0, const float* fog9 = nullptr)
{
    const int nMedia = media5 ? (mediaSpheres < count ? mediaSpheres : count) : 0;
    bool anyMedium = false;
    for (int i = 0; i < nMedia; ++i) anyMedium = anyMedium || has_medium(media5 + 5 * i);
    std::vector<int> em;
    if (emissives) em.assign(emissives, emissives + emissiveCount);
    else
        for (int i = 0; i < count; ++i)
            if (mats[i].emissive[0] > 0 || mats[i].emissive[1] > 0 || mats[i].emissive[2] > 0) em.push_back(i);
    nLights = (int)em.size();
    L = scene_blob_layout(count, nLights);
    L.flags = sceneFlags & ~(uint32_t)(kSceneMedia | kSceneFog);
    if (anyMedium)
    {
        L.flags |= kSceneMedia;
        L.totalBytes += media_bytes(count);    // geomBytes stays: the section is material data
    }
    const bool fog = has_fog(fog9);
    if (fog)
    {
        L.flags |= kSceneFog;
        L.totalBytes += kFogBytes;
    }
    int simdCount = (count + 3) / 4 * 4;
    blob.assign(L.totalBytes, 0);
    Q4* sph = (Q4*)(blob.data() + L.offSph);
    float* invR = (float*)(blob.data() + L.offInvRadius);
    LightRec* lights = (LightRec*)(blob.data() + L.offLights);
    Q4* matA = (Q4*)(blob.data() + L.offMatA);
    Q4* matB = (Q4*)(blob.data() + L.offMatB);
    float* matRi = (float*)(blob.data() + L.offMatRi);
    for (int i = 0; i < simdCount; ++i)
    {
        if (i < count)
        {
            const Sphere20& s = spheres[i];
            sph[i].x = s.center[0]; sph[i].y = s.center[1]; sph[i].z = s.center[2];
            sph[i].w = s.radius * s.radius;          // Test.cpp:329
            invR[i] = 1.0f / s.radius;               // Maths.h:359
        }
        else
        {
            sph[i].x = sph[i].y = sph[i].z = 10000.0f; sph[i].w = 0.0f; invR[i] = 0.0f; // Maths.h:382-387
        }
    }
    for (int i = 0; i < count; ++i)
    {
        const Material36& m = mats[i];
        matA[i].x = m.albedo[0]; matA[i].y = m.albedo[1]; matA[i].z = m.albedo[2];
        memcpy(&matA[i].w, &m.type, 4);
        matB[i].x = m.emissive[0]; matB[i].y = m.emissive[1]; matB[i].z = m.emissive[2];
        matB[i].w = ((sceneFlags & kSceneMitsuba) && m.type == kMetal) ? 0.0f : m.roughness;   // Test.cpp:143-145
        matRi[i] = m.ri;
    }
    // entry [count]: all-zero (Lambert, black) — what the reference's out-of-bounds material read amounts to
    if (anyMedium)
    {
        Q4* media = (Q4*)(blob.data() + media_offset(L.offMatRi, count));
        float* g = (float*)(media + count + 1);
        for (int i = 0; i < nMedia; ++i)
        {
            const float* m = media5 + 5 * i;
            media[i].x = m[0]; media[i].y = m[1]; media[i].z = m[2]; media[i].w = m[3];
            g[i] = m[4];
        }
    }
    if (fog)
    {
        float* f = (float*)(blob.data() + fog_offset(L.offMatRi, count, L.flags));
        for (int k = 0; k < 9; ++k) f[k] = fog9[k];
    }
    for (int j = 0; j < nLights; ++j)
    {
        int i = em[j];
        LightRec& R = lights[j];
        R.cx = spheres[i].center[0]; R.cy = spheres[i].center[1]; R.cz = spheres[i].center[2];
        R.radius = spheres[i].radius;
        R.ex = mats[i].emissive[0]; R.ey = mats[i].emissive[1]; R.ez = mats[i].emissive[2];
        R.id = i;
    }
}

// ParamPairs of a packed scene of at most kParamPairSpheres padded spheres, bit-identical to the pair array the kernels
// build in shared memory (build_sphK, build_sph_pairs): K = |s|^2 - r^2 in double (the float products are exact in
// double, so contraction cannot change it) rounded to float, padded spheres K = 1e30; unused entries zero.
inline void build_param_pairs(const std::vector<unsigned char>& blob, const SceneBlobLayout& L, int count, ParamPairs& pp)
{
    memset(&pp, 0, sizeof(pp));
    const int simdCount = (count + 3) / 4 * 4;
    if (simdCount > kParamPairSpheres) return;
    const Q4* sph = (const Q4*)(blob.data() + L.offSph);
    for (int i = 0; i < simdCount; ++i)
    {
        const Q4 s = sph[i];
        const double K = (double)s.x * s.x + (double)s.y * s.y + (double)s.z * s.z - (double)s.w;
        float* f = pp.f + (i >> 1) * 8 + (i & 1);
        f[0] = s.x; f[2] = s.y; f[4] = s.z;
        f[6] = -(i < count ? (float)K : 1.0e30f);
    }
}

// IEEE binary16 bits of x rounded to nearest-even (mode 0), up (+1) or down (-1); |x| must stay below 65504.
inline uint16_t half_bits(double x, int mode)
{
    const double ax = fabs(x);
    int e = 0;
    if (ax > 0) { frexp(ax, &e); --e; }                 // ax in [2^e, 2^(e+1))
    const double q = ldexp(1.0, (e > -14 ? e : -14) - 10);
    double k = x / q;                                    // exact: q is a power of two
    k = mode > 0 ? ceil(k) : mode < 0 ? floor(k) : nearbyint(k);
    const double v = fabs(k * q);
    const uint16_t sign = (k < 0 || (k == 0 && signbit(x))) ? 0x8000u : 0u;
    if (v < ldexp(1.0, -14)) return (uint16_t)(sign | (uint16_t)(v / ldexp(1.0, -24)));
    int ev = 0;
    const double m = frexp(v, &ev);                      // v = m 2^ev, m in [0.5, 1)
    return (uint16_t)(sign | (uint16_t)((ev - 1 + 15) << 10) | (uint16_t)(m * 2048.0 - 1024.0));
}

// Sweep form 5's pass-1 operands (FastHitterKH, tpt_fast.cu; the bound is derived in DESIGN §3.1c). A sphere is a pass-1
// candidate when, in half precision with u = 2^-11, xu = s.u - o.u and xv = s.v - o.v (u, v an orthonormal basis
// around d) give xu^2 + xv^2 - R'^2 < 0: its line passes within R' of the centre. R' is the radius widened by the error
// bound (E per coordinate, Rw for the FP32 rounding of form 2, the basis and |d|) for origins with |o| <= kHalfOriginBound and |d|^2 within 2^-18 of 1, so the candidate set contains every sphere
// form 2's FP32 pass 2 accepts. Returns false (form 4 keeps the scene) when a scene has more than kParamPairSpheres
// padded spheres or a sphere whose intermediates could leave the half range.
inline bool build_half_pairs(const std::vector<unsigned char>& blob, const SceneBlobLayout& L, int count, ParamPairs& pp)
{
    const int simdCount = (count + 3) / 4 * 4;
    if (simdCount > kParamPairSpheres) return false;
    const Q4* sph = (const Q4*)(blob.data() + L.offSph);
    const double u = ldexp(1.0, -11), Om = kHalfOriginBound, kLimit = 30000.0;
    for (int base = 0; base < simdCount; base += 32)
    {
        const int n = simdCount - base < 32 ? simdCount - base : 32, h = n / 2;
        for (int j = 0; j < n; ++j)
        {
            uint16_t x = 0, y = 0, z = 0, nr2 = half_bits(60000.0, 0);   // padding: q >= 60000, never a candidate
            if (base + j < count)
            {
                const Q4 s = sph[base + j];
                const double S = sqrt((double)s.x * s.x + (double)s.y * s.y + (double)s.z * s.z), R2 = s.w;
                const double E = u * (5.01 * S + 4.01 * Om) + ldexp(1.0, -20);
                const double Rw = sqrt(R2 + ldexp(S * S + Om * Om + R2, -15));
                const double Rp2 = (Rw + 1.4143 * E) * (Rw + 1.4143 * E) / (1.0 - u) * (1.0 + ldexp(1.0, -20));
                if ((S + Om + 1.0) * (S + Om + 1.0) > kLimit || Rp2 > kLimit) return false;
                x = half_bits(s.x, 0); y = half_bits(s.y, 0); z = half_bits(s.z, 0);
                nr2 = half_bits(-Rp2, -1);
            }
            uint32_t* w = pp.h + (base / 2 + j % h) * kHalfPairWords;
            const int sh = j < h ? 0 : 16;
            w[0] |= (uint32_t)x << sh; w[1] |= (uint32_t)y << sh; w[2] |= (uint32_t)z << sh;
            w[3] |= (uint32_t)nr2 << sh;
        }
    }
    return true;
}

inline SceneView scene_view_from_blob(const unsigned char* base, const SceneBlobLayout& L, int count, int nLights)
{
    SceneView v;
    v.sph = (const Q4*)(base + L.offSph);
    v.invRadius = (const float*)(base + L.offInvRadius);
    v.lights = (const LightRec*)(base + L.offLights);
    v.matA = (const Q4*)(base + L.offMatA);
    v.matB = (const Q4*)(base + L.offMatB);
    v.matRi = (const float*)(base + L.offMatRi);
    v.media = (const Q4*)(base + media_offset(L.offMatRi, count));
    v.fog = (const Q4*)(base + fog_offset(L.offMatRi, count, L.flags));
    v.count = count;
    v.simdCount = (count + 3) / 4 * 4;
    v.nLights = sampled_lights(L.flags, nLights);
    v.flags = L.flags;
    v.maxDepth = scene_max_depth(L.flags);
    v.sphShared = 0;
    v.envLo = v.envHi = 0;     // host views never look up an environment
    v.envW = v.envH = 0;
    v.tex = v.emit = TexSet{};     // nor textures
    return v;
}

} // namespace tpt
