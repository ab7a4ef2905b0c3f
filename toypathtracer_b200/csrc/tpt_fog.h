// Fog between the spheres (tpt_set_fog, kSceneFog; DESIGN §3.16): the geometry of its ball and its phase function,
// shared by the pack, the fast kernels and the host checks (tests/host_sim/fog_check.cpp).
#pragma once
#include <stdint.h>
#include <math.h>

namespace tpt {

#ifdef __CUDACC__
#define TPT_FOG_HD __host__ __device__ __forceinline__
#else
#define TPT_FOG_HD inline
#endif

// The blob's fog section: three 16 B records {c.xyz, R}, {sigma_a.rgb, sigma_s}, {g, 0, 0, 0}.
constexpr uint32_t kFogBytes = 48;

// The fog part of the ray segment o + s d, s in [0, t], d a unit vector, in the ball {c, R}: returns its length
// L = |[0, t] ∩ [t_in, t_out]| and puts where it starts, max(t_in, 0), in *tin (0 when L is 0). The chord's half-length
// comes from R^2 - |h|^2, h the offset of the line's closest point from c, which keeps near-tangent lines accurate where
// b^2 - (|o - c|^2 - R^2) would cancel.
TPT_FOG_HD float fog_chord(float ox, float oy, float oz, float dx, float dy, float dz, float t, float cx, float cy, float cz,
                           float R, float* tin)
{
    const float px = ox - cx, py = oy - cy, pz = oz - cz;
    const float b = px * dx + py * dy + pz * dz;
    const float hx = px - b * dx, hy = py - b * dy, hz = pz - b * dz;
    const float disc = R * R - (hx * hx + hy * hy + hz * hz);
    *tin = 0.0f;
    if (!(disc > 0.0f)) return 0.0f;
    const float q = sqrtf(disc);
    const float a = fmaxf(-b - q, 0.0f);
    const float L = fminf(q - b, t) - a;
    if (!(L > 0.0f)) return 0.0f;
    *tin = a;
    return L;
}

// The Henyey-Greenstein phase function p(cos) = (1 - g^2) / (4 pi (1 + g^2 - 2 g cos)^(3/2)), per steradian, with cos the
// cosine between the incoming and the outgoing direction; exactly 1 / (4 pi) for |g| < 1e-3, where hg_sample (tpt_fast.cu)
// samples uniformly.
constexpr float kFogInv4Pi = 0.0795774715f;
TPT_FOG_HD float hg_phase(float cosT, float g)
{
    if (!(fabsf(g) >= 1e-3f)) return kFogInv4Pi;
    const float den = 1.0f + g * g - 2.0f * g * cosT;
    return (1.0f - g * g) * kFogInv4Pi / (den * sqrtf(den));
}

} // namespace tpt
