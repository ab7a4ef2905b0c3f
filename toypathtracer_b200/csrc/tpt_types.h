// Data layouts shared by the host API and the kernels.
// The three raw structs are byte-for-byte the reference's scene export (GetSceneDesc, Cpp/Source/Test.cpp:377-384;
// sizes asserted by the reference's GPU shells at Cpp/Windows/TestWin.cpp:132-134):
//   Sphere   20 B  Cpp/Source/Maths.h:354-364     {float center[3]; float radius; float invRadius}
//   Material 36 B  Cpp/Source/Test.cpp:36-44      {int type; float albedo[3]; float emissive[3]; float roughness; float ri}
//   Camera   88 B  Cpp/Source/Maths.h:444-449     {origin, lowerLeftCorner, horizontal, vertical, uu, vv, ww (float3pack each); float lensRadius}
#pragma once
#include <stdint.h>

namespace tpt {

struct Sphere20 { float center[3]; float radius; float invRadius; };
struct Material36 { int type; float albedo[3]; float emissive[3]; float roughness; float ri; };
struct Camera88 { float origin[3], lowerLeftCorner[3], horizontal[3], vertical[3], uu[3], vv[3], ww[3]; float lensRadius; };

static_assert(sizeof(Sphere20) == 20, "Sphere layout");
static_assert(sizeof(Material36) == 36, "Material layout");
static_assert(sizeof(Camera88) == 88, "Camera layout");

enum MaterialType { kLambert = 0, kMetal = 1, kDielectric = 2 };

// 16-byte quad usable from host-only builds too (float4 on device).
struct alignas(16) Q4 { float x, y, z, w; };

// One record per emissive sphere (Test.cpp:321-338 builds the id list; Test.cpp:96-133 consumes it).
struct alignas(16) LightRec
{
    float cx, cy, cz, radius;   // s_Spheres[i]
    float ex, ey, ez;           // s_SphereMats[i].emissive
    int id;
};

// One set of lat-long sphere textures as the kernels see it (tpt_set_textures, tpt_set_emission_textures): the address
// of its W x H RGBA texels, layer-major (row 0 = the +y pole, global memory) and of the int32 layer of each sphere id below
// `spheres` (-1: none; begin_call keeps `spheres` at most the scene's count, so padding spheres are never textured). The
// addresses travel as 32-bit halves, which keeps the struct 4-byte aligned (an 8-byte aligned kernel parameter changes
// how the compiler loads the fields around it). `tabWords` also keeps the struct a multiple of 8 bytes, so the kernel
// parameters behind SceneBlobLayout keep the 8-byte pairing of their constant-bank loads (an odd number of added words
// changed untextured kernels' SASS): for the emission set, the int32 words from the sphere table to the layers' sampling
// tables (tpt_env_tables.h, emit_table_words of the uploaded table's length); 0 for the albedo set, which has none.
struct TexSet
{
    uint32_t texLo, texHi, tabLo, tabHi;
    int W, H, spheres;
    uint32_t tabWords;
};

// Device-side scene, SoA, padded like the reference's SpheresSoA (Maths.h:368-404):
//   sph[i]  = {centerX, centerY, centerZ, sqRadius}, i < simdCount, entries >= count are the
//             "impossible" spheres (centre 10000, r^2 = 0, invRadius 0)
//   matA[i] = {albedo.xyz, type (int bits)}, matB[i] = {emissive.xyz, roughness}, matC[i] = ri
//             i <= count; entry [count] is the all-zero material the reference's out-of-bounds read
//             amounts to (see DESIGN.md "padded-sphere hits").
struct SceneView
{
    const Q4* sph;
    const float* invRadius;
    const Q4* matA;
    const Q4* matB;
    const float* matRi;
    const Q4* media;      // kSceneMedia: {sigma_a.rgb, sigma_s}[count + 1], then g[count + 1] (media_offset, tpt_scene_pack.h)
    const Q4* fog;        // kSceneFog: {c.xyz, R}, {sigma_a.rgb, sigma_s}, {g, 0, 0, 0} (fog_offset, tpt_scene_pack.h)
    const LightRec* lights;
    int count, simdCount, nLights;
    uint32_t flags;       // kScene* bits
    int maxDepth;         // the call's "max_depth" (scene_max_depth of flags): read only where TEX (path_step)
    uint32_t sphShared;   // device: 32-bit shared-memory address of sph[] (always staged), for ld.shared.v4
    uint32_t envLo, envHi; // kSceneEnvironment: address of the envW x envH RGBA texels of the lat-long environment (row 0 =
    int envW, envH;        // zenith, global memory) in two halves, as SceneBlobLayout carries it; its sampling tables follow
                           // the texels (tpt_env_tables.h)
    TexSet tex;            // kSceneTextures: tpt_set_textures' albedo layers
    TexSet emit;           // kSceneEmissionTextures: tpt_set_emission_textures' emission layers
};

// Blob layout in global memory (one contiguous, 16 B-aligned allocation so a single bulk copy stages it
// into shared memory): [sph simdCount*16][matA (count+1)*16][matB (count+1)*16][lights nLights*32]
// [invRadius simdCount*4][matRi (count+1)*4], each section padded to 16 B.
struct SceneBlobLayout
{
    uint32_t offSph, offMatA, offMatB, offLights, offInvRadius, offMatRi, totalBytes;
    uint32_t geomBytes; // bytes of [sph .. end] needed by intersection + lights only (== totalBytes here)
    uint32_t flags;     // kScene* bits (travels to the kernels with the layout)
    // tpt_set_environment's map (kSceneEnvironment): its device address as two 32-bit halves, which keeps the struct 4-byte
    // aligned (an 8-byte aligned kernel parameter changes how the compiler loads the fields around it), and its size.
    // Not part of the blob: each call's copy of the layout gets them (begin_call).
    uint32_t envLo, envHi;
    int envW, envH;
    // tpt_set_textures' albedo layers (kSceneTextures) and tpt_set_emission_textures' emission layers
    // (kSceneEmissionTextures), the same way.
    TexSet tex, emit;
};

// DO_MITSUBA_COMPARE (Config.h:25) as a runtime switch: constant sky (Test.cpp:226-227) and zero Metal roughness
// (Test.cpp:143-145; applied when the scene is packed). Its third effect, zero aperture (Test.cpp:312-313), is camera
// data and therefore the caller's (the Test.h shim's UpdateTest builds the camera).
// DO_LIGHT_SAMPLING (Config.h:24) switched OFF at run time: no explicit light sampling at Lambert vertices (no light
// draws, no shadow rays, Test.cpp:95-133) and the emission of every hit is added (the doMaterialE suppression of
// Test.cpp:209-215 is compiled out there). The kernels see it as a light count of 0 (sampled_lights()) plus the
// emission rule (emission_after_lambert()).
// An environment set with tpt_set_environment: a lat-long radiance map replaces the sky at the fast kernels' miss sites
// (fast_sky) for the calls issued while it is set; the mitsuba constant sky included, its zero Metal roughness not.
// kSceneEnvSampling ("environment_sampling" active for the call, set by begin_call with kSceneEnvironment): the slab
// queue's sampling instances take one environment sample per light-sampled Lambert vertex (sample_env), with the map's
// tables behind its texels (tpt_env_tables.h).
// kSceneTextures (tpt_set_textures, set by begin_call): the slab queue's reference-form instances and the AOV kernel
// multiply the albedo of a hit on a textured sphere by its layer's lat-long lookup at the hit's normal (sphere_texture).
// kSceneEmissionTextures (tpt_set_emission_textures, set by begin_call): the same instances multiply the emission of a hit
// on a sphere with an emission layer, and that of a light where its shadow ray meets it, by the layer's lookup there.
// kSceneEmitSampling ("emission_texture_sampling" active for the call, set by begin_call with kSceneEmissionTextures): the
// same instances take one texture sample per light with a sampleable emission layer at light-sampled Lambert vertices
// (sample_emit), and weight that light's cone rays against it.
// kSceneMedia (tpt_set_media, set by the pack when some sphere of the scene has a medium): the blob carries the media
// section behind matRi, and the same instances absorb and scatter along path segments that end on the inside face of a
// glass sphere with a medium (medium_step).
// kSceneDepth ("max_depth" other than the reference's 10 for the call, set by begin_call): the value travels in bits
// kSceneDepthShift.. of the call's flags (depth_flags, scene_max_depth), and the same instances end paths at that depth
// instead, with Russian roulette past depth 10 when it is larger (path_step).
// kSceneFog (tpt_set_fog, set by the pack when the context's fog has a non-zero sigma): the blob carries the fog section
// behind the media section, and the same instances absorb and scatter along path segments in air inside the fog's ball,
// sample the lights at fog scatter vertices and attenuate shadow rays in air (fog_step, fog_transmittance).
enum SceneFlags : uint32_t { kSceneMitsuba = 1u, kSceneNoLightSampling = 2u, kSceneEnvironment = 4u, kSceneEnvSampling = 8u,
                             kSceneTextures = 16u, kSceneEmissionTextures = 32u, kSceneEmitSampling = 64u, kSceneMedia = 128u,
                             kSceneDepth = 256u, kSceneFog = 512u };
// Either texture set: the calls that have one run the instances that look textures up (pick_queue, fast_auto_variant).
constexpr uint32_t kSceneAnyTextures = kSceneTextures | kSceneEmissionTextures;
// What only the slab queue's reference-form instances (sweep form 0, path_step's ENVM 2 and TEX) compute: a call with any of
// these runs them (pick_queue, fast_auto_variant, tpt_draw's variant checks).
constexpr uint32_t kSceneRefForm = kSceneEnvSampling | kSceneAnyTextures | kSceneMedia | kSceneDepth | kSceneFog;

// "max_depth": the reference's compile-time cap (TPT_MAX_DEPTH, tpt_integrator.cuh) is the default and the depth from
// which Russian roulette runs; the option takes 1..kMaxPathDepth. A per-call value, never part of the scene's blob or the
// layout the upload compares: it exists only in the copy of the layout a call passes to its kernels.
constexpr int kRefMaxDepth = 10;
constexpr int kMaxPathDepth = 256;
constexpr int kSceneDepthShift = 16;
constexpr uint32_t kSceneDepthMask = 0x1ffu;   // 9 bits: 1..256
// The flag bits of a call with max_depth n: none for the default.
inline constexpr uint32_t depth_flags(int n)
{
    return n == kRefMaxDepth ? 0u : kSceneDepth | ((uint32_t)n & kSceneDepthMask) << kSceneDepthShift;
}
// The max_depth of a call's flags.
#ifdef __CUDACC__
__host__ __device__
#endif
inline constexpr int scene_max_depth(uint32_t flags)
{
    return (flags & kSceneDepth) ? (int)(flags >> kSceneDepthShift & kSceneDepthMask) : kRefMaxDepth;
}

// Number of lights the integrators sample: the scene's emissive list with light sampling on, none with it off. The blob
// keeps the light table either way, so toggling the switch uploads the same bytes.
inline int sampled_lights(uint32_t sceneFlags, int nLights) { return (sceneFlags & kSceneNoLightSampling) ? 0 : nLights; }

// The fast slab queue's pass-1 operands for scenes of at most kParamPairSpheres padded spheres (sweep form 4): the pair
// array of the expanded form, pair p = spheres 2p, 2p+1 as f[8p ..] = {x0, x1, y0, y1, z0, z1, -K0, -K1}, built on the
// host (build_param_pairs) and passed by value in a __grid_constant__ kernel parameter, so that pass 1 reads the sphere
// values from the constant bank into uniform registers instead of from shared memory into vector registers.
// h: sweep form 5's half-precision pass 1 (build_half_pairs), four packed half2 words per pair {X, Y, Z, -R'^2};
// pair p of the block of n spheres at 32B holds sphere 32B + p in its low half and sphere 32B + n/2 + p in its high half.
constexpr int kParamPairSpheres = 64;
constexpr int kHalfPairWords = 4;
constexpr float kHalfOriginBound = 16.0f;   // form 5's bound holds for ray origins with |o| <= kHalfOriginBound
struct ParamPairs
{
    float f[kParamPairSpheres * 4];
    uint32_t h[kParamPairSpheres / 2 * kHalfPairWords];
    int half;           // 1: the form-4 kernels sweep with form 5's half-precision pass 1 on h (0: FP32 pass 1 on f)
};

struct DrawParams
{
    Camera88 cam;
    int width, height;
    int row0, numRows;        // rows y_i = row0 + i*rowStep, i in [0,numRows)  (Test.cpp:266 TraceRowJob(start,end))
    int rowStep;              // 1 = contiguous band; world_size = rows interleaved across GPUs
    int packed;               // 0: row y_i lives at image row y_i (full image); 1: at image row i (packed band)
    int frame0, numFrames;    // frames [frame0, frame0+numFrames), N spp = N/spp reference frames
    int spp;                  // DO_SAMPLES_PER_PIXEL (Config.h:22)
    unsigned flags;           // kFlagAnimate = 1, kFlagProgressive = 2 (Test.h:4-8)
    int zeroAlpha;            // fast mode, prev weight 0: 1 = write alpha 0, 0 = keep the buffer's alpha (Maths.h:38: never written)
    float invWidth, invHeight;
    float* image;             // full image base, width*height*4 floats, row 0 = bottom (device)
    float* scratch;           // exact mode, numFrames > 1: [numFrames][numRows][width] float4 per-frame colours
    unsigned long long* rayCounter; // [numFrames] in exact mode, [1] in fast mode
    unsigned int* workCounter;      // persistent kernels: next tile
    const float* rays;        // tpt_trace_rays: numRays caller rays {o.xyz, d.xyz}, 4-byte aligned; `image` gets one float4 per ray
    uint32_t numRays;
    // tpt_draw_samples: numRays list entries, pixel indices y * width + x (null: entry i is pixel i); `image` (sum4) and sq4
    // get one float4 per entry. badPixel: the index check's result, ~0 when every index is inside the image.
    const int* pixels;
    float* sq4;
    const unsigned long long* badPixel;
    // tpt_trace_irradiance: the numRays `rays` are surface points {p.xyz, n.xyz}, and each sample starts as a white Lambert
    // vertex at (p, n) instead of a ray from p (launch-uniform). pointIds: null, or numRays sphere ids, entry i the sphere
    // point i lies on (that sphere's light is not sampled from it).
    int pointStart;
    const int* pointIds;
    // tpt_trace_samples (launch-uniform): with `sums`, image (sum4) and, when set, sq4 get (v, 1) and (v^2, 0) per sample
    // instead of the mean. entries: null (entry i is input i), or numRays indices into the inputs `rays`, entry k tracing
    // input entries[k] with that input's streams and ids; checked against the inputs before the launch (badPixel).
    int sums;
    const int* entries;
};

} // namespace tpt
