// Drop-in replacement for the reference's Cpp/Source/Test.cpp: exports the six functions of
// Cpp/Source/Test.h:10-17 with identical C++ signatures, so any reference shell (Cpp/Windows/TestWin.cpp,
// Cpp/Apple/Renderer.mm, Cpp/Emscripten/main.cpp) links against this file + libtpt_b200.so unchanged.
// Host side keeps what UpdateTest does (scene animation, camera construction, emissive list — Test.cpp:302-342);
// DrawTest forwards to the CUDA kernels through the C-ABI (include/tpt_b200.h). No tracing happens on the CPU.
//
// Extra C entry points (not in Test.h) select the mode/device: tpt_shim_set_mode(), tpt_shim_context(), and the
// reference's two compile-time scene switches as runtime ones: tpt_shim_set_variant(bigScene, mitsubaCompare)
// (DO_BIG_SCENE Test.cpp:10-11, DO_MITSUBA_COMPARE Config.h:25), and the third one, DO_LIGHT_SAMPLING (Config.h:24),
// as tpt_shim_set_light_sampling(on).
// Environment: TPT_MODE=exact|fast|refgpu|refgpu_fast (default exact: results bit-identical to the reference),
// TPT_DEVICE=<n>, TPT_PIN_BACKBUFFER=1 (cudaHostRegister the caller's backbuffer once), TPT_BIG_SCENE=0|1,
// TPT_MITSUBA=0|1, TPT_LIGHT_SAMPLING=0|1.
#include "../../include/tpt_b200.h"   // (include/tpt_test_shim.h documents this file's exports)
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

enum TestFlags { kFlagAnimate = (1 << 0), kFlagProgressive = (1 << 1) };

void InitializeTest();
void ShutdownTest();
void UpdateTest(float time, int frameCount, int screenWidth, int screenHeight, unsigned testFlags);
void DrawTest(float time, int frameCount, int screenWidth, int screenHeight, float* backbuffer, int& outRayCount, unsigned testFlags);
void GetObjectCount(int& outCount, int& outObjectSize, int& outMaterialSize, int& outCamSize);
void GetSceneDesc(void* outObjects, void* outMaterials, void* outCam, void* outEmissives, int* outEmissiveCount);

namespace {

const float kPI = 3.1415926f; // Maths.h:9

struct Sphere { float center[3]; float radius; float invRadius; };                               // Maths.h:354-364
struct Material { int type; float albedo[3]; float emissive[3]; float roughness; float ri; };   // Test.cpp:36-44
struct Camera { float origin[3], lowerLeftCorner[3], horizontal[3], vertical[3], uu[3], vv[3], ww[3]; float lensRadius; }; // Maths.h:444-449
enum { Lambert = 0, Metal = 1, Dielectric = 2 };

const int kMaxSphereCount = 46;
int kSphereCount = 46;             // 46 spheres (2 emissive) with DO_BIG_SCENE, 9 spheres (1 emissive) without (Test.cpp:10)
bool s_Mitsuba = false;            // DO_MITSUBA_COMPARE (Config.h:25)
bool s_LightSampling = true;       // DO_LIGHT_SAMPLING (Config.h:24)
Sphere s_Spheres[kMaxSphereCount];
Material s_SphereMats[kMaxSphereCount];
int s_EmissiveSpheres[kMaxSphereCount];
int s_EmissiveSphereCount;
Camera s_Cam;
bool s_SceneBuilt = false;

tpt_context* s_Ctx = nullptr;
int s_Mode = TPT_MODE_EXACT;

void setSphere(int i, float x, float y, float z, float r)
{
    s_Spheres[i].center[0] = x; s_Spheres[i].center[1] = y; s_Spheres[i].center[2] = z;
    s_Spheres[i].radius = r; s_Spheres[i].invRadius = 0.0f;
}
void setMat(int i, int type, float ar, float ag, float ab, float er, float eg, float eb, float rough, float ri)
{
    Material& m = s_SphereMats[i];
    m.type = type; m.albedo[0] = ar; m.albedo[1] = ag; m.albedo[2] = ab;
    m.emissive[0] = er; m.emissive[1] = eg; m.emissive[2] = eb; m.roughness = rough; m.ri = ri;
}

// The reference's 46-sphere scene (data of Test.cpp:13-31 and :46-64, DO_BIG_SCENE = 1), rebuilt
// procedurally: ground, 8 hero spheres, 4 rows x 9 small spheres at z = -3..-6, x = 4..-4, one extra light.
void buildScene()
{
    setSphere(0, 0, -100.5f, -1, 100);
    setSphere(1, 2, 0, -1, 0.5f);   setSphere(2, 0, 0, -1, 0.5f);   setSphere(3, -2, 0, -1, 0.5f);
    setSphere(4, 2, 0, 1, 0.5f);    setSphere(5, 0, 0, 1, 0.5f);    setSphere(6, -2, 0, 1, 0.5f);
    setSphere(7, 0.5f, 1, 0.5f, 0.5f);
    setSphere(8, -1.5f, 1.5f, 0.f, 0.3f);
    for (int row = 0; row < 4; ++row)
        for (int k = 0; k < 9; ++k)
            setSphere(9 + row * 9 + k, (float)(4 - k), 0, (float)(-3 - row), 0.5f);
    setSphere(45, 1.5f, 1.5f, -2, 0.3f);

    setMat(0, Lambert, 0.8f, 0.8f, 0.8f, 0, 0, 0, 0, 0);
    setMat(1, Lambert, 0.8f, 0.4f, 0.4f, 0, 0, 0, 0, 0);
    setMat(2, Lambert, 0.4f, 0.8f, 0.4f, 0, 0, 0, 0, 0);
    setMat(3, Metal, 0.4f, 0.4f, 0.8f, 0, 0, 0, 0, 0);
    setMat(4, Metal, 0.4f, 0.8f, 0.4f, 0, 0, 0, 0, 0);
    setMat(5, Metal, 0.4f, 0.8f, 0.4f, 0, 0, 0, 0.2f, 0);
    setMat(6, Metal, 0.4f, 0.8f, 0.4f, 0, 0, 0, 0.6f, 0);
    setMat(7, Dielectric, 0.4f, 0.4f, 0.4f, 0, 0, 0, 0, 1.5f);
    setMat(8, Lambert, 0.8f, 0.6f, 0.2f, 30, 25, 15, 0, 0);
    static const float grey[9] = {0.1f, 0.2f, 0.3f, 0.4f, 0.5f, 0.6f, 0.7f, 0.8f, 0.9f};
    static const float hue[9][3] = {{0.8f, 0.1f, 0.1f}, {0.8f, 0.5f, 0.1f}, {0.8f, 0.8f, 0.1f}, {0.4f, 0.8f, 0.1f}, {0.1f, 0.8f, 0.1f},
                                    {0.1f, 0.8f, 0.5f}, {0.1f, 0.8f, 0.8f}, {0.1f, 0.1f, 0.8f}, {0.5f, 0.1f, 0.8f}};
    for (int k = 0; k < 9; ++k)
    {
        setMat(9 + k, Lambert, grey[k], grey[k], grey[k], 0, 0, 0, 0, 0);
        setMat(18 + k, Metal, grey[k], grey[k], grey[k], 0, 0, 0, 0, 0);
        setMat(27 + k, Metal, hue[k][0], hue[k][1], hue[k][2], 0, 0, 0, 0, 0);
        setMat(36 + k, k == 8 ? Metal : Lambert, hue[k][0], hue[k][1], hue[k][2], 0, 0, 0, 0, 0);
    }
    setMat(45, Lambert, 0.1f, 0.2f, 0.5f, 3, 10, 20, 0, 0);
    s_SceneBuilt = true;
}

struct v3 { float x, y, z; };
inline v3 mk(float x, float y, float z) { v3 r = {x, y, z}; return r; }
inline v3 operator-(v3 a, v3 b) { return mk(a.x - b.x, a.y - b.y, a.z - b.z); }
inline v3 operator*(float a, v3 b) { return mk(a * b.x, a * b.y, a * b.z); }
inline v3 operator*(v3 a, float b) { return mk(a.x * b, a.y * b, a.z * b); }
inline float dot(v3 a, v3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
inline v3 cross(v3 a, v3 b) { return mk(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
inline v3 normalize(v3 v) { return v * (1.0f / sqrtf(dot(v, v))); }
inline void st(float* p, v3 v) { p[0] = v.x; p[1] = v.y; p[2] = v.z; }

// Camera constructor, Maths.h:418-435
void buildCamera(v3 lookFrom, v3 lookAt, v3 vup, float vfov, float aspect, float aperture, float focusDist)
{
    s_Cam.lensRadius = aperture / 2;
    float theta = vfov * kPI / 180;
    float halfHeight = tanf(theta / 2);
    float halfWidth = aspect * halfHeight;
    v3 org = lookFrom;
    v3 w = normalize(lookFrom - lookAt);
    v3 u = normalize(cross(vup, w));
    v3 v = cross(w, u);
    st(s_Cam.origin, org);
    st(s_Cam.ww, w); st(s_Cam.uu, u); st(s_Cam.vv, v);
    st(s_Cam.lowerLeftCorner, org - halfWidth * focusDist * u - halfHeight * focusDist * v - focusDist * w);
    st(s_Cam.horizontal, 2 * halfWidth * focusDist * u);
    st(s_Cam.vertical, 2 * halfHeight * focusDist * v);
}

void die(const char* what, int code)
{
    fprintf(stderr, "toypathtracer_b200: %s failed (%d): %s\n", what, code, s_Ctx ? tpt_last_error(s_Ctx) : "no context");
    abort(); // the Test.h API is void-returning (SURVEY §8b "Errors: none"); there is no CPU path to fall back to
}

} // namespace

extern "C" void tpt_shim_set_mode(int mode) { s_Mode = mode; }
// Restores the un-animated scene (the reference keeps animated positions in its static arrays forever,
// Test.cpp:304-308; a reference shell never needs this, tests do).
extern "C" void tpt_shim_reset_scene() { buildScene(); }
// DO_BIG_SCENE / DO_MITSUBA_COMPARE at run time. The 9-sphere scene is the first 9 entries of the tables (Test.cpp:15-24,
// :48-57). Takes effect with the next UpdateTest().
extern "C" void tpt_shim_set_variant(int bigScene, int mitsubaCompare)
{
    kSphereCount = bigScene ? 46 : 9;
    s_Mitsuba = mitsubaCompare != 0;
    buildScene();
}
// DO_LIGHT_SAMPLING at run time (on by default, like the reference's Config.h). Takes effect with the next UpdateTest().
extern "C" void tpt_shim_set_light_sampling(int on) { s_LightSampling = on != 0; }
extern "C" tpt_context* tpt_shim_context() { return s_Ctx; }

// Test.cpp:240-246
void InitializeTest()
{
    if (s_Ctx) return;
    if (!s_SceneBuilt) buildScene();
    const char* m = getenv("TPT_MODE");
    if (m && !strcmp(m, "fast")) s_Mode = TPT_MODE_FAST;
    if (m && !strcmp(m, "exact")) s_Mode = TPT_MODE_EXACT;
    if (m && !strcmp(m, "refgpu")) s_Mode = TPT_MODE_REFGPU;
    if (m && !strcmp(m, "refgpu_fast")) s_Mode = TPT_MODE_REFGPU_FAST;
    const char* big = getenv("TPT_BIG_SCENE");
    const char* mit = getenv("TPT_MITSUBA");
    if (big || mit) tpt_shim_set_variant(big ? atoi(big) : (kSphereCount == 46), mit ? atoi(mit) : (int)s_Mitsuba);
    const char* ls = getenv("TPT_LIGHT_SAMPLING");
    if (ls) tpt_shim_set_light_sampling(atoi(ls));
    const char* d = getenv("TPT_DEVICE");
    int rc = tpt_create(d ? atoi(d) : 0, &s_Ctx);
    if (rc) die("tpt_create", rc);
    // A shell's backbuffer lives as long as the app (TestWin.cpp:73, Renderer.mm:148): page-locking it once lets
    // the per-frame copies run at full PCIe rate. Opt-in because the buffer must outlive the context.
    // DrawTest is called frame after frame: in exact mode let consecutive calls share trace launches (adaptive frame
    // lookahead, bit-identical pixels and ray counts; TPT_EXACT_LOOKAHEAD=0 switches it off, N > 1 fixes the window)
    const char* la = getenv("TPT_EXACT_LOOKAHEAD");
    tpt_set_option(s_Ctx, "exact_lookahead", la ? atoi(la) : -1);
    const char* pin = getenv("TPT_PIN_BACKBUFFER");
    if (pin && atoi(pin)) tpt_set_option(s_Ctx, "register_host", 1);
}

// Test.cpp:248-253
void ShutdownTest()
{
    tpt_destroy(s_Ctx);
    s_Ctx = nullptr;
}

// Test.cpp:302-342
void UpdateTest(float time, int frameCount, int screenWidth, int screenHeight, unsigned testFlags)
{
    (void)frameCount;
    if (!s_SceneBuilt) buildScene();
    if (testFlags & kFlagAnimate)
    {
        s_Spheres[1].center[1] = cosf(time) + 1.0f;
        s_Spheres[8].center[2] = sinf(time) * 0.3f;
    }
    float distToFocus = 3;
    float aperture = s_Mitsuba ? 0.0f : 0.1f;    // Test.cpp:311-315
    if (kSphereCount == 46) aperture *= 0.2f;    // DO_BIG_SCENE, Test.cpp:316-318
    s_EmissiveSphereCount = 0;
    for (int i = 0; i < kSphereCount; ++i)
    {
        s_Spheres[i].invRadius = 1.0f / s_Spheres[i].radius; // Maths.h:359
        const Material& smat = s_SphereMats[i];
        if (smat.emissive[0] > 0 || smat.emissive[1] > 0 || smat.emissive[2] > 0)
            s_EmissiveSpheres[s_EmissiveSphereCount++] = i;
    }
    buildCamera(mk(0, 2, 3), mk(0, 0, 0), mk(0, 1, 0), 60, float(screenWidth) / float(screenHeight), aperture, distToFocus);
    if (s_Ctx)
    {
        tpt_set_option(s_Ctx, "mitsuba_compare", s_Mitsuba ? 1 : 0);
        tpt_set_option(s_Ctx, "light_sampling", s_LightSampling ? 1 : 0);
        int rc = tpt_set_scene(s_Ctx, s_Spheres, s_SphereMats, kSphereCount, &s_Cam, s_EmissiveSpheres, s_EmissiveSphereCount);
        if (rc) die("tpt_set_scene", rc);
    }
}

// Test.cpp:344-367
void DrawTest(float time, int frameCount, int screenWidth, int screenHeight, float* backbuffer, int& outRayCount, unsigned testFlags)
{
    (void)time;
    if (!s_Ctx) InitializeTest();
    long long rays = 0;
    int rc = tpt_draw(s_Ctx, frameCount, 1, screenWidth, screenHeight, 0, screenHeight, 1, 0,
                      backbuffer, 0, testFlags, s_Mode, &rays, nullptr, nullptr);
    if (rc) die("tpt_draw", rc);
    outRayCount = (int)rays; // one 4-spp frame stays below 2^31 up to 3840x2160 (SURVEY §9.9)
}

// Test.cpp:369-375
void GetObjectCount(int& outCount, int& outObjectSize, int& outMaterialSize, int& outCamSize)
{
    outCount = kSphereCount;
    outObjectSize = sizeof(Sphere);
    outMaterialSize = sizeof(Material);
    outCamSize = sizeof(Camera);
}

// Test.cpp:377-384
void GetSceneDesc(void* outObjects, void* outMaterials, void* outCam, void* outEmissives, int* outEmissiveCount)
{
    memcpy(outObjects, s_Spheres, kSphereCount * sizeof(s_Spheres[0]));
    memcpy(outMaterials, s_SphereMats, kSphereCount * sizeof(s_SphereMats[0]));
    memcpy(outCam, &s_Cam, sizeof(s_Cam));
    memcpy(outEmissives, s_EmissiveSpheres, s_EmissiveSphereCount * sizeof(s_EmissiveSpheres[0]));
    *outEmissiveCount = s_EmissiveSphereCount;
}
