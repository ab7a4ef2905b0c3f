/* libtoytest_b200.so — the drop-in for the reference's Cpp/Source/Test.cpp (toypathtracer_b200/csrc/test_shim.cpp).
 *
 * The six functions below are the reference's own API, Cpp/Source/Test.h:10-17, with identical C++ signatures (C++
 * linkage: a reference shell includes ITS Test.h and links this library instead of Test.cpp + Maths.cpp + enkiTS).
 * They are repeated here only to document the boundary; the extern "C" functions after them are the additions a
 * shell may call to pick what the reference selects at compile time. */
#ifndef TPT_TEST_SHIM_H
#define TPT_TEST_SHIM_H

#include "tpt_b200.h"

#ifdef __cplusplus
/* Cpp/Source/Test.h:4-8 */
/* enum TestFlags { kFlagAnimate = (1 << 0), kFlagProgressive = (1 << 1) }; */
void InitializeTest();                                                                         /* Test.h:10 */
void ShutdownTest();                                                                           /* Test.h:11 */
void UpdateTest(float time, int frameCount, int screenWidth, int screenHeight, unsigned testFlags);                 /* Test.h:13 */
void DrawTest(float time, int frameCount, int screenWidth, int screenHeight, float* backbuffer, int& outRayCount,
              unsigned testFlags);                                                             /* Test.h:14 */
void GetObjectCount(int& outCount, int& outObjectSize, int& outMaterialSize, int& outCamSize); /* Test.h:16 */
void GetSceneDesc(void* outObjects, void* outMaterials, void* outCam, void* outEmissives, int* outEmissiveCount);   /* Test.h:17 */

extern "C" {
#endif

/* Mode DrawTest() renders in: TPT_MODE_EXACT (default; bit-identical to the reference), TPT_MODE_FAST, TPT_MODE_REFGPU,
 * TPT_MODE_REFGPU_FAST. Environment equivalent: TPT_MODE=exact|fast|refgpu|refgpu_fast. */
void tpt_shim_set_mode(int mode);
/* The reference's compile-time scene switches at run time: DO_BIG_SCENE (Test.cpp:10-11; 46 vs 9 spheres) and
 * DO_MITSUBA_COMPARE (Config.h:25; constant sky, zero Metal roughness, zero aperture). Rebuilds the scene tables; takes
 * effect with the next UpdateTest(). Environment: TPT_BIG_SCENE=0|1, TPT_MITSUBA=0|1. */
void tpt_shim_set_variant(int bigScene, int mitsubaCompare);
/* The reference's third compile-time switch, DO_LIGHT_SAMPLING (Config.h:24), at run time: on (default) = explicit light
 * sampling with shadow rays; off = a plain path tracer that adds every hit's emission (Test.cpp:95-133 and :209-215
 * compiled out). UpdateTest() passes it to tpt_set_option("light_sampling") before every tpt_set_scene(); takes effect
 * with the next UpdateTest(). Environment: TPT_LIGHT_SAMPLING=0|1. */
void tpt_shim_set_light_sampling(int on);
/* Restores the un-animated scene (the reference keeps animated positions in its static arrays, Test.cpp:304-308). */
void tpt_shim_reset_scene(void);
/* The C-ABI context behind the shim (NULL before InitializeTest()), for tpt_set_option() etc. */
tpt_context* tpt_shim_context(void);

#ifdef __cplusplus
}
#endif
#endif
