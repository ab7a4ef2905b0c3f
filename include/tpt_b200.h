/* tpt_b200 — C-ABI of the CUDA-native ToyPathTracer hot path (H100, sm_90a).
 *
 * This library replaces what the reference's DrawTest() does on the CPU (Cpp/Source/Test.cpp:344-367 ->
 * TraceRowJob :266-300 -> Trace :195-234 -> HitWorld/HitSpheres Maths.cpp:50-203 -> Scatter :83-193) with
 * hand-written sm_90a CUDA kernels. It sits exactly where the reference's own GPU back-ends sit: the shell
 * calls UpdateTest(), pulls the scene with GetObjectCount()/GetSceneDesc() (raw 20 B Sphere / 36 B Material /
 * 88 B Camera structs + emissive id list, Cpp/Windows/TestWin.cpp:258-283) and dispatches a kernel instead of
 * DrawTest(). Plain pointers and sizes only; every function returns 0 on success or a CUDA error code
 * (tpt_last_error() gives the text). There is no CPU fallback: without a CUDA device tpt_create() fails.
 *
 * A drop-in C++ translation unit exporting the six functions of Cpp/Source/Test.h on top of this ABI is
 * toypathtracer_b200/csrc/test_shim.cpp (see INTEGRATION.md).
 */
#ifndef TPT_B200_H
#define TPT_B200_H

#ifdef __cplusplus
extern "C" {
#endif

typedef struct tpt_context tpt_context;

/* Rendering modes.
 * TPT_MODE_EXACT  bit-identical to the reference C++ path: per-(frame,row) XorShift32 streams (Test.cpp:280),
 *                 no FMA contraction, glibc-faithful sinf/cosf/powf, back-to-front colour fold. Same pixels,
 *                 same ray counts.
 * TPT_MODE_FAST   same estimator, one RNG stream per (pixel, sample, frame); statistically equivalent image and
 *                 rays/sample. Throughput mode. */
#define TPT_MODE_EXACT 0
#define TPT_MODE_FAST 1
/* TPT_MODE_REFGPU       the estimator of the reference's own GPU back-ends (Cpp/Windows/ComputeShader.hlsl:353-395 and the
 *                       Metal port): per-PIXEL seed (x*1973 + y*9277 + frames*26699)|1, analytic disk/sphere samplers,
 *                       saturating schlick, <= 10 path segments, lerp(col, prev, f) blend, alpha written as 1 — for like-
 *                       for-like comparison with the reference's published D3D11/Metal numbers (readme.md:64-77). Strict
 *                       IEEE arithmetic: bit-equal to the CPU restatement oracle/refgpu_restate.cpp.
 * TPT_MODE_REFGPU_FAST  the same with GPU-native arithmetic (FMA, MUFU), as a real shader compiler would emit. */
#define TPT_MODE_REFGPU 2
#define TPT_MODE_REFGPU_FAST 3

/* testFlags of Cpp/Source/Test.h:4-8 */
#define TPT_FLAG_ANIMATE 1u
#define TPT_FLAG_PROGRESSIVE 2u

/* Replaces InitializeTest() (Test.cpp:240-246, which only creates the CPU task scheduler): binds a context to
 * CUDA device `device`. */
int tpt_create(int device, tpt_context** out);
/* Replaces ShutdownTest() (Test.cpp:248-253). */
void tpt_destroy(tpt_context* ctx);
int tpt_device_count(void);
const char* tpt_last_error(tpt_context* ctx);

/* Takes exactly what GetSceneDesc() exports (Test.cpp:377-384): `count` 20 B spheres, `count` 36 B materials,
 * one 88 B camera, the emissive sphere ids (Test.cpp:321-338). emissives == NULL derives the list from the
 * materials the way UpdateTest does; ids outside [0,count) or a negative count are refused. invRadius is recomputed
 * (Maths.h:359). Call after every UpdateTest(). The call never blocks on the GPU: the packed scene goes through a
 * pinned staging buffer into the one of two device copies that no draw in flight reads (the per-frame
 * UpdateSubresource of Cpp/Windows/TestWin.cpp:261-283 as an async double-buffered upload); draws issued afterwards
 * wait for it on the device. Bytes identical to the scene already resident are not uploaded again. */
int tpt_set_scene(tpt_context* ctx, const void* spheres20, const void* materials36, int count,
                  const void* camera88, const int* emissives, int emissiveCount);
/* Environment lighting for the fast mode: a lat-long (equirectangular) radiance map that replaces the sky. While it is
 * set, every path of a TPT_MODE_FAST tpt_draw (all fast variants), tpt_trace_rays, tpt_trace_irradiance,
 * tpt_draw_samples and tpt_trace_samples that leaves the scene adds the map's radiance in its direction instead of the
 * reference's gradient sky or "mitsuba_compare"'s constant sky ("mitsuba_compare"'s zero Metal roughness still applies).
 * By default the map is reached by bounce rays only, like the sky, so "light_sampling" on and off both stay unbiased;
 * "environment_sampling" (tpt_set_option) adds an importance-sampled direction towards it at Lambert vertices, for which
 * this call also builds the map's sampling tables. tpt_draw_aovs and tpt_trace_aovs are unaffected (a miss stays zeros and id -1). tpt_draw in
 * TPT_MODE_EXACT, TPT_MODE_REFGPU and TPT_MODE_REFGPU_FAST is refused while a map is set: those modes reproduce the
 * reference, which has no environment.
 *   rgba      width * height float4 texels, row-major, row 0 at the zenith (+y): an image stored top row first is
 *             upright. Alpha is ignored; R, G and B must be finite and not negative (sign
 *             bit clear, so -0 is refused too). NULL removes the environment (the calls that
 *             follow see the reference sky again).
 *   onDevice  0: host memory; 1: device memory of the context's device, 16-byte aligned, whose contents are complete
 *             when the call is made (a small kernel checks the texels there).
 * Refused, with tpt_last_error text: width or height below 1, width * height >= 2^31, a misaligned device buffer or one
 * on another device, a texel with a negative or non-finite R, G or B (the error names it). A refused map leaves the environment as it was.
 * The call copies the texels and returns once they have been read, so the caller may free or reuse its buffer; it is a
 * set-up call that may block. Calls issued before it keep the environment they were issued with, even while in flight,
 * and calls issued after it see the new one, without any synchronisation by the caller (two device copies, as for the
 * scene). The environment belongs to the context: tpt_set_scene keeps it, tpt_destroy frees it.
 * Mapping of a unit direction d (fast module, env_radiance):
 *   phi = atan2f(d.x, -d.z), theta = acosf(clamp(d.y, -1, 1)),
 *   u = (phi + pi) / (2 pi) * width, v = theta / pi * height (continuous texel coordinates),
 *   texel (i, j) has its centre at (i + 1/2, j + 1/2); bilinear filtering, columns wrap, rows clamp; every blend is
 *   a + f * (b - a), so a constant map returns its constant exactly.
 * The map's centre column lies along -z (where the reference camera looks), +x to its right: the reference view shows the
 * map unmirrored.
 * Memory: each of the two device copies holds the texels and the sampling tables behind them, 24 * width * height +
 * 8 * height bytes (the texels' alpha carries each cell's sampling probability; toypathtracer_b200/csrc/tpt_env_tables.h
 * pins the tables).
 * While a map is set, the slab queue runs its 6-CTA instances where it would pick the 8-CTA ones (long draws and caller
 * calls, "fast_variant" 9): those have no lookup, which would make them spill at 64 registers. */
int tpt_set_environment(tpt_context* ctx, const float* rgba, int width, int height, int onDevice);
/* Albedo textures for the fast mode: lat-long images bound to spheres by sphere id (which is also the material id). While
 * they are set, every hit of a TPT_MODE_FAST tpt_draw, tpt_trace_rays, tpt_trace_irradiance, tpt_draw_samples and
 * tpt_trace_samples on a textured sphere uses albedo x T(n) wherever the untextured estimator uses the material's albedo:
 * a Lambert vertex's throughput (its light cones, its environment sample and its bounce, with "light_sampling" on or off)
 * and a Metal vertex's tint. Glass uses no albedo; emission has textures of its own (tpt_set_emission_textures). The
 * lookup draws no random numbers, so every sample stream stays where it was. tpt_trace_irradiance's starting vertex stays white; later vertices on textured
 * spheres are textured. tpt_draw_aovs and tpt_trace_aovs report the textured albedo for every material type.
 *   n         the hit's shading normal (pos - centre) / radius.
 *   T(n)      the bilinear lookup of the sphere's layer in the direction n, with the mapping tpt_set_environment pins:
 *             phi = atan2f(n.x, -n.z), theta = acosf(clamp(n.y, -1, 1)), texel centres at (i + 1/2, j + 1/2), columns
 *             wrap, rows clamp, every blend a + f * (b - a) (a constant layer returns its constant exactly). Row 0 is at the
 *             sphere's +y pole, the centre column along -z and +x to its right.
 *   rgba      layers * height * width float4 texels, layer-major, then row-major. All layers share width x height (resample
 *             textures of other sizes). Alpha is ignored; R, G and B must be finite and not negative (-0 is refused too).
 *             NULL removes the textures.
 *   sphereLayers  numSpheres int32 in HOST memory: entry i is the layer of sphere i, or -1 for none. Sphere ids at or past
 *             numSpheres, and the padding spheres of the sweep, are untextured.
 *   onDevice  0: host texels; 1: device texels of the context's device, 16-byte aligned, complete when the call is made (a
 *             small kernel checks them there). sphereLayers is host memory either way.
 * Refused, with tpt_last_error text naming the offending value: width, height or layers below 1, width * height * layers
 * >= 2^31, numSpheres < 0, a layer outside [-1, layers), a texel with a negative or non-finite R, G or B (the error names
 * its layer, x and y), a misaligned device buffer or one on another device. A refused call leaves the textures as they were.
 * Lifetime and ordering are tpt_set_environment's: a set-up call that may block and returns once the texels have been
 * read; calls issued before it keep the textures they were issued with, even while in flight; tpt_set_scene keeps them,
 * tpt_destroy frees them. Memory: two device copies of 16 * width * height * layers + 4 * numSpheres bytes at most.
 * Kernels: only the slab queue's reference-form (sweep form 0) 6-CTA and 768-thread instances carry the lookup, so that no
 * instance an untextured call runs does. While textures are set every fast call runs them: tpt_draw's auto variant is 3
 * (host-buffer draws stage through the slab queue instead of storing into page-locked memory), 9 runs the 6-CTA instance,
 * and an explicit "fast_variant" 0, 1, 2, 4, 5, 6, 7 or 8 is refused. tpt_draw in TPT_MODE_EXACT, TPT_MODE_REFGPU and
 * TPT_MODE_REFGPU_FAST is refused: those modes reproduce the reference, which has no textures. Textures and
 * "environment_sampling" run in the same instances and combine. */
int tpt_set_textures(tpt_context* ctx, const float* rgba, int width, int height, int layers,
                     const int* sphereLayers, int numSpheres, int onDevice);
/* Emission textures for the fast mode: lat-long images bound to spheres by sphere id, the matching half of
 * tpt_set_textures. While they are set, the emitted radiance of a hit on sphere id with shading normal n is
 * emissive[id] x T(n), with T(n) the same bilinear lookup (mapping, orientation, blends) as tpt_set_textures' layers.
 * It applies wherever a TPT_MODE_FAST tpt_draw, tpt_trace_rays, tpt_trace_irradiance, tpt_draw_samples and
 * tpt_trace_samples add emission: a camera or caller ray's first hit, hits after Metal and glass bounces, Lambert hits
 * with "light_sampling" 0, the ends of a path absorbed by Metal or failed by glass, the depth cap, and a light cone's
 * shadow ray that reaches its light. There T is evaluated at the normal of the point where the shadow ray meets the
 * light (not at the cone's axis or the sampled direction). The products are taken in that order: emissive x T first,
 * then the throughput times that (on a light's shadow ray (throughput x albedo x (emissive x T)) x the cone's weight), so
 * a constant layer c gives the bits of the untextured scene whose emission is emissive x c rounded to float.
 * A sphere whose material emission is zero stays dark whatever its layer: the light list, and with it the set of spheres
 * light sampling aims at, stays the one tpt_set_scene made, so the estimator stays unbiased with cone sampling left as it
 * is (uniform in the light's subtended cone; only its variance depends on the texture). The lookup draws no random
 * numbers, so every sample stream stays where it was. Spheres without a layer (-1), ids at or past numSpheres and the
 * padding spheres of the sweep keep emissive[id]. tpt_draw_aovs and tpt_trace_aovs do not change, nor do
 * tpt_trace_irradiance's self-skip rule and environment sampling. Albedo and emission textures on one sphere combine, each
 * acting on its own term.
 * "emission_texture_sampling" (tpt_set_option) adds a sample drawn from a light's layer to its cone sample, from sampling
 * tables this call builds on the host for every layer (device texels are copied back for it).
 * Arguments, refusals (with the same error texts, headed tpt_set_emission_textures), NULL to remove, lifetime, ordering
 * and kernels are those of tpt_set_textures. Memory: two device copies of 24 * width * height * layers +
 * 8 * height * layers + 4 * numSpheres bytes (+ 4 when numSpheres is odd) at most: the texels (their alpha holds each
 * cell's sampling probability), the sphere table and the sampling tables (toypathtracer_b200/csrc/tpt_env_tables.h). The
 * two calls are independent: each has its own size, layers and sphere table, and either can
 * be made without the other. While emission textures are set every fast call runs the instances that carry the lookups:
 * tpt_draw's auto variant is 3 (host-buffer draws stage through the slab queue), 9 runs the 6-CTA instance, an explicit
 * "fast_variant" 0, 1, 2, 4, 5, 6, 7 or 8 is refused, and tpt_draw in TPT_MODE_EXACT, TPT_MODE_REFGPU and
 * TPT_MODE_REFGPU_FAST is refused. */
int tpt_set_emission_textures(tpt_context* ctx, const float* rgba, int width, int height, int layers,
                              const int* sphereLayers, int numSpheres, int onDevice);
/* Homogeneous participating media inside glass spheres for the fast mode: tinted or milky glass, smoke, jade.
 *   media5    numSpheres records of 5 floats in HOST memory, {sigma_a.r, sigma_a.g, sigma_a.b, sigma_s, g}: record i is
 *             the medium inside sphere i. sigma_a is the absorption coefficient per colour channel and sigma_s the grey
 *             scattering coefficient, both per world unit; g is the Henyey-Greenstein asymmetry (g > 0 scatters forward).
 *             A record whose sigma_a and sigma_s are all zero is "no medium". Sphere ids at or past numSpheres or the
 *             scene's count, and the padding spheres of the sweep, have none. NULL or numSpheres 0 removes all media.
 * A medium acts only inside a sphere whose material is glass; on any other sphere it is kept but has no effect (a later
 * tpt_set_scene may make that sphere glass). Estimator: a path ray whose segment of length t ended on the inside face
 * (dot(d, normal) > 0) of a glass sphere with a medium, before the depth cap is tested and before any emission is added,
 *   1. with sigma_s > 0 draws u and takes t_s = -ln(1 - u) / sigma_s (finite: u <= 1 - 2^-24); with sigma_s = 0 draws
 *      nothing (t_s = +inf);
 *   2. t_s < t: scatters at o + d t_s. Past the depth cap the path ends and adds nothing (a medium emits nothing);
 *      otherwise the throughput takes exp(-sigma_a t_s) per channel, the direction becomes a Henyey-Greenstein sample
 *      around d from two more draws xi1 (cos theta) and xi2 (phi = 2 pi xi2), the depth grows by one, and the next hit
 *      adds its emission. The hit itself is not shaded. The continuation is an ordinary path ray, traced and counted.
 *      cos theta = (1 + g^2 - s^2) / (2 g), s = (1 - g^2) / (1 - g + 2 g xi1), clamped to [-1, 1], when |g| >= 1e-3;
 *      1 - 2 xi1 otherwise;
 *   3. t_s >= t: the throughput takes exp(-sigma_a t) and the hit is shaded as without media.
 * Absorption is applied continuously and scattering sampled exactly, so the estimator is unbiased with RGB sigma_a and
 * no ratio weights. A path none of whose segments ends on the inside face of a glass sphere with sigma_s > 0 draws the
 * same random numbers as without media; a medium with sigma_s = 0 draws none. No light sampling at medium vertices.
 * Limits: the medium of a segment is that of the sphere whose inside face it ends on (a segment inside a glass sphere
 * that ends on the outside of a sphere nested in it runs in vacuum); scatter events count against the depth cap, so
 * dense media lose energy to it at the default cap of 10: the option "max_depth" (tpt_set_option) raises it, with Russian
 * roulette past depth 10.
 * Refused, with tpt_last_error text naming the sphere and the field ("tpt_set_media: sphere 3 has sigma_s = -1"):
 * numSpheres < 0, a non-finite sigma or one with its sign bit set (-0 included), a g that is NaN or has |g| >= 1. A
 * refused call leaves the media as they were.
 * Lifetime and ordering: the media belong to the context; tpt_set_scene keeps them and applies them to the new scene's
 * ids, and before any scene they are stored for the first one. The call re-packs the current scene with a media section
 * and uploads it as tpt_set_scene does (tpt_last_scene_upload_bytes reports that upload): it never blocks on the GPU,
 * calls issued before it keep the media they were issued with, even while in flight, and calls issued after it see the
 * new ones. A scene none of whose spheres has a medium keeps the bytes of its blob and every call its default kernel.
 * Only TPT_MODE_FAST uses media. While the current scene has one, every fast call (tpt_draw, tpt_trace_rays,
 * tpt_trace_irradiance, tpt_draw_samples, tpt_trace_samples) runs the slab queue's reference-form instances that carry
 * the textures: tpt_draw's auto variant is 3, 9 runs the 6-CTA instance, an explicit "fast_variant" 0, 1, 2, 4, 5, 6, 7
 * or 8 is refused, and tpt_draw in TPT_MODE_EXACT, TPT_MODE_REFGPU and TPT_MODE_REFGPU_FAST is refused. Media combine
 * with textures, "environment_sampling" and "emission_texture_sampling". tpt_draw_aovs and tpt_trace_aovs, which record
 * first hits, do not change. */
int tpt_set_media(tpt_context* ctx, const float* media5, int numSpheres);
/* Homogeneous fog in the air between the spheres for the fast mode, lit by the lights: beams, glows around lamps, haze.
 *   fog9      9 floats in HOST memory, {c.x, c.y, c.z, R, sigma_a.r, sigma_a.g, sigma_a.b, sigma_s, g}: the fog fills the
 *             ball B = {c, R} minus the scene's spheres. sigma_a is the absorption coefficient per colour channel and
 *             sigma_s the grey scattering coefficient, both per world unit; g is the Henyey-Greenstein asymmetry. NULL, or
 *             a record whose sigmas are all zero, removes the fog.
 * Which segments are in air: a ray segment [o, o + t d] runs in air when it ends on the outside face of a sphere
 * (dot(d, normal) <= 0) or leaves the scene (t = TPT_MAX_T); this holds for path rays and every kind of shadow ray. A
 * segment that ends on an inside face runs in that sphere (tpt_set_media's rule). The fog length of a segment in air is
 * L = |[0, t] ∩ [t_in, t_out]|, the part of it inside B.
 * Estimator: a path ray's segment in air, after the "max_depth" roulette on a hit and before the depth cap is tested and
 * any emission or sky is added (a miss takes no roll),
 *   1. with L > 0 and sigma_s > 0 draws u and takes t_s = -ln(1 - u) / sigma_s, measured along the fog part of the
 *      segment; with sigma_s = 0 it draws nothing and the throughput takes exp(-sigma_a L);
 *   2. t_s < L: the path scatters at o + d (max(t_in, 0) + t_s) and the throughput takes exp(-sigma_a t_s). Past the
 *      depth cap the path ends and adds nothing; otherwise the depth grows by one, once per event. With light sampling
 *      off two draws xi1, xi2 give the direction hg_sample(d, g, xi1, xi2) (tpt_set_media's HG sample) and the next hit
 *      adds its emission. With it on, the vertex works like a Lambert vertex with the phase function
 *      p(cos) = (1 - g^2) / (4 pi (1 + g^2 - 2 g cos)^(3/2)) (exactly 1 / (4 pi) for |g| < 1e-3) for cos / pi: first the
 *      HG direction is drawn (xi1, xi2) and kept; then every light in order (none is excluded) takes one cone sample
 *      (2 draws) and its shadow ray, which, when it reaches light j, adds thr E_j omega p(dot(d, l)) T_shadow; then the
 *      path bounces along the kept direction, and emission after the bounce follows the rule after a Lambert vertex.
 *      Fog vertices take no "environment_sampling" sample (their bounce's miss keeps full weight) and no
 *      "emission_texture_sampling" sample (their cone rays keep full weight and still take the emission texture's
 *      lookup where they meet the light);
 *   3. t_s >= L: the throughput takes exp(-sigma_a L) and the hit or miss is handled as without fog.
 * The rays that leave a fog scatter point (its cone rays and its continuation) take hits from distance 0 rather than
 * TPT_MIN_T: the point lies in air but may lie within TPT_MIN_T of a surface, which they must not skip.
 * Every shadow ray in air (Lambert and fog-vertex cones, environment samples that miss, emission-texture samples) takes
 * T_shadow = exp(-(sigma_a + sigma_s) L) per channel and draws nothing. A path that never crosses B with sigma_s > 0 draws
 * the same random numbers as without fog.
 * Limit: a segment inside a glass sphere that ends on the outside of a sphere nested in it counts as air.
 * Refused, with tpt_last_error text naming the field ("tpt_set_fog: radius = -1"): a non-finite centre; a radius that is
 * not finite or not > 0; a sigma that is non-finite or has its sign bit set (-0 included); a g that is NaN or has
 * |g| >= 1. A refused call leaves the fog as it was.
 * Lifetime and ordering are tpt_set_media's: the fog belongs to the context, tpt_set_scene keeps it, a fog set before any
 * scene is stored for the first one, and the call re-packs the current scene with a fog section and uploads it as
 * tpt_set_scene does (identical bytes are not uploaded again; tpt_last_scene_upload_bytes reports the upload). It never
 * blocks on the GPU, and calls issued before it keep the fog they were issued with, even while in flight.
 * Only TPT_MODE_FAST uses fog. While it is set, every fast call (tpt_draw, tpt_trace_rays, tpt_trace_irradiance,
 * tpt_draw_samples, tpt_trace_samples) runs the slab queue's reference-form instances that carry the textures: an
 * explicit "fast_variant" other than -1, 3 or 9 is refused, and so is tpt_draw in TPT_MODE_EXACT, TPT_MODE_REFGPU and
 * TPT_MODE_REFGPU_FAST. Fog combines with media, textures, "max_depth", "environment_sampling" and
 * "emission_texture_sampling". tpt_draw_aovs and tpt_trace_aovs, which record first hits, do not change. */
int tpt_set_fog(tpt_context* ctx, const float* fog9);
/* Camera only (UpdateTest rebuilds it every frame from the aspect ratio, Test.cpp:341). */
int tpt_set_camera(tpt_context* ctx, const void* camera88);

/* DO_SAMPLES_PER_PIXEL (Config.h:22), default 4. */
int tpt_set_spp(tpt_context* ctx, int spp);
/* Implementation knobs (benchmarks/tests): "fast_variant" (-1 auto (default): 3 for device buffers (7 from 1024 spheres when the packed pair array does not fit in shared memory), 8 for host-buffer
 * draws that can store straight into page-locked memory; 0 megakernel, 1/2 persistent tiles, 3/4 persistent slab queue with 128-bit L2
 * reductions (3 picks its 8-CTA/SM 64-register instance by itself for long draws; 9 forces that instance), 5 CTA-owned tiles,
 * 6/7 block wavefront with material sort, 8 warp-owned pixel groups with coalesced 128-bit write-out), "host_zero_copy" (default 1: with variant 8 a host-buffer draw whose `prev` has zero weight writes its finished
 * pixels directly into the caller's page-locked buffer over PCIe — no staging image, no device-to-host copy), "exact_lanes"
 * (0 auto; 64..67 = split kernel: one PATH warp per (frame,row) chain walks the RNG stream, 1..4 SHADE warps do the light
 * sampling / fold / blend off the critical path (auto for <= 2400 chains); 32 or 8 lanes per chain as nested loops; 1 = one
 * thread per chain as a flat one-sweep-per-step state machine (auto for >= 100 000 chains); 2 = one thread per chain
 * nested, 9 = 8 lanes flat: measured slower, kept for comparison; 68/69 timing probes; 70 = the split kernel as 2-CTA
 * clusters with the roles on different SMs and the rings over DSMEM, 71 = shade warps calling out-of-line libm: both measured
 * slower, kept for comparison), "register_host" (1: page-lock the caller's host backbuffer with cudaHostRegister the first
 * time it is seen so both copies run at full PCIe rate; only safe when the buffer outlives the context, as a
 * reference shell's does; default 0 — buffers that are already pinned are detected by CUDA on their own), "host_bands" (1..8, default 3:
 * host-buffer fast draws are split into row bands on separate streams so the D2H of one band overlaps the tracing of
 * the next), "host_progress" (default 1: with fast variant 3/4/9 a single kernel publishes per-band completion counters and the
 * copy stream waits on them with cuStreamWaitValue32, "progress_bands" bands, default 4; 0 falls back to host_bands),
 * "fast_kform" (fast kernels' sphere sweep: 0 reference form, 1 expanded form, 2 (default) expanded form on a pair-interleaved
 * sphere array, one 128-bit shared load per coordinate of two spheres — the slab queue of a scene of at most 64 padded
 * spheres takes that array in its kernel parameters instead, so its first pass reads the spheres as constant operands,
 * and where the scene passes the half-precision gate its first pass tests two spheres per packed half instruction with a
 * folded-in error bound (same hits and distances); 4 as 2 but without that half-precision first pass, for A/B comparisons;
 * 3 as 2 but with the array always in shared memory, for A/B comparisons; 1 to 4 only when the scene passes the gate in
 * tpt_set_scene — a scene that fails it gets, with 2 to 4, the packed sweep made conservative by a folded-in error bound
 * plus reference-form hit decisions, and the reference form otherwise; per context), "fast_alpha_zero" (default 0; 1: fast-mode draws whose `prev` has zero weight write
 * alpha = 0 instead of keeping the buffer's alpha — saves the read over NVLink when the buffer is a peer GPU's),
 * "exact_lookahead" (default 0; L > 1: an exact-mode draw of ONE frame that misses the cache traces frames [f, f+L) in a
 * single launch and keeps their per-frame colours; the calls for the following frames only blend their cached frame into
 * the caller's buffer. Bit-identical results and per-frame ray counts; trades L frames of latency on a miss for batch
 * throughput (one 720p frame alone cannot fill the GPU: `height` serial RNG chains). Never used with kFlagAnimate; any
 * scene / camera / size / row-range / spp change invalidates the cache. -1 = adaptive: the first call traces one frame,
 * and every time the caller has walked to the end of the cached window and asks for the frame right after it, the next
 * window doubles (1, 2, 4, 8, 16 frames) — no first-call latency; the Test.h shim sets this, TPT_EXACT_LOOKAHEAD overrides),
 * "scene_upload_always" (default 0; 1: tpt_set_scene uploads the scene blob even when its bytes equal the resident scene's —
 * bench.py's end-to-end leg, so that every step carries its host -> device copy),
 * "mitsuba_compare" (default 0; DO_MITSUBA_COMPARE of Config.h:25 as a runtime switch, applied by the NEXT
 * tpt_set_scene: constant sky (0.15, 0.21, 0.3) (Test.cpp:226-227) and zero Metal roughness (Test.cpp:143-145); the
 * switch's third effect, zero aperture (Test.cpp:312-313), is camera data: the Test.h shim's UpdateTest applies it),
 * "light_sampling" (default 1; 0 = DO_LIGHT_SAMPLING 0 of Config.h:24 as a runtime switch, applied by the NEXT
 * tpt_set_scene: no explicit light sampling at Lambert vertices (no light draws, no shadow rays, Test.cpp:95-133) and
 * every hit adds its emission (the doMaterialE suppression of Test.cpp:209-215 is off). Exact and reference-GPU strict
 * modes stay bit-identical to the reference built that way. The flag is part of the scene: toggling it re-uploads the
 * scene and invalidates the exact_lookahead cache),
 * "environment_sampling" (default 0; any non-zero value is 1: fast calls importance-sample tpt_set_environment's map at
 * light-sampled Lambert vertices. After the light cones, such a vertex draws one direction from the map's tables
 * (proportional to sin theta times the brightest texel the bilinear filter can blend into each cell) and traces its
 * shadow ray, and the vertex's bounce, when it leaves the scene, is weighted against it with the power heuristic. An
 * estimator switch like "light_sampling", not a speed path: both are unbiased and their outputs differ. Read by each
 * call when it is issued, like the map, not a scene flag: toggling it uploads nothing. Active for a call only with the
 * option on, a map set, "light_sampling" on and a map with some non-zero weight; a call where it is not active runs
 * exactly as without it. While active: only the slab queue's reference-form (sweep form 0) instances sample, and every
 * fast call runs them (measured: the sampling code in the packed-sweep instances cost map-less draws 20 %); tpt_draw's
 * auto variant is 3 (never 7 or 8;
 * host-buffer draws stage through the slab queue instead of storing into page-locked memory), 9 runs the 6-CTA
 * instance, and an explicit "fast_variant" 0, 1, 2, 4, 5, 6, 7 or 8 is refused; Metal and glass vertices, Lambert
 * vertices hit from inside their sphere, the AOV calls and the exact and reference-GPU modes do not sample it),
 * "emission_texture_sampling" (default 0; any non-zero value is 1: fast calls importance-sample each light that has an
 * emission layer by that layer; an estimator switch like "environment_sampling": unbiased, outputs differ from the default;
 * read by each call when it is issued, not a scene flag, so toggling it uploads nothing. Active for a call (kSceneEmitSampling)
 * only with the option on, emission textures set, "light_sampling" on and some layer with a non-zero weight; a call where
 * it is not active runs exactly as without it (same kernel, streams and ray counts). At a light-sampled Lambert vertex o
 * with facing normal nl, each light j it samples (never its own sphere) whose sphere has a sampleable layer gets, right
 * after its cone sample (2 draws, its shadow ray traced as before), one texture sample: six draws in sample_env's order
 * (row, row alias test, column, column alias test, u offset, v offset) from the layer's tables give the unit normal n_x by
 * the inverse lat-long mapping and the point x = c + r n_x. Its shadow ray, along l = normalize(x - o), is traced (and
 * counted in the call's rays) only when x faces o (n_x . (o - x) > 0), m = l . nl > 0 and sin theta_x > 0; the next light
 * follows, then the environment sample, then the bounce. Densities in solid angle at o: the cone's pc = 1 / omega,
 * omega = 2 pi (1 - cos_max) as the cone sampler computes it, and the texture sample's
 * pt(x) = P_cell(n_x) W H / (2 pi^2 sin theta_x) / r^2 * |x - o|^2 / cos_x, cos_x = n_x . normalize(o - x), P_cell the
 * realised probability of the layer cell that holds x's (u, v). Weights, the power heuristic with one sample each: a cone ray that reaches
 * light j at x adds (throughput x albedo x (emissive x T(n_x))) x m omega / pi x pc^2 / (pc^2 + pt(x)^2); a texture ray
 * that reaches it adds the same product, T at the normal where it meets the light, times (m / pi) pt / (pt^2 + pc^2),
 * fixed when the sample is drawn (the kernels evaluate both with q = pt omega, which is the same value). A light without
 * a layer, with layer -1, or with a layer whose weights are all zero draws nothing extra and its cone ray keeps full
 * weight; so does every light at a vertex inside or on it (d <= r). Metal and glass vertices, "light_sampling" 0, the
 * AOV calls and the exact and reference-GPU modes are unchanged; tpt_trace_irradiance, tpt_draw_samples and
 * tpt_trace_samples sample as draws do. Tables: built by tpt_set_emission_textures for every layer whether or not the
 * option is on, as tpt_set_environment builds the map's: the same weights (sin theta x the 3 x 3 maximum of mean RGB), alias
 * tables and realised probabilities; they cost 8 * width * height * layers + 8 * height * layers bytes per device copy,
 * plus 4 bytes of padding behind an odd sphere table. Kernels and routing are emission textures': the slab queue's
 * reference-form 6-CTA and 768-thread instances),
 * "max_depth" (1..256, default 10, the reference's compile-time cap; out of range it is refused with "max_depth: 1..256"
 * and keeps its value: the fast estimator's path depth cap. Read by each call when it is issued, like
 * "environment_sampling", not a scene flag: setting it uploads nothing, and calls already issued keep the value they were
 * issued with. Depth counts Lambert bounces, Metal and glass continuations and medium scatter events. A path ray's hit at
 * depth >= max_depth adds its emission and ends the path, and a medium scatter event there ends it with nothing added.
 * Russian roulette, only when max_depth > 10: at every path ray's hit at depth >= 10, before the medium's draw, the cap
 * test and any emission, the path draws u from its own stream; with q = min(1, max(thr.r, thr.g, thr.b)) of its
 * throughput, u >= q ends it with nothing added, and otherwise the throughput becomes thr / q and the hit is shaded as
 * without the roll. Shadow rays and misses take no roll. So a path that ends before depth 10 draws the same numbers as
 * with the default, max_depth <= 10 draws nothing extra, and the roll is unbiased: a call with max_depth n converges to
 * the image with cap n. max_depth 10 is the default call exactly (kernels, streams, ray counts and bits). Applies to
 * tpt_draw in TPT_MODE_FAST, tpt_trace_rays, tpt_trace_irradiance (a point keeps a camera path's budget, from depth 0),
 * tpt_draw_samples and tpt_trace_samples; tpt_draw_aovs and tpt_trace_aovs, which record first hits, do not change.
 * While it is not 10 every such call runs the slab queue's reference-form 6-CTA and 768-thread instances: tpt_draw's auto
 * variant is 3, 9 runs the 6-CTA instance, an explicit "fast_variant" 0, 1, 2, 4, 5, 6, 7 or 8 is refused, and tpt_draw
 * in TPT_MODE_EXACT, TPT_MODE_REFGPU and TPT_MODE_REFGPU_FAST is refused (those keep the reference's 10 for parity; set
 * it back to 10 for them). It combines with media, textures, "environment_sampling" and "emission_texture_sampling"). */
int tpt_set_option(tpt_context* ctx, const char* key, int value);

/* Replaces DrawTest() (Test.cpp:344-367) for frames [frameCount, frameCount+numFrames) — numFrames*spp samples
 * per pixel accumulated with the reference's progressive blend (Test.cpp:272-276,293-295) — over the rows
 * y_i = row0 + i*rowStep, i in [0,numRows) (TraceRowJob's [start,end) generalised for multi-GPU sharding).
 *   backbuffer        width*height*4 floats, row 0 = bottom, RGBA; read as `prev` and updated in place exactly like
 *                     the reference's (Test.cpp:293-296; alpha is preserved). With `packed` != 0 the buffer holds
 *                     only the numRows rendered rows, back to back.
 *   bufferOnDevice    0: host pointer (copied in/out inside the call; the call is synchronous like DrawTest)
 *                     1: device pointer (work is enqueued on `cudaStream`, no host synchronisation unless a ray
 *                        count is requested)
 *   outRayCount       NULL or receives the number of rays (every HitWorld call: camera, bounce, shadow —
 *                     Test.cpp:122,199) of this call; 64-bit because 3840x2160x64 spp exceeds INT_MAX.
 *   outRaysPerFrame   NULL or numFrames entries (exact mode only; fast mode fills entry 0 with the total).
 *   cudaStream        a cudaStream_t (NULL = the context's own stream).
 * numRows == 0 is an empty shard: nothing is traced or copied, the ray counts are 0.
 * Alpha: never written in exact mode (Maths.h:38). Fast mode keeps it too, except for a HOST buffer drawn with zero
 * `prev` weight (flags without kFlagProgressive, or frame 0): `prev` is then not uploaded and the rendered rows get
 * alpha = 0 — what every reference shell's zero-initialised buffer holds (TestWin.cpp:73-74).
 * Ordering: a context owns one scene and one set of counters; its draws execute in issue order even when they are
 * enqueued on different streams (each draw waits on the previous draw's end event). Use one context per thread. */
int tpt_draw(tpt_context* ctx, int frameCount, int numFrames, int width, int height,
             int row0, int numRows, int rowStep, int packed,
             float* backbuffer, int bufferOnDevice, unsigned testFlags, int mode,
             long long* outRayCount, long long* outRaysPerFrame, void* cudaStream);

/* Fast-mode radiance estimates for n caller-supplied rays in the current scene — other projections (panoramas, fisheye,
 * orthographic, stereo), many small views in one launch, a sparse set of pixels, or rays made by torch code.
 *   rays6             n rays of 6 floats {o.xyz, d.xyz} (the layout of tpt_debug_hit); directions need not be unit length,
 *                     they are normalised on load. A device buffer may have any 4-byte alignment (a row slice of an
 *                     (N, 6) tensor is only 8-byte aligned).
 *   out4              n float4: out4[i] = (r, g, b, 0), the mean over `spp` samples of ray i's path radiance with the
 *                     estimator of TPT_MODE_FAST (scene options as for a fast draw: "light_sampling", "mitsuba_compare",
 *                     "fast_kform", scenes past 64 KB of blob). A device buffer must be 16-byte aligned. A ray with a
 *                     non-finite component, or whose direction does not normalise to a finite non-zero vector (zero
 *                     length, or a squared length that underflows or overflows float), is not traced: (0, 0, 0, 0).
 *   raysOnDevice / outOnDevice
 *                     0: host pointer, copied in / out inside the call, and the call is synchronous
 *                     1: device pointer of the context's device (or mapped host memory), used in place on `cudaStream`;
 *                        without host buffers the host only synchronises when a ray count is requested
 *   spp, frame        sample s of ray i draws from the stream pixel_seed(i * spp + s, frame) of the fast mode: the same
 *                     frame gives the same result, different frames independent ones, so averaging calls with frames
 *                     0, 1, 2, ... refines the estimates progressively. n * spp must not exceed 2^32.
 *   outRayCount       NULL or receives the number of rays traced (path and shadow rays; untraced rays add none).
 *   cudaStream        a cudaStream_t (NULL = the context's own stream).
 * n == 0 launches nothing and reports 0 rays. The draw's blend and `prev` play no part. Ordering and accounting are those
 * of tpt_draw: the call runs after the context's previous draw (or trace) and after the scene upload, and counts toward
 * tpt_read_ray_count, tpt_last_kernel_ms and tpt_last_launch_count. Null pointers, n < 0, spp < 1, n * spp > 2^32, a
 * misaligned device buffer or one on another device are refused (tpt_last_error gives the reason). */
int tpt_trace_rays(tpt_context* ctx, const float* rays6, int raysOnDevice, long long n, int spp, int frame,
                   float* out4, int outOnDevice, long long* outRayCount, void* cudaStream);

/* Fast-mode irradiance E(p, n) at n caller-supplied surface points: the light arriving over the hemisphere around the normal
 * n at p, what lightmaps and irradiance probes store, or the second pass of a renderer that takes its first hits from
 * tpt_trace_aovs.
 *   points6           n points of 6 floats {p.xyz, n.xyz}, the layout of rays6, loaded, validated and normalised exactly as
 *                     tpt_trace_rays loads rays (same alignment). A point with a non-finite component, or a normal that does
 *                     not normalise, is not traced: (0, 0, 0, 0), and it adds no rays.
 *   ids               NULL, or n int32 sphere ids (host or device like points6, 4-byte aligned): point i lies on sphere
 *                     ids[i], whose light is then not sampled from it (a light never samples itself). Any other value, -1
 *                     included, has no effect; the id is only compared, never used as an index. A point on an emissive
 *                     sphere must pass that sphere's id: otherwise it samples its own sphere as a light, which costs a
 *                     shadow ray per sample and is not the estimator a draw's vertex on that sphere uses.
 *   out4              n float4: out4[i] = (E.r, E.g, E.b, 0), pi x the mean over `spp` samples of the radiance a white
 *                     Lambert surface at (p, n) reflects, with the estimator and scene options of tpt_trace_rays. Each
 *                     sample is a Lambert vertex that a camera path has just reached at p, facing n: it draws its bounce
 *                     direction, then samples the lights' cones with shadow rays, then continues along the bounce with the
 *                     depth budget of a camera path after its first hit; the vertex adds no emission of its own. So for
 *                     a camera ray whose first hit is a Lambert sphere `id` at (p, n), the expected tpt_trace_rays value
 *                     is Le[id] + albedo[id] * E(p, n, id) / pi.
 *   spp, frame        sample s of point i draws from the stream pixel_seed(i * spp + s, frame), as for tpt_trace_rays.
 *   outRayCount       NULL or receives the number of rays traced: shadow rays, the bounce and the path's later rays. The
 *                     point itself is not a ray.
 * Buffers, streams, limits, refusals, ordering and accounting (tpt_read_ray_count, tpt_last_kernel_ms,
 * tpt_last_launch_count, tpt_debug_last_kernels) are those of tpt_trace_rays; n == 0 launches nothing. */
int tpt_trace_irradiance(tpt_context* ctx, const float* points6, const int* ids, int pointsOnDevice, long long n,
                         int spp, int frame, float* out4, int outOnDevice, long long* outRayCount, void* cudaStream);

/* First-hit AOVs (arbitrary output values) of the fast mode: the denoiser guides, depth, mask and id buffers that go next
 * to an image. One nearest-hit query per sample, no shading. Outputs, per pixel or per ray; each pointer may be NULL (not
 * written), but not all three:
 *   albedo4           float4 (albedo.rgb, coverage): the stored albedo of the hit sphere's material, whatever its type,
 *                     and 1 for a hit; a miss adds zeros.
 *   normal4           float4 (normal.xyz, depth): (hit - centre) * invRadius as the renderer shades with it (not flipped
 *                     toward the ray, not renormalised), and the distance t along the unit direction; a miss adds zeros.
 *   ids               int32: the id of the hit sphere, -1 for a miss.
 * A hit on a padding sphere (id >= count, possible with the reference-form sweep only) reports the all-zero material and
 * a zero normal, as the draw sees it.
 * Float4 device buffers must be 16-byte aligned and ids 4-byte aligned. Host buffers are staged through the context and
 * make the call synchronous. Ordering and accounting are those of tpt_draw: one ray per traced sample counts toward
 * outRayCount and tpt_read_ray_count, and tpt_last_kernel_ms / tpt_last_launch_count describe the call. Bad arguments are
 * refused (tpt_last_error gives the reason).
 *
 * tpt_draw_aovs: the AOVs of the pixels a fast-mode tpt_draw with the same frameCount, numFrames, width, height, row
 * region, testFlags, spp and scene traces. Sample s of frame f of pixel (x, y) uses exactly that draw's camera ray
 * (stream pixel_seed((y * width + x) * spp + s, f), pixel jitter, lens sample) and its slab-queue sweep form, so the AOVs
 * describe the primary hits of fast variants 3 and 8. The float4 outputs are blended like the image:
 * out = prev * wPrev + sum_f w_f * mean_f (all four components; `prev` is not read when its weight is 0), so buffers kept
 * next to the backbuffer and drawn with the same arguments accumulate over the same samples, progressive rendering
 * included. ids is not blended: each call writes the id of sample 0 of frame frameCount. The row region (row0, numRows,
 * rowStep, packed), the buffer sizes (width*height pixels, or numRows with `packed`) and numRows == 0 are as in tpt_draw;
 * other rows are not touched. numFrames <= 256. Host float4 buffers are uploaded only when `prev` has weight.
 *
 * tpt_trace_aovs: the AOVs of n caller rays {o.xyz, d.xyz}, loaded, validated and normalised as tpt_trace_rays does (same
 * alignment of rays6). Deterministic: coverage is 0 or 1 and depth is in world units whatever the length of the given
 * direction. An untraceable ray (non-finite component, or a direction that does not normalise) gives zeros and id -1 and
 * adds no rays. n <= 2^32 - 1; n == 0 launches nothing. */
int tpt_draw_aovs(tpt_context* ctx, int frameCount, int numFrames, int width, int height,
                  int row0, int numRows, int rowStep, int packed,
                  float* albedo4, float* normal4, int* ids, int buffersOnDevice, unsigned testFlags,
                  long long* outRayCount, void* cudaStream);
int tpt_trace_aovs(tpt_context* ctx, const float* rays6, int raysOnDevice, long long n,
                   float* albedo4, float* normal4, int* ids, int outOnDevice,
                   long long* outRayCount, void* cudaStream);

/* Per-pixel sample sums and second moments of the fast draw's own samples, for all pixels or a caller-listed subset: what
 * adaptive sampling needs (learn how noisy each pixel is, then trace more samples for the noisy ones only).
 *   pixels            n linear pixel indices y * width + x (row 0 = bottom) of a width x height image; duplicates and any
 *                     order are allowed. NULL = every pixel 0 .. width * height - 1, and then n must be width * height.
 *   spp               samples per listed entry. Sample s of pixel p is exactly the fast draw's: stream
 *                     pixel_seed(p * spp + s, frame), pixel jitter and lens sample (fast_camera_ray), then the estimator of
 *                     TPT_MODE_FAST with the scene options of a fast draw ("light_sampling", "mitsuba_compare",
 *                     "fast_kform", scenes past 64 KB of blob). So one call with pixels = NULL and the context's spp traces
 *                     the samples of tpt_draw(frame, 1, ..., TPT_MODE_FAST) at zero `prev` weight, and calls with frame + 1,
 *                     frame + 2, ... give independent further samples. width * height * spp must not exceed 2^32.
 *   sum4              n float4, ACCUMULATED: entry i receives += (sum r, sum g, sum b, spp) over its samples. Zero it once,
 *                     then add calls; mean = sum.rgb / sum.w.
 *   sq4               NULL, or n float4 accumulated as += (sum r^2, sum g^2, sum b^2, 0): with sum4 it gives the unbiased
 *                     per-pixel variance (sq - sum^2 / w) / (w - 1) over any number of calls.
 *   buffersOnDevice   0: host pointers, staged through the context (sum4 and sq4 are uploaded, since the call adds to
 *                     them) and the call is synchronous; 1: device pointers of the context's device (or mapped host
 *                     memory), pixels 4-byte and sum4 / sq4 16-byte aligned.
 *   outRayCount       NULL or receives the number of rays traced (path and shadow rays).
 * An index outside [0, width * height) is found on the device before anything is traced: the call then traces nothing,
 * adds nothing and fails, tpt_last_error naming the first such entry. A call with a pixel list is therefore synchronous;
 * one with pixels = NULL and device buffers synchronises only when a ray count is requested. n == 0 (an empty list, so
 * pixels and sum4 must still be non-NULL) launches nothing and reads no buffer.
 * Ordering and accounting are those of tpt_draw. NULL sum4, n < 0, spp < 1, width * height * spp > 2^32, a misaligned
 * device buffer or one on another device are refused (tpt_last_error gives the reason). */
int tpt_draw_samples(tpt_context* ctx, int frame, int width, int height,
                     const int* pixels, long long n, int spp,
                     float* sum4, float* sq4, int buffersOnDevice,
                     long long* outRayCount, void* cudaStream);

/* Per-entry sample sums and second moments of tpt_trace_rays (points = 0) or tpt_trace_irradiance (points = 1), for all
 * inputs or a caller-listed subset: what adaptive sampling of caller rays and surface points needs (panoramas, lightmaps,
 * irradiance probes), as tpt_draw_samples gives it for image pixels.
 *   in6, numIn        numIn rays {o, d} (points = 0) or surface points {p, n} (points = 1), 6 floats each, loaded, validated
 *                     and normalised exactly as tpt_trace_rays / tpt_trace_irradiance load them (same alignment).
 *   ids               NULL, or numIn int32 sphere ids with tpt_trace_irradiance's meaning (id i belongs to input i). Only
 *                     taken with points = 1.
 *   entries           n int32 indices into in6, any order, duplicates allowed. NULL = every input, and then n must be numIn.
 *   spp, frame        samples per listed entry. Sample s of input i at `frame` is exactly the sample tpt_trace_rays /
 *                     tpt_trace_irradiance traces for input i: stream pixel_seed(i * spp + s, frame), keyed by the INPUT,
 *                     not by the list position. So an all-input call traces the samples of the mean call with the same spp
 *                     and frame, a list call traces for each listed input the samples the all-input call traces for it,
 *                     and frame + 1, frame + 2, ... give independent further samples. numIn * spp must not exceed 2^32.
 *   sum4              n float4, ACCUMULATED: entry k (list position) receives += (sum v.r, sum v.g, sum v.b, count), v being
 *                     the path radiance for rays and pi x the white-Lambert radiance for points; sum.rgb / sum.w estimates
 *                     what tpt_trace_rays / tpt_trace_irradiance return.
 *   sq4               NULL, or n float4 accumulated as += (sum v.r^2, sum v.g^2, sum v.b^2, 0).
 *   buffersOnDevice   0: host pointers, staged through the context (sum4 and sq4 are uploaded, since the call adds to them)
 *                     and the call is synchronous; 1: device pointers of the context's device (or mapped host memory),
 *                     in6, ids and entries 4-byte, sum4 / sq4 16-byte aligned.
 *   outRayCount       NULL or receives the number of rays traced (as tpt_trace_rays / tpt_trace_irradiance count them).
 * An input that tpt_trace_rays would not trace (a non-finite component, or a direction or normal that does not normalise)
 * adds NOTHING: its entries' counts stay as they were and it adds no rays. (tpt_draw_samples always adds spp.)
 * An index outside [0, numIn) is found on the device before anything is traced: the call then traces nothing, adds nothing
 * and fails, tpt_last_error naming the first such entry and its value. A call with a list is therefore synchronous; one
 * without it and with device buffers synchronises only when a ray count is requested. n == 0 launches nothing and reads
 * no buffer. n must not exceed 2^32 - 1, nor the slabs (64 entries x one sample) 2^31 - 1.
 * Ordering and accounting (tpt_read_ray_count, tpt_last_kernel_ms, tpt_last_launch_count, tpt_debug_last_kernels) are
 * those of tpt_trace_rays. NULL in6 or sum4, ids with points = 0, n != numIn without a list, n or numIn < 0, spp < 1, a
 * misaligned device buffer or one on another device are refused (tpt_last_error gives the reason). */
int tpt_trace_samples(tpt_context* ctx, const float* in6, const int* ids, int points, long long numIn,
                      const int* entries, long long n, int spp, int frame,
                      float* sum4, float* sq4, int buffersOnDevice,
                      long long* outRayCount, void* cudaStream);

/* Rays traced by all draws since the last call of this function (synchronises the stream). */
int tpt_read_ray_count(tpt_context* ctx, void* cudaStream, long long* outRays);
/* Device time (CUDA events on the launching stream) of the kernels of the most recent tpt_draw, in ms. */
int tpt_last_kernel_ms(tpt_context* ctx, float* outMs);
/* Number of kernel launches issued by the most recent tpt_draw. */
int tpt_last_launch_count(tpt_context* ctx);
/* Bytes the most recent tpt_set_scene copied host -> device: the packed scene blob, or 0 when its bytes were already
 * resident (a shell calls UpdateTest every frame; option "scene_upload_always" = 1 copies regardless). */
long long tpt_last_scene_upload_bytes(tpt_context* ctx);

/* Optional epilogue ("next" row of SURVEY §8f): linear float RGBA -> 8-bit sRGB RGBA with Y flip, the
 * presentation step of the reference shells (Cpp/Windows/PixelShader.hlsl:1-15). dst = width*height*4 bytes. */
int tpt_tonemap_srgb8(tpt_context* ctx, const float* image, int imageOnDevice, int width, int height,
                      unsigned char* dst, int dstOnDevice, void* cudaStream);
/* The reference's other two 8-bit conversions in the same pass: transfer 0 = the above, 1 = min(sqrtf(x)*255, 255), the
 * WebAssembly shell's cheap gamma (Cpp/Emscripten/main.cpp:67-79, which also flips Y), 2 = the C# TGA writer's
 * LinearToSRGB with its 255.9 truncation (Cs/Program.cs:34-68: bgr = 1, flipY = 0 — TGA rows are bottom-up like the
 * backbuffer's). */
int tpt_tonemap_rgba8(tpt_context* ctx, const float* image, int imageOnDevice, int width, int height,
                      unsigned char* dst, int dstOnDevice, int transfer, int bgr, int flipY, void* cudaStream);

/* Multi-GPU, one process per GPU: device memory that another process's kernels can write into directly over
 * NVLink/NVSwitch (CUDA IPC). The root rank allocates the image and exports a 64-byte handle; every other rank
 * opens it and passes the returned pointer as a device `backbuffer` to tpt_draw with its own row shard
 * (row0 = rank, rowStep = world, packed = 0): the trace kernel's 128-bit stores / vector reductions then land in
 * the root's HBM as the pixels finish — no separate gather. The reference has no counterpart (single device). */
int tpt_mem_alloc(tpt_context* ctx, unsigned long long bytes, void** outDevPtr);      /* zero-filled */
int tpt_mem_free(tpt_context* ctx, void* devPtr);
int tpt_mem_copy(tpt_context* ctx, void* dst, const void* src, unsigned long long bytes, int kind /*1 H2D, 2 D2H, 3 D2D*/);
int tpt_ipc_export(tpt_context* ctx, void* devPtr, void* outHandle64);
int tpt_ipc_open(tpt_context* ctx, const void* handle64, void** outDevPtr);
int tpt_ipc_close(tpt_context* ctx, void* devPtr);

/* Diagnostic used by the parity tests: evaluates the device-side libm restatement the exact mode uses
 * (toypathtracer_b200/csrc/tpt_libm.cuh) on n host floats. fn: 0 = sinf, 1 = cosf, 2 = powf(x, 5), 3 = powf(x, 1.0f/3.0f)
 * (the REFGPU mode's pow(x, 1.0/3.0), ComputeShader.hlsl:33). */
int tpt_debug_libm(tpt_context* ctx, int fn, const float* in, float* out, long long n);
/* Diagnostic used by the parity tests: nearest hit (HitWorld, Test.cpp:85-106) of n host rays {o.xyz, d.xyz} in the
 * current scene with one sweep form of the fast kernels (kform 0 reference form, 1 expanded, 2 expanded on packed pairs,
 * 3 conservative packed pass + reference-form decisions, 4 expanded on packed pairs read from the kernel parameters: scenes
 * of at most 64 padded spheres only, 5 as 4 with the half-precision first pass: scenes that pass its gate only), tMin/tMax as Trace uses them. outId -1 = miss. */
int tpt_debug_hit(tpt_context* ctx, int kform, const float* rays6, int* outId, float* outT, long long n);
/* Diagnostic: the mangled names of the trace kernels (path tracing and first-hit AOV kernels, not the helpers that clear,
 * blend or count) that the CALLING THREAD's most recent tpt_draw, tpt_trace_rays, tpt_trace_irradiance, tpt_trace_samples,
 * tpt_draw_samples, tpt_draw_aovs or tpt_trace_aovs launched, in launch order, separated by '\n' and NUL-terminated in buf[cap].
 *   - The record is per host thread, not per context: a call on another thread, or on another context from this
 *     thread, replaces it.
 *   - A call resets it when it starts launching (an empty call too). A call refused before that leaves the previous
 *     record; a call that fails after it holds the launches made before the failure.
 *   - Only the first 16 launches are named. The return value counts all of them, so a result above 16 means the list
 *     was cut off (long multi-launch draws, e.g. exact mode split over many frame batches).
 * Returns that count, or minus an error code (buffer too small, CUDA error). */
int tpt_debug_last_kernels(tpt_context* ctx, char* buf, int cap);
/* Diagnostic: device timestamps (ms since the start of the last progress-mode host draw) of the trace kernel's end,
 * each band copy's end and the draw's end. Returns minus the number of entries written. */
int tpt_debug_timeline(tpt_context* ctx, float* outMs, int capacity);

#ifdef __cplusplus
}
#endif
#endif
