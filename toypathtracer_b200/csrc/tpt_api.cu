// C-ABI of include/tpt_b200.h: context, scene upload, draw dispatch, host<->device plumbing.
// No torch types, no CPU rendering path: every draw ends in a kernel launch or an error.
#include "../../include/tpt_b200.h"
#include "tpt_launch.h"
#include "tpt_scene_pack.h"
#include "tpt_device_utils.cuh"
#include "tpt_integrator.cuh"
#include "tpt_env_tables.h"
#include <cuda.h>      // types only: cuStreamWaitValue32 is resolved at run time (cudaGetDriverEntryPoint), libcuda is not linked
#include <cmath>
#include <string>
#include <vector>
#include <string.h>
#include <stdarg.h>
#include <stdio.h>

using namespace tpt;

thread_local KernelRecord tpt::t_lastKernels = {};

// Device staging allocations of host buffers (tpt_context::staging). kStageImage holds tpt_draw's image, the input of
// tpt_tonemap_rgba8, tpt_trace_rays' out4 and tpt_draw_samples' sum4; the others hold the buffers they are named after.
enum Staging { kStageImage, kStageRays, kStageAlbedo, kStageNormal, kStageIds, kStagePixels, kStageSq4, kNumStaging };

// Set-up data that the calls read on the device (tpt_set_environment's map, tpt_set_textures' and
// tpt_set_emission_textures' layers), in two device slots
// with the scene blob's discipline: a new upload goes into the slot that is not current, on the upload stream after that
// slot's last use (slot_begin_upload, slot_finish_upload); calls wait on the current slot's upload and mark its last use
// (begin_call and finish_call through slot_use and slot_used). So a call keeps the data it was issued with, even while
// it is in flight, and the caller never synchronises.
struct DeviceSlots
{
    void* ptr[2] = {nullptr, nullptr};
    size_t cap[2] = {0, 0};
    int cur = 1;                                  // the first upload goes into slot 0
    bool have = false;                            // the calls issued from now on read slot `cur`
    cudaEvent_t uploadDone[2] = {nullptr, nullptr};
    cudaEvent_t lastUse[2] = {nullptr, nullptr};
};

// One set of sphere textures (tpt_set_textures' albedo, tpt_set_emission_textures' emission): its slots, each
// [layers x h x w float4 texels][spheres int32 layers], with the emission set's sampling tables behind them
// (tpt_env_tables.h), and the sizes of the current one.
struct TextureSlots
{
    DeviceSlots slots;
    int w = 0, h = 0, layers = 0, spheres = 0;
    bool tables = false;       // the current slot has sampling tables (the emission set)
    bool sampleable = false;   // ... and some layer with a non-zero weight
};

struct tpt_context
{
    int device = 0;
    int numSMs = 132;
    cudaStream_t stream = nullptr;
    cudaEvent_t evStart = nullptr, evStop = nullptr;
    bool haveTiming = false;
    std::string lastError;

    // scene: two device blobs + two pinned staging buffers. tpt_set_scene never blocks the host: the new blob goes
    // into the slot the draws in flight are NOT reading, on its own stream (the per-frame scene update of the
    // reference's GPU shells, Cpp/Windows/TestWin.cpp:261-283, as an async double-buffered upload); draws wait on the
    // slot's upload event, uploads wait on the slot's last-use event.
    unsigned char* dBlobs[2] = {nullptr, nullptr};
    size_t blobCap[2] = {0, 0};
    unsigned char* hBlob[2] = {nullptr, nullptr};
    size_t hBlobCap[2] = {0, 0};
    int curBlob = 0;
    cudaStream_t uploadStream = nullptr;
    cudaEvent_t uploadDone[2] = {nullptr, nullptr};
    cudaEvent_t blobLastUse[2] = {nullptr, nullptr};
    std::vector<unsigned char> lastBlob;          // bytes of the blob currently on the device (skip identical uploads)
    cudaEvent_t lastDraw = nullptr;               // end of the most recent draw: draws of one context are serialised in
    cudaStream_t lastDrawStream = nullptr;        // issue order even when they are enqueued on different streams
    bool haveLastDraw = false;
    SceneDev scene{};
    Camera88 cam{};
    bool haveScene = false;
    int spp = 4;

    // environment (tpt_set_environment), albedo textures (tpt_set_textures) and emission textures
    // (tpt_set_emission_textures): each in its own DeviceSlots. They belong to the context, not to the scene:
    // tpt_set_scene leaves them alone.
    DeviceSlots env;
    int envW = 0, envH = 0;                       // of the current slot
    bool envSampleable = false;                   // the current slot's map has sampling tables (some weight is not zero)
    int envSampling = 0;                          // "environment_sampling"
    TextureSlots tex, emit;
    int emitSampling = 0;                         // "emission_texture_sampling"
    int maxDepth = kRefMaxDepth;                  // "max_depth"
    // tpt_set_media's records (5 floats per sphere id), which also belong to the context: every pack of a scene puts them
    // in its blob, so tpt_set_media re-packs the current scene from its inputs, kept here with the flags it was packed with.
    std::vector<float> media;
    // tpt_set_fog's record (9 floats; empty: none), which the packs put in the blob the same way.
    std::vector<float> fog;
    std::vector<Sphere20> sceneSpheres;
    std::vector<Material36> sceneMats;
    std::vector<int> sceneEmissives;
    bool sceneEmissivesGiven = false;
    uint32_t scenePackFlags = 0;

    // options
    int fastVariant = -1;     // -1 = auto (fast_auto_variant)
    int fastKForm = 2;        // 0: reference-form sweep, 1: expanded form, 2: expanded form on the pair array (slab queue: in the
                              // kernel parameter for scenes of <= 64 padded spheres), 3: as 2 with the pair array always in
                              // shared memory (A/B), 4: as 2 without the half-precision pass 1 of form 5 (A/B); gated
                              // per scene by kformOk
    int fastAlphaZero = 0;
    int sceneUploadAlways = 0;   // 1: tpt_set_scene copies the blob even when its bytes are the resident scene's (benchmarks: a real H2D per step)
    long long lastSceneUploadBytes = 0;
    uint32_t sceneFlags = 0;  // kScene* bits for the next tpt_set_scene    // 1: fast-mode draws whose `prev` has zero weight write alpha = 0 instead of preserving it
    int exactLanes = 0;
    // Exact mode, one frame per call (the drop-in's DrawTest): a frame is only `height` serial RNG chains, far too few to
    // fill the GPU, while 16 frames at once do. With "exact_lookahead" = L > 1 a
    // cache miss traces frames [f, f+L) in ONE launch into a per-frame colour cache and the calls for f+1 .. f+L-1 only
    // blend their cached frame into the caller's buffer (per-frame colours do not depend on the buffer, Test.cpp:283-291):
    // same bits, same per-frame ray counts, L frames of latency on a miss. Not used under kFlagAnimate (the scene of a
    // future frame is not known yet); any scene, camera, size, row-range or spp change invalidates the cache.
    // "exact_lookahead" = -1 is the adaptive form for callers that render frame after frame (the drop-in's DrawTest): the
    // first call traces one frame; each time the caller walks to the end of the cached window and asks for the frame right
    // after it, with nothing else changed, the next window doubles (1, 2, 4, 8, 16 frames). No first-call latency, at most
    // half of the traced frames are speculative when the caller stops or changes anything.
    int exactLookahead = 0;
    int lookLastServed = -1;        // last frame handed out from the current window
    bool lookKeyValid = false;      // `look` describes the last one-frame exact draw (even a window of 1)
    struct LookKey { int frame0, n, width, height, row0, numRows, rowStep, spp; unsigned long long sceneGen; Camera88 cam; } look{};
    bool lookValid = false;
    float* dLook = nullptr; size_t lookCap = 0;
    unsigned long long* dLookRays = nullptr; size_t lookRaysCap = 0;
    unsigned long long sceneGen = 0;
    int registerHost = 0;
    size_t maxScratchBytes = (size_t)8 << 30;

    // buffers
    struct { void* ptr = nullptr; size_t cap = 0; } staging[kNumStaging];   // grown by ensure, see Staging
    unsigned long long* dBadPixel = nullptr;           // tpt_draw_samples' index check, and its page-locked copy
    unsigned long long* hBadPixel = nullptr;
    float* dScratch = nullptr; size_t scratchCap = 0;  // exact mode per-frame colours
    unsigned long long* dRayCounters = nullptr; int rayCounterCap = 0;   // [numFrames]
    unsigned long long* dAccum = nullptr;              // [0] total since last read, [1] last draw total
    unsigned int* dWork = nullptr;                     // ring of work-counter slots, one per draw (kWorkSlots x 32 uints)
    unsigned workSlot = 0;
    unsigned long long* hPinned = nullptr; int hPinnedCap = 0;
    void* registeredPtr = nullptr; size_t registeredBytes = 0;
    int lastLaunches = 0;

    // host-buffer draws: row bands pipelined over several streams (kernel of band b+1 overlaps D2H of band b)
    static const int kMaxBands = 8;
    static const int kWorkSlots = 32;
    int hostBands = 3;
    cudaStream_t bandStream[kMaxBands] = {};
    cudaEvent_t bandEvent[kMaxBands] = {};
    cudaEvent_t forkEvent = nullptr;

    // progress-triggered D2H (fast variants 3/4/9): the trace kernel publishes per-band completion counters, the copy
    // stream waits on them with stream memory operations and copies a band while later bands are still being traced
    typedef CUresult (*WaitValue32Fn)(CUstream, CUdeviceptr, cuuint32_t, unsigned int);
    WaitValue32Fn waitValue32 = nullptr;
    int hostProgress = 1;
    int hostZeroCopy = 1;     // fast variant 8 stores finished pixels straight into page-locked host buffers
    int progressBands = 4;
    unsigned int* dBandDone = nullptr;
    cudaStream_t copyStream = nullptr;
    // diagnostics: timestamps of the last progress-mode draw (kernel end, each band copy end), see tpt_debug_timeline
    cudaEvent_t tlKernelEnd = nullptr, tlBand[16] = {};
    int tlBands = 0;
};

static int fail(tpt_context* ctx, cudaError_t e, const char* what)
{
    if (ctx)
    {
        char buf[512];
        snprintf(buf, sizeof(buf), "%s: %s (%s)", what, cudaGetErrorString(e), cudaGetErrorName(e));
        ctx->lastError = buf;
    }
    return (int)e ? (int)e : -1;
}
static int fail_msg(tpt_context* ctx, const char* msg)
{
    if (ctx) ctx->lastError = msg;
    return (int)cudaErrorInvalidValue;
}
__attribute__((format(printf, 2, 3))) static int fail_msgf(tpt_context* ctx, const char* fmt, ...)
{
    char msg[256];
    va_list args;
    va_start(args, fmt);
    vsnprintf(msg, sizeof(msg), fmt, args);
    va_end(args);
    return fail_msg(ctx, msg);
}
#define CK(call, what) do { cudaError_t _e = (call); if (_e != cudaSuccess) return fail(ctx, _e, what); } while (0)

namespace tpt {
// sums the per-frame counters of one draw into the running totals
// hostMirror (optional): page-locked host memory the caller of tpt_draw reads after the stream sync — the per-frame counts
// arrive there by this kernel's own stores, which saves the separate 8-byte D2H copy (one DMA round trip per draw).
__global__ void k_accumulate_rays(const unsigned long long* perFrame, int n, unsigned long long* accum, unsigned long long* hostMirror)
{
    unsigned long long s = 0;
    for (int i = 0; i < n; ++i) { const unsigned long long v = perFrame[i]; s += v; if (hostMirror) hostMirror[i] = v; }
    accum[0] += s;
    accum[1] = s;
}

// The reference's three presentation conversions of the linear float image to 8 bits per channel (row f.1):
//   transfer 0  LinearToSRGB of the D3D11/Metal presentation pass (Cpp/Windows/PixelShader.hlsl:1-15), rounded
//   transfer 1  min(sqrtf(x) * 255, 255) truncated — the WebAssembly shell's cheap gamma (Cpp/Emscripten/main.cpp:67-79)
//   transfer 2  the C# TGA writer's LinearToSRGB: min((uint)(x * 255.9f), 255) (Cs/Program.cs:61-67)
// flipY: row 0 of the float image is the bottom (the Emscripten shell flips, the TGA writer does not: TGA is bottom-up);
// bgr: TGA channel order (Cs/Program.cs:36-41).
__global__ void k_tonemap_rgba8(const float4* __restrict__ img, int width, int height, uchar4* __restrict__ dst, int transfer, int bgr, int flipY)
{
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= width * height) return;
    const int x = idx % width, y = idx / width;
    float4 c = ld_stream_f4(reinterpret_cast<const float*>(img + (size_t)(flipY ? height - 1 - y : y) * width + x));
    auto enc = [transfer](float v) -> unsigned char {
        if (transfer == 1) return (unsigned char)fminf(__fsqrt_rn(v) * 255.0f, 255.0f);
        v = fmaxf(v, 0.0f);
        v = fmaxf(1.055f * __powf(v, 0.416666667f) - 0.055f, 0.0f);
        if (transfer == 2) { unsigned u = (unsigned)(v * 255.9f); return (unsigned char)(u < 255u ? u : 255u); }
        return (unsigned char)(fminf(v, 1.0f) * 255.0f + 0.5f);
    };
    const unsigned char r = enc(c.x), g = enc(c.y), b = enc(c.z);
    dst[idx] = bgr ? make_uchar4(b, g, r, 255) : make_uchar4(r, g, b, 255);
}
} // namespace tpt

// tpt_set_environment's channel rule: finite with the sign bit clear. As an int32, such a float lies in [0, +Inf's bits):
// negative values (-0 included) are below, +Inf and NaN at or above. The device check runs the list check on these ints.
static const long long kEnvBitsLimit = 0x7f800000LL;
static bool env_channel_ok(float v)
{
    int32_t b;
    memcpy(&b, &v, 4);
    return b >= 0 && b < kEnvBitsLimit;
}

extern "C" {

int tpt_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}

int tpt_create(int device, tpt_context** out)
{
    if (!out) return (int)cudaErrorInvalidValue;
    *out = nullptr;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess) return (int)e;
    if (n <= 0) return (int)cudaErrorNoDevice;   // no CPU fallback, by design
    if (device < 0 || device >= n) return (int)cudaErrorInvalidDevice;
    tpt_context* ctx = new tpt_context();
    ctx->device = device;
    e = cudaSetDevice(device);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&ctx->numSMs, cudaDevAttrMultiProcessorCount, device);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaEventCreate(&ctx->evStart);
    if (e == cudaSuccess) e = cudaEventCreate(&ctx->evStop);
    if (e == cudaSuccess) e = cudaMalloc(&ctx->dAccum, 2 * sizeof(unsigned long long));
    if (e == cudaSuccess) e = cudaMemset(ctx->dAccum, 0, 2 * sizeof(unsigned long long));
    if (e == cudaSuccess) e = cudaMalloc(&ctx->dWork, tpt_context::kWorkSlots * 32 * sizeof(unsigned int));   // per draw: 8 bands x 4 uints
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&ctx->uploadStream, cudaStreamNonBlocking);
    for (int i = 0; i < 2 && e == cudaSuccess; ++i)
    {
        e = cudaEventCreateWithFlags(&ctx->uploadDone[i], cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ctx->blobLastUse[i], cudaEventDisableTiming);
        for (DeviceSlots* s : {&ctx->env, &ctx->tex.slots, &ctx->emit.slots})
        {
            if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s->uploadDone[i], cudaEventDisableTiming);
            if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s->lastUse[i], cudaEventDisableTiming);
        }
    }
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ctx->lastDraw, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ctx->forkEvent, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaMalloc(&ctx->dBandDone, 64);
    if (e == cudaSuccess) e = cudaEventCreate(&ctx->tlKernelEnd);
    for (int b = 0; b < 16 && e == cudaSuccess; ++b) e = cudaEventCreate(&ctx->tlBand[b]);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&ctx->copyStream, cudaStreamNonBlocking);
    if (e == cudaSuccess)
    {
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuStreamWaitValue32", &fn, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            ctx->waitValue32 = (tpt_context::WaitValue32Fn)fn;
        else (void)cudaGetLastError();
    }
    int prLo = 0, prHi = 0;
    if (e == cudaSuccess) e = cudaDeviceGetStreamPriorityRange(&prLo, &prHi);   // prHi is the numerically smallest
    for (int b = 0; b < tpt_context::kMaxBands && e == cudaSuccess; ++b)
    {
        int pr = prHi + b; if (pr > prLo) pr = prLo;                              // earlier bands first
        e = cudaStreamCreateWithPriority(&ctx->bandStream[b], cudaStreamNonBlocking, pr);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ctx->bandEvent[b], cudaEventDisableTiming);
    }
    if (e != cudaSuccess) { tpt_destroy(ctx); return (int)e; }
    *out = ctx;
    return 0;
}

void tpt_destroy(tpt_context* ctx)
{
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaDeviceSynchronize();
    if (ctx->registeredPtr) cudaHostUnregister(ctx->registeredPtr);
    for (auto& s : ctx->staging) cudaFree(s.ptr);
    cudaFree(ctx->dBadPixel); cudaFree(ctx->dScratch); cudaFree(ctx->dRayCounters); cudaFree(ctx->dLook); cudaFree(ctx->dLookRays);
    cudaFree(ctx->dAccum); cudaFree(ctx->dWork);
    for (int i = 0; i < 2; ++i)
    {
        cudaFree(ctx->dBlobs[i]);
        if (ctx->hBlob[i]) cudaFreeHost(ctx->hBlob[i]);
        if (ctx->uploadDone[i]) cudaEventDestroy(ctx->uploadDone[i]);
        if (ctx->blobLastUse[i]) cudaEventDestroy(ctx->blobLastUse[i]);
        for (DeviceSlots* s : {&ctx->env, &ctx->tex.slots, &ctx->emit.slots})
        {
            cudaFree(s->ptr[i]);
            if (s->uploadDone[i]) cudaEventDestroy(s->uploadDone[i]);
            if (s->lastUse[i]) cudaEventDestroy(s->lastUse[i]);
        }
    }
    if (ctx->uploadStream) cudaStreamDestroy(ctx->uploadStream);
    if (ctx->lastDraw) cudaEventDestroy(ctx->lastDraw);
    if (ctx->tlKernelEnd) cudaEventDestroy(ctx->tlKernelEnd);
    for (int b = 0; b < 16; ++b) if (ctx->tlBand[b]) cudaEventDestroy(ctx->tlBand[b]);
    if (ctx->hPinned) cudaFreeHost(ctx->hPinned);
    if (ctx->hBadPixel) cudaFreeHost(ctx->hBadPixel);
    for (int b = 0; b < tpt_context::kMaxBands; ++b)
    {
        if (ctx->bandStream[b]) cudaStreamDestroy(ctx->bandStream[b]);
        if (ctx->bandEvent[b]) cudaEventDestroy(ctx->bandEvent[b]);
    }
    if (ctx->forkEvent) cudaEventDestroy(ctx->forkEvent);
    if (ctx->copyStream) cudaStreamDestroy(ctx->copyStream);
    cudaFree(ctx->dBandDone);
    if (ctx->evStart) cudaEventDestroy(ctx->evStart);
    if (ctx->evStop) cudaEventDestroy(ctx->evStop);
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
}

const char* tpt_last_error(tpt_context* ctx) { return ctx ? ctx->lastError.c_str() : "null context"; }

} // extern "C"

// The scene upload of tpt_set_scene, tpt_set_media and tpt_set_fog: packs a scene (its inputs as tpt_set_scene takes them,
// the flags it is packed with, mediaSpheres media records and the fog record fog9, null for none) and makes the blob the
// scene the calls issued from now on read.
// Identical bytes are not uploaded again; otherwise the blob goes into the slot the calls in flight are not reading, on
// the upload stream, and the host never blocks on the GPU. On failure the context's scene is the one it was.
static int upload_scene(tpt_context* ctx, const char* fn, const Sphere20* spheres, const Material36* mats, int count,
                        const int* emissives, int emissiveCount, uint32_t packFlags, const float* media5, int mediaSpheres,
                        const float* fog9)
{
    std::vector<unsigned char> blob;
    SceneBlobLayout L;
    int nLights = 0;
    pack_scene_blob(spheres, mats, count, emissives, emissiveCount, blob, L, nLights, packFlags, media5, mediaSpheres, fog9);
    ParamPairs pairs;
    build_param_pairs(blob, L, count, pairs);
    const bool halfOk = build_half_pairs(blob, L, count, pairs);
    // geometry + light table must fit in shared memory next to the kernels' static shared arrays
    const uint32_t kMaxStage = 200 * 1024;
    if (L.geomBytes > kMaxStage) return fail_msgf(ctx, "%s: too many spheres for shared-memory staging", fn);
    // A reference shell calls UpdateTest + upload every frame although the scene only changes under kFlagAnimate
    // (Test.cpp:304-308): identical bytes are not uploaded again.
    const bool same = ctx->haveScene && ctx->scene.count == count && ctx->scene.layout.flags == L.flags && blob == ctx->lastBlob;
    ctx->lastSceneUploadBytes = 0;
    if (!same || ctx->sceneUploadAlways)
    {
        const int slot = ctx->haveScene ? (ctx->curBlob ^ 1) : 0;
        // the slot's previous contents may still be read by draws issued before the last upload (device side: the
        // upload stream waits on the slot's last-use event) and its staging buffer by that upload's DMA (host side)
        CK(cudaEventSynchronize(ctx->uploadDone[slot]), "sync staging slot");
        if (blob.size() > ctx->blobCap[slot])
        {
            CK(cudaEventSynchronize(ctx->blobLastUse[slot]), "sync before scene realloc");
            cudaFree(ctx->dBlobs[slot]); ctx->dBlobs[slot] = nullptr; ctx->blobCap[slot] = 0;
            CK(cudaMalloc(&ctx->dBlobs[slot], blob.size()), "cudaMalloc scene");
            ctx->blobCap[slot] = blob.size();
        }
        if (blob.size() > ctx->hBlobCap[slot])
        {
            if (ctx->hBlob[slot]) cudaFreeHost(ctx->hBlob[slot]);
            ctx->hBlob[slot] = nullptr; ctx->hBlobCap[slot] = 0;
            CK(cudaMallocHost(&ctx->hBlob[slot], blob.size()), "cudaMallocHost scene staging");
            ctx->hBlobCap[slot] = blob.size();
        }
        memcpy(ctx->hBlob[slot], blob.data(), blob.size());
        CK(cudaStreamWaitEvent(ctx->uploadStream, ctx->blobLastUse[slot], 0), "upload waits for the slot's readers");
        CK(cudaMemcpyAsync(ctx->dBlobs[slot], ctx->hBlob[slot], blob.size(), cudaMemcpyHostToDevice, ctx->uploadStream), "scene upload");
        CK(cudaEventRecord(ctx->uploadDone[slot], ctx->uploadStream), "upload event");
        ctx->curBlob = slot;
        ctx->lastSceneUploadBytes = (long long)blob.size();
        ctx->lastBlob.swap(blob);
        if (!same) ++ctx->sceneGen;              // a forced re-upload of identical bytes is not a new scene (frame-lookahead key)
    }
    ctx->scene.blob = ctx->dBlobs[ctx->curBlob];
    ctx->scene.layout = L;
    ctx->scene.count = count;
    ctx->scene.pairs = pairs;
    ctx->scene.halfOk = halfOk;
    ctx->scene.nLights = sampled_lights(L.flags, nLights);   // 0 with light sampling off: every light loop is empty
    // small scenes: stage everything (spheres + materials); large ones: geometry only, materials from L2
    ctx->scene.stagedBytes = L.totalBytes <= 64 * 1024 ? L.totalBytes : L.geomBytes;
    // Expanded-form sweep gate (FastHitterK, tpt_fast.cu). With u = 2^-24 the expanded form evaluates
    // c = |s-o|^2 - r^2 with |dc| <= ~4u (|s| + |o|)^2, the reference form (Maths.cpp:97-102) with |dc| <= ~4u |s-o|^2 + u r^2.
    // The gate |s|^2 <= 128 + 2 r^2 keeps (|s| + |o|)^2 within a small multiple of max(r^2, 128) for origins inside the
    // scene's extent (|o|^2 <= 128), i.e. the expanded form is no worse than ~8x the reference form's own bound for small
    // spheres and BETTER than it for huge ones (ground sphere r = 100: 2 s.o ~ 400 vs |co|^2 ~ 10^4). The bound is not
    // what the parity claim rests on: tests/test_gpu_configs.py and tests/test_gpu_light_sampling.py compare kform 0
    // and 1 against the bit-exact mode at >= 16k spp, overall and per first-hit material.
    ctx->scene.kformOk = true;
    for (int i = 0; i < count; ++i)
    {
        const Sphere20& s = spheres[i];
        const double c2 = (double)s.center[0] * s.center[0] + (double)s.center[1] * s.center[1] + (double)s.center[2] * s.center[2];
        if (c2 > 128.0 + 2.0 * (double)s.radius * s.radius) ctx->scene.kformOk = false;
    }
    ctx->haveScene = true;
    return 0;
}

extern "C" {

int tpt_set_scene(tpt_context* ctx, const void* spheres20, const void* materials36, int count,
                  const void* camera88, const int* emissives, int emissiveCount)
{
    if (!ctx) return (int)cudaErrorInvalidValue;
    if (!spheres20 || !materials36 || !camera88 || count <= 0) return fail_msg(ctx, "tpt_set_scene: bad arguments");
    CK(cudaSetDevice(ctx->device), "cudaSetDevice");
    // the caller's emissive list indexes spheres/materials (Test.cpp:96-100): refuse what would read out of bounds
    if (emissives)
    {
        if (emissiveCount < 0 || emissiveCount > count) return fail_msg(ctx, "tpt_set_scene: emissiveCount out of range");
        for (int i = 0; i < emissiveCount; ++i)
            if (emissives[i] < 0 || emissives[i] >= count) return fail_msg(ctx, "tpt_set_scene: emissive id out of range");
    }
    if (int r = upload_scene(ctx, "tpt_set_scene", (const Sphere20*)spheres20, (const Material36*)materials36, count, emissives,
                             emissiveCount, ctx->sceneFlags, ctx->media.empty() ? nullptr : ctx->media.data(),
                             (int)(ctx->media.size() / 5), ctx->fog.empty() ? nullptr : ctx->fog.data()))
        return r;
    // the inputs tpt_set_media re-packs
    ctx->sceneSpheres.assign((const Sphere20*)spheres20, (const Sphere20*)spheres20 + count);
    ctx->sceneMats.assign((const Material36*)materials36, (const Material36*)materials36 + count);
    ctx->sceneEmissivesGiven = emissives != nullptr;
    if (emissives) ctx->sceneEmissives.assign(emissives, emissives + emissiveCount);
    else ctx->sceneEmissives.clear();
    ctx->scenePackFlags = ctx->sceneFlags;
    memcpy(&ctx->cam, camera88, sizeof(Camera88));
    return 0;
}

int tpt_set_media(tpt_context* ctx, const float* media5, int numSpheres)
{
    if (!ctx) return (int)cudaErrorInvalidValue;
    if (numSpheres < 0) return fail_msgf(ctx, "tpt_set_media: numSpheres = %d is negative", numSpheres);
    if (!media5) numSpheres = 0;
    static const char* const kField[5] = {"sigma_a.r", "sigma_a.g", "sigma_a.b", "sigma_s", "g"};
    for (int i = 0; i < numSpheres; ++i)
    {
        const float* m = media5 + 5 * (size_t)i;
        for (int f = 0; f < 4; ++f)
            if (!env_channel_ok(m[f])) return fail_msgf(ctx, "tpt_set_media: sphere %d has %s = %g", i, kField[f], (double)m[f]);
        if (!(fabsf(m[4]) < 1.0f)) return fail_msgf(ctx, "tpt_set_media: sphere %d has g = %g", i, (double)m[4]);
    }
    std::vector<float> media(media5, media5 + 5 * (size_t)numSpheres);
    if (ctx->haveScene)
    {
        CK(cudaSetDevice(ctx->device), "cudaSetDevice");
        if (int r = upload_scene(ctx, "tpt_set_media", ctx->sceneSpheres.data(), ctx->sceneMats.data(),
                                 (int)ctx->sceneSpheres.size(), ctx->sceneEmissivesGiven ? ctx->sceneEmissives.data() : nullptr,
                                 (int)ctx->sceneEmissives.size(), ctx->scenePackFlags, media.empty() ? nullptr : media.data(),
                                 numSpheres, ctx->fog.empty() ? nullptr : ctx->fog.data()))
            return r;
    }
    ctx->media.swap(media);
    return 0;
}

int tpt_set_fog(tpt_context* ctx, const float* fog9)
{
    if (!ctx) return (int)cudaErrorInvalidValue;
    static const char* const kField[9] = {"centre.x", "centre.y", "centre.z", "radius", "sigma_a.r", "sigma_a.g", "sigma_a.b",
                                          "sigma_s", "g"};
    if (fog9)
    {
        for (int f = 0; f < 3; ++f)
            if (!std::isfinite(fog9[f])) return fail_msgf(ctx, "tpt_set_fog: %s = %g", kField[f], (double)fog9[f]);
        if (!(std::isfinite(fog9[3]) && fog9[3] > 0.0f)) return fail_msgf(ctx, "tpt_set_fog: radius = %g", (double)fog9[3]);
        for (int f = 4; f < 8; ++f)
            if (!env_channel_ok(fog9[f])) return fail_msgf(ctx, "tpt_set_fog: %s = %g", kField[f], (double)fog9[f]);
        if (!(fabsf(fog9[8]) < 1.0f)) return fail_msgf(ctx, "tpt_set_fog: g = %g", (double)fog9[8]);
    }
    // a record whose sigmas are all zero is no fog: stored as none, so the blob keeps the plain scene's bytes
    std::vector<float> fog;
    if (has_fog(fog9)) fog.assign(fog9, fog9 + 9);
    if (ctx->haveScene)
    {
        CK(cudaSetDevice(ctx->device), "cudaSetDevice");
        if (int r = upload_scene(ctx, "tpt_set_fog", ctx->sceneSpheres.data(), ctx->sceneMats.data(),
                                 (int)ctx->sceneSpheres.size(), ctx->sceneEmissivesGiven ? ctx->sceneEmissives.data() : nullptr,
                                 (int)ctx->sceneEmissives.size(), ctx->scenePackFlags,
                                 ctx->media.empty() ? nullptr : ctx->media.data(), (int)(ctx->media.size() / 5),
                                 fog.empty() ? nullptr : fog.data()))
            return r;
    }
    ctx->fog.swap(fog);
    return 0;
}

int tpt_set_camera(tpt_context* ctx, const void* camera88)
{
    if (!ctx || !camera88) return (int)cudaErrorInvalidValue;
    memcpy(&ctx->cam, camera88, sizeof(Camera88));
    return 0;
}

int tpt_set_spp(tpt_context* ctx, int spp)
{
    if (!ctx) return (int)cudaErrorInvalidValue;
    if (spp < 1 || spp > 4096) return fail_msg(ctx, "tpt_set_spp: spp out of range");
    ctx->spp = spp;
    return 0;
}

int tpt_set_option(tpt_context* ctx, const char* key, int value)
{
    if (!ctx || !key) return (int)cudaErrorInvalidValue;
    if (!strcmp(key, "fast_variant")) { if (value < -1 || value > 9) return fail_msg(ctx, "fast_variant: -1 (auto), 0..9"); ctx->fastVariant = value; return 0; }
    if (!strcmp(key, "exact_lanes")) { if (value != 0 && value != 1 && value != 2 && value != 8 && value != 9 && value != 32 && (value < 64 || value > 71)) return fail_msg(ctx, "exact_lanes: 0,1,2,8,9,32,64..71"); ctx->exactLanes = value; return 0; }
    if (!strcmp(key, "exact_lookahead")) { if (value < -1 || value > 256) return fail_msg(ctx, "exact_lookahead: -1 (adaptive), 0..256"); ctx->exactLookahead = value; ctx->lookValid = false; ctx->lookKeyValid = false; return 0; }
    if (!strcmp(key, "register_host")) { ctx->registerHost = value ? 1 : 0; return 0; }
    if (!strcmp(key, "fast_kform")) { if (value < 0 || value > 4) return fail_msg(ctx, "fast_kform: 0..4"); ctx->fastKForm = value; return 0; }
    if (!strcmp(key, "fast_alpha_zero")) { ctx->fastAlphaZero = value ? 1 : 0; return 0; }
    if (!strcmp(key, "scene_upload_always")) { ctx->sceneUploadAlways = value ? 1 : 0; return 0; }
    if (!strcmp(key, "mitsuba_compare")) { ctx->sceneFlags = value ? (ctx->sceneFlags | kSceneMitsuba) : (ctx->sceneFlags & ~(uint32_t)kSceneMitsuba); return 0; }
    if (!strcmp(key, "environment_sampling")) { ctx->envSampling = value ? 1 : 0; return 0; }
    if (!strcmp(key, "emission_texture_sampling")) { ctx->emitSampling = value ? 1 : 0; return 0; }
    if (!strcmp(key, "max_depth")) { if (value < 1 || value > kMaxPathDepth) return fail_msg(ctx, "max_depth: 1..256"); ctx->maxDepth = value; return 0; }
    if (!strcmp(key, "light_sampling")) { ctx->sceneFlags = value ? (ctx->sceneFlags & ~(uint32_t)kSceneNoLightSampling) : (ctx->sceneFlags | kSceneNoLightSampling); return 0; }
    if (!strcmp(key, "host_progress")) { ctx->hostProgress = value ? 1 : 0; return 0; }
    if (!strcmp(key, "host_zero_copy")) { ctx->hostZeroCopy = value ? 1 : 0; return 0; }
    if (!strcmp(key, "progress_bands")) { if (value < 1 || value > 16) return fail_msg(ctx, "progress_bands: 1..16"); ctx->progressBands = value; return 0; }
    if (!strcmp(key, "host_bands")) { if (value < 1 || value > tpt_context::kMaxBands) return fail_msg(ctx, "host_bands: 1..8"); ctx->hostBands = value; return 0; }
    if (!strcmp(key, "max_scratch_mb")) { if (value < 16) return fail_msg(ctx, "max_scratch_mb: >= 16"); ctx->maxScratchBytes = (size_t)value << 20; return 0; }
    return fail_msg(ctx, "tpt_set_option: unknown key");
}

static int ensure(tpt_context* ctx, void** p, size_t* cap, size_t bytes, const char* what)
{
    if (bytes <= *cap) return 0;
    CK(cudaStreamSynchronize(ctx->stream), "sync before realloc");
    cudaFree(*p); *p = nullptr; *cap = 0;
    CK(cudaMalloc(p, bytes), what);
    *cap = bytes;
    return 0;
}

// The slot a new upload of `bytes` goes into (*slot): the one that is not current, grown when it is too small (after its
// last reader, issued before the previous upload, has finished), with the upload stream ordered after that reader.
// `what` names the data in error texts.
static int slot_begin_upload(tpt_context* ctx, DeviceSlots& s, size_t bytes, const char* what, int* slot)
{
    const std::string w = what;
    *slot = s.cur ^ 1;
    if (bytes > s.cap[*slot])
    {
        CK(cudaEventSynchronize(s.lastUse[*slot]), ("sync before " + w + " realloc").c_str());
        cudaFree(s.ptr[*slot]); s.ptr[*slot] = nullptr; s.cap[*slot] = 0;
        CK(cudaMalloc(&s.ptr[*slot], bytes), ("cudaMalloc " + w).c_str());
        s.cap[*slot] = bytes;
    }
    CK(cudaStreamWaitEvent(ctx->uploadStream, s.lastUse[*slot], 0), (w + " upload waits for the slot's readers").c_str());
    return 0;
}

// After the upload's copies into `slot` were enqueued on the upload stream: the slot becomes current once they have been
// read (a set-up call: it returns once the caller's data has been read, so the caller may then free or reuse it).
static int slot_finish_upload(tpt_context* ctx, DeviceSlots& s, int slot, const char* what)
{
    const std::string w = what;
    CK(cudaEventRecord(s.uploadDone[slot], ctx->uploadStream), (w + " upload event").c_str());
    CK(cudaStreamSynchronize(ctx->uploadStream), (w + " upload sync").c_str());
    s.cur = slot;
    s.have = true;
    return 0;
}

// begin_call: the call reads the current slot, once its upload has landed; its address into *addr.
static int slot_use(tpt_context* ctx, const DeviceSlots& s, cudaStream_t stream, const char* what, uint64_t* addr)
{
    CK(cudaStreamWaitEvent(stream, s.uploadDone[s.cur], 0), (std::string("wait for ") + what + " upload").c_str());
    *addr = (uint64_t)(uintptr_t)s.ptr[s.cur];
    return 0;
}

// finish_call: the next upload into the call's slot waits for this call.
static int slot_used(tpt_context* ctx, const DeviceSlots& s, cudaStream_t stream, const char* what)
{
    if (s.have) CK(cudaEventRecord(s.lastUse[s.cur], stream), (std::string(what) + " last-use event").c_str());
    return 0;
}

// begin_call's part for one texture set, while it is set: the call reads its current slot (slot_use), sees `flag` and
// gets the slot's addresses and sizes in *out.
static int use_textures(tpt_context* ctx, const TextureSlots& ts, cudaStream_t stream, const char* what, uint32_t flag,
                        SceneDev* scene, TexSet* out)
{
    if (!ts.slots.have) return 0;
    uint64_t tex = 0;
    if (int r = slot_use(ctx, ts.slots, stream, what, &tex)) return r;
    const uint64_t tab = tex + (uint64_t)16 * ts.w * ts.h * ts.layers;
    scene->layout.flags |= flag;
    out->texLo = (uint32_t)tex;
    out->texHi = (uint32_t)(tex >> 32);
    out->tabLo = (uint32_t)tab;
    out->tabHi = (uint32_t)(tab >> 32);
    out->W = ts.w;
    out->H = ts.h;
    // sphere ids past the scene's count are padding spheres, which are never textured
    out->spheres = ts.spheres < scene->count ? ts.spheres : scene->count;
    out->tabWords = ts.tables ? (uint32_t)emit_table_words(ts.spheres) : 0u;
    return 0;
}

// Prologue of a call that traces (tpt_draw, tpt_trace_rays). One context = one scene blob, one set of counters: calls are
// ordered in issue order even across streams, and the scene they read must have landed (tpt_set_scene uploads
// asynchronously on its own stream). Returns the call's stream and the scene with the context's sweep-form option applied.
static int begin_call(tpt_context* ctx, void* cudaStreamArg, cudaStream_t* stream, SceneDev* scene)
{
    CK(cudaSetDevice(ctx->device), "cudaSetDevice");
    *stream = cudaStreamArg ? (cudaStream_t)cudaStreamArg : ctx->stream;
    if (ctx->haveLastDraw && ctx->lastDrawStream != *stream) CK(cudaStreamWaitEvent(*stream, ctx->lastDraw, 0), "order after previous draw");
    CK(cudaStreamWaitEvent(*stream, ctx->uploadDone[ctx->curBlob], 0), "wait for scene upload");
    *scene = ctx->scene;
    if (ctx->env.have)
    {
        // the call reads the environment that is current now, in its slot, once that slot's upload has landed
        uint64_t env = 0;
        if (int r = slot_use(ctx, ctx->env, *stream, "environment", &env)) return r;
        scene->layout.flags |= kSceneEnvironment;
        scene->layout.envLo = (uint32_t)env;
        scene->layout.envHi = (uint32_t)(env >> 32);
        scene->layout.envW = ctx->envW;
        scene->layout.envH = ctx->envH;
        // "environment_sampling" is read here, per call, like the map: not a scene flag, so toggling it uploads nothing
        if (ctx->envSampling && ctx->envSampleable && !(scene->layout.flags & kSceneNoLightSampling))
            scene->layout.flags |= kSceneEnvSampling;
    }
    if (int r = use_textures(ctx, ctx->tex, *stream, "textures", kSceneTextures, scene, &scene->layout.tex)) return r;
    if (int r = use_textures(ctx, ctx->emit, *stream, "emission textures", kSceneEmissionTextures, scene, &scene->layout.emit))
        return r;
    // "emission_texture_sampling", like "environment_sampling": read per call, not a scene flag
    if (ctx->emitSampling && ctx->emit.slots.have && ctx->emit.sampleable && !(scene->layout.flags & kSceneNoLightSampling))
        scene->layout.flags |= kSceneEmitSampling;
    // "max_depth", read per call as well: only this call's copy of the layout carries it, never the blob or ctx->scene
    scene->layout.flags |= depth_flags(ctx->maxDepth);
    scene->kformOk = scene->kformOk && ctx->fastKForm != 0;
    scene->kformMode = ctx->fastKForm;
    scene->pairs.half = scene->halfOk && scene->kformOk && ctx->fastKForm == 2;
    return 0;
}

// Zeroes the call's `n` ray counters (one per frame) and starts its kernel timing.
static int start_kernels(tpt_context* ctx, cudaStream_t stream, int n)
{
    if (n > ctx->rayCounterCap)
    {
        CK(cudaStreamSynchronize(stream), "sync before counter realloc");
        cudaFree(ctx->dRayCounters); ctx->dRayCounters = nullptr; ctx->rayCounterCap = 0;
        CK(cudaMalloc(&ctx->dRayCounters, (size_t)n * sizeof(unsigned long long)), "cudaMalloc counters");
        ctx->rayCounterCap = n;
    }
    CK(cudaMemsetAsync(ctx->dRayCounters, 0, (size_t)n * sizeof(unsigned long long), stream), "zero counters");
    ctx->lastLaunches = 0;
    clear_kernels();
    CK(cudaEventRecord(ctx->evStart, stream), "event record");
    return 0;
}

// Ends the kernel timing and folds the call's `n` ray counters into the running totals (tpt_read_ray_count) and, when
// the caller wants the counts, into page-locked memory that finish_call reads.
static int finish_kernels(tpt_context* ctx, cudaStream_t stream, int n, bool wantCounts)
{
    CK(cudaEventRecord(ctx->evStop, stream), "event record");
    ctx->haveTiming = true;
    if (wantCounts && n > ctx->hPinnedCap)
    {
        if (ctx->hPinned) cudaFreeHost(ctx->hPinned);
        ctx->hPinned = nullptr; ctx->hPinnedCap = 0;
        CK(cudaMallocHost(&ctx->hPinned, (size_t)n * sizeof(unsigned long long)), "cudaMallocHost");
        ctx->hPinnedCap = n;
    }
    note_launch();
    k_accumulate_rays<<<1, 1, 0, stream>>>(ctx->dRayCounters, n, ctx->dAccum, wantCounts ? ctx->hPinned : nullptr);
    CK(cudaGetLastError(), "accumulate launch");
    ctx->lastLaunches = t_lastKernels.launches;
    return 0;
}

// Epilogue after the call's last copy: the next call orders after this one and the next scene upload into this blob slot
// after it. The host synchronises only to read the counts back, or because the call had host buffers (synchronous then).
static int finish_call(tpt_context* ctx, cudaStream_t stream, int n, bool hostBuffers, long long* outRayCount, long long* outPerFrame)
{
    CK(cudaEventRecord(ctx->lastDraw, stream), "draw end event");
    CK(cudaEventRecord(ctx->blobLastUse[ctx->curBlob], stream), "scene last-use event");
    if (int r = slot_used(ctx, ctx->env, stream, "environment")) return r;
    if (int r = slot_used(ctx, ctx->tex.slots, stream, "textures")) return r;
    if (int r = slot_used(ctx, ctx->emit.slots, stream, "emission textures")) return r;
    ctx->lastDrawStream = stream; ctx->haveLastDraw = true;
    if (outRayCount || outPerFrame)
    {
        CK(cudaStreamSynchronize(stream), "stream sync");     // the counts were stored into hPinned by k_accumulate_rays
        long long total = 0;
        for (int i = 0; i < n; ++i)
        {
            total += (long long)ctx->hPinned[i];
            if (outPerFrame) outPerFrame[i] = (long long)ctx->hPinned[i];
        }
        if (outRayCount) *outRayCount = total;
    }
    else if (hostBuffers)
        CK(cudaStreamSynchronize(stream), "stream sync");
    return 0;
}

// A call with nothing to trace: no launch, no rays (none in each of its `numFrames` frames either).
static int empty_call(tpt_context* ctx, long long* outRayCount, long long* outPerFrame = nullptr, int numFrames = 0)
{
    if (outRayCount) *outRayCount = 0;
    if (outPerFrame) for (int i = 0; i < numFrames; ++i) outPerFrame[i] = 0;
    ctx->lastLaunches = 0;
    clear_kernels();
    return 0;
}

// The work-counter slot of the next launch sequence: the ring leaves the slots of the calls still in flight alone.
static unsigned int* next_work_counter(tpt_context* ctx)
{
    return ctx->dWork + (size_t)(ctx->workSlot++ % tpt_context::kWorkSlots) * 32;
}

// Parameters of a draw of the rows y_i = row0 + i*rowStep (or the packed band) of a width x height image through the
// context's camera; the rest is zero.
static DrawParams image_params(const tpt_context* ctx, int width, int height, int row0, int numRows, int rowStep, int packed,
                               int spp, unsigned flags)
{
    DrawParams p;
    memset(&p, 0, sizeof(p));
    p.cam = ctx->cam;
    p.width = width; p.height = height;
    p.row0 = row0; p.numRows = numRows; p.rowStep = rowStep; p.packed = packed ? 1 : 0;
    p.spp = spp;
    p.flags = flags;
    p.invWidth = 1.0f / (float)width;     // Test.cpp:270-271
    p.invHeight = 1.0f / (float)height;
    return p;
}

} // extern "C" (the caller-buffer helpers below are templates, which cannot have C linkage)

// A row region of a draw's image: rows y_i = row0 + i*rowStep (or the packed band) of `width` pixels.
struct RowRegion { int width, row0, numRows, rowStep, packed; };

enum { kCopyUp = 1, kCopyDown = 2 };

// One caller buffer of tpt_draw, tpt_trace_rays, tpt_trace_irradiance, tpt_trace_aovs, tpt_draw_aovs, tpt_draw_samples or
// tpt_tonemap_rgba8. A null `ptr` is a buffer the caller left out: it is neither checked nor staged.
struct CallerBuffer
{
    const char* name;                   // as the error texts name it
    void* ptr;                          // the caller's
    bool onDevice;                      // device memory (or mapped host memory); otherwise staged
    int align;                          // bytes a device pointer must be aligned to
    size_t bytes;                       // the whole buffer: the size of its staging allocation
    Staging staging;                    // the allocation a host buffer is staged through
    int copy;                           // kCopyUp: a host buffer is uploaded before the kernels, kCopyDown: downloaded after
    const RowRegion* rows = nullptr;    // a draw buffer: only the region's rows of pixBytes-byte pixels are copied
    size_t pixBytes = 16;
    void* dev = nullptr;                // what the kernels use, set by stage_in
};

// A device buffer must be addressable by the context's device: its own memory, or mapped host memory.
static int check_device_buffer(tpt_context* ctx, const char* fn, const void* ptr, const char* name)
{
    cudaPointerAttributes attr;
    if (cudaPointerGetAttributes(&attr, ptr) != cudaSuccess || attr.type == cudaMemoryTypeUnregistered)
    {
        (void)cudaGetLastError();
        return fail_msgf(ctx, "%s: device %s is not CUDA memory", fn, name);
    }
    if ((attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged) && attr.device != ctx->device)
        return fail_msgf(ctx, "%s: device %s lives on device %d, the context on device %d", fn, name, attr.device, ctx->device);
    return 0;
}

// The device buffers of call `fn`: all aligned, then each addressable by the context's device.
template <int N>
static int check_buffers(tpt_context* ctx, const char* fn, const CallerBuffer (&bufs)[N])
{
    for (const CallerBuffer& b : bufs)
        if (b.ptr && b.onDevice && ((uintptr_t)b.ptr & (uintptr_t)(b.align - 1)))
            return fail_msgf(ctx, "%s: device %s is not %d-byte aligned", fn, b.name, b.align);
    for (const CallerBuffer& b : bufs)
        if (b.ptr && b.onDevice)
            if (int r = check_device_buffer(ctx, fn, b.ptr, b.name)) return r;
    return 0;
}

// Copies a buffer between host and device: all of it, or only its region's rows.
static cudaError_t copy_buffer(const CallerBuffer& b, void* dstBase, const void* srcBase, cudaMemcpyKind kind, cudaStream_t stream)
{
    char* dst = (char*)dstBase;
    const char* src = (const char*)srcBase;
    if (!b.rows) return cudaMemcpyAsync(dst, src, b.bytes, kind, stream);
    const RowRegion& r = *b.rows;
    const size_t rowBytes = (size_t)r.width * b.pixBytes;
    if (r.packed) return cudaMemcpyAsync(dst, src, rowBytes * r.numRows, kind, stream);
    const size_t off = (size_t)r.row0 * rowBytes;
    if (r.rowStep == 1) return cudaMemcpyAsync(dst + off, src + off, rowBytes * r.numRows, kind, stream);
    return cudaMemcpy2DAsync(dst + off, rowBytes * r.rowStep, src + off, rowBytes * r.rowStep, rowBytes, r.numRows, kind, stream);
}

// Gives every buffer the pointer its kernels use: a host buffer's staging allocation, grown to the buffer's size and
// uploaded when the record says so.
template <int N>
static int stage_in(tpt_context* ctx, cudaStream_t stream, CallerBuffer (&bufs)[N])
{
    for (CallerBuffer& b : bufs)
    {
        b.dev = b.ptr;
        if (!b.ptr || b.onDevice) continue;
        auto& st = ctx->staging[b.staging];
        if (int r = ensure(ctx, &st.ptr, &st.cap, b.bytes, b.name)) return r;
        b.dev = st.ptr;
        if (b.copy & kCopyUp) CK(copy_buffer(b, b.dev, b.ptr, cudaMemcpyHostToDevice, stream), b.name);
    }
    return 0;
}

// Copies the host buffers the record says so back from their staging allocations.
template <int N>
static int stage_out(tpt_context* ctx, cudaStream_t stream, const CallerBuffer (&bufs)[N])
{
    for (const CallerBuffer& b : bufs)
        if (b.ptr && !b.onDevice && (b.copy & kCopyDown)) CK(copy_buffer(b, b.ptr, b.dev, cudaMemcpyDeviceToHost, stream), b.name);
    return 0;
}

// The device index check of a caller list (tpt_draw_samples, tpt_trace_samples): its word and the pinned host word
// its result comes back in, allocated on first use.
static int ensure_index_check(tpt_context* ctx)
{
    if (ctx->dBadPixel) return 0;
    CK(cudaMalloc(&ctx->dBadPixel, sizeof(unsigned long long)), "cudaMalloc index check");
    CK(cudaMallocHost(&ctx->hBadPixel, sizeof(unsigned long long)), "cudaMallocHost index check");
    return 0;
}

// The end of a caller-buffer call of one frame: the ray count, the index check's result (list = the call had a list),
// the host outputs, and the synchronisation (sync: a host buffer; a list makes the call synchronous too, its index check
// being the call's result, which the caller then reads from *ctx->hBadPixel).
template <int N>
static int end_caller_call(tpt_context* ctx, cudaStream_t stream, const CallerBuffer (&bufs)[N], bool list, bool sync,
                           long long* outRayCount)
{
    if (int r = finish_kernels(ctx, stream, 1, outRayCount != nullptr)) return r;
    if (list) CK(cudaMemcpyAsync(ctx->hBadPixel, ctx->dBadPixel, sizeof(unsigned long long), cudaMemcpyDeviceToHost, stream), "D2H index check");
    if (int r = stage_out(ctx, stream, bufs)) return r;
    return finish_call(ctx, stream, 1, sync || list, outRayCount, nullptr);
}

// Page-locks (and maps) the caller's host buffer once ("register_host"): copies run at full PCIe rate and the kernels can
// store into it directly. Failure is not fatal.
static void register_host(tpt_context* ctx, void* host, size_t bytes)
{
    if (ctx->registeredPtr == host && ctx->registeredBytes == bytes) return;
    if (ctx->registeredPtr) { cudaHostUnregister(ctx->registeredPtr); ctx->registeredPtr = nullptr; }
    if (cudaHostRegister(host, bytes, cudaHostRegisterMapped) == cudaSuccess)
    {
        ctx->registeredPtr = host; ctx->registeredBytes = bytes;
    }
    else (void)cudaGetLastError();
}

// Exact mode, one frame per call, with frame lookahead (see tpt_context::exactLookahead): a miss traces the window
// [p.frame0, p.frame0 + L) into the lookahead cache; the frame is then blended from the cache into the image and its ray
// count copied to the call's counter (a window of one frame is traced straight into the image).
static int draw_exact_lookahead(tpt_context* ctx, const DrawParams& p, const SceneDev& sc, cudaStream_t stream)
{
    const int frame = p.frame0;
    tpt_context::LookKey k{};
    k.width = p.width; k.height = p.height; k.row0 = p.row0; k.numRows = p.numRows; k.rowStep = p.rowStep; k.spp = p.spp;
    k.sceneGen = ctx->sceneGen; k.cam = p.cam;
    const tpt_context::LookKey& c = ctx->look;
    const size_t perFrame = (size_t)p.numRows * p.width * 4;           // floats
    const bool sameSetup = c.width == k.width && c.height == k.height && c.row0 == k.row0 && c.numRows == k.numRows &&
                           c.rowStep == k.rowStep && c.spp == k.spp && c.sceneGen == k.sceneGen && !memcmp(&c.cam, &k.cam, sizeof(Camera88));
    const bool hit = ctx->lookValid && frame >= c.frame0 && frame < c.frame0 + c.n && sameSetup;
    if (!hit)
    {
        size_t L = ctx->exactLookahead > 1 ? (size_t)ctx->exactLookahead : 1;
        if (ctx->exactLookahead == -1 && ctx->lookKeyValid && sameSetup && frame == c.frame0 + c.n &&
            ctx->lookLastServed == c.frame0 + c.n - 1)
            L = c.n >= 8 ? 16 : (size_t)c.n * 2;           // the caller consumed the whole window and continues: double it
        const size_t fit = ctx->maxScratchBytes / (perFrame * 4);
        if (L > fit) L = fit < 1 ? 1 : fit;
        int r = ensure(ctx, (void**)&ctx->dLook, &ctx->lookCap, L * perFrame * 4, "cudaMalloc lookahead cache");
        if (r) return r;
        r = ensure(ctx, (void**)&ctx->dLookRays, &ctx->lookRaysCap, L * sizeof(unsigned long long), "cudaMalloc lookahead counters");
        if (r) return r;
        CK(cudaMemsetAsync(ctx->dLookRays, 0, L * sizeof(unsigned long long), stream), "zero lookahead counters");
        DrawParams pl = p;
        pl.numFrames = (int)L; pl.scratch = ctx->dLook; pl.rayCounter = ctx->dLookRays;
        cudaError_t e = launch_exact(pl, sc, ctx->exactLanes, ctx->numSMs, stream, /*resolve*/ L == 1);
        if (e != cudaSuccess) return fail(ctx, e, "kernel launch");
        k.frame0 = frame; k.n = (int)L;
        ctx->look = k; ctx->lookValid = L > 1; ctx->lookKeyValid = true; ctx->lookLastServed = frame;
        if (L == 1) { CK(cudaMemcpyAsync(ctx->dRayCounters, ctx->dLookRays, 8, cudaMemcpyDeviceToDevice, stream), "counter copy"); return 0; }
    }
    const int i = frame - ctx->look.frame0;
    ctx->lookLastServed = frame;
    DrawParams pr = p;
    pr.scratch = ctx->dLook + (size_t)i * perFrame;
    const cudaError_t e = launch_resolve_exact(pr, stream);
    CK(cudaMemcpyAsync(ctx->dRayCounters, ctx->dLookRays + i, 8, cudaMemcpyDeviceToDevice, stream), "counter copy");
    return e == cudaSuccess ? 0 : fail(ctx, e, "kernel launch");
}

// Host-buffer fast draws can hand the image to the caller's buffer `host` in bands, so that the D2H copies overlap the
// tracing. Here ONE kernel for the whole image publishes per-band completion counters; the copy stream waits on them
// (cuStreamWaitValue32) and copies a band while later bands are still being traced.
static int draw_progress_bands(tpt_context* ctx, const DrawParams& p, const SceneDev& sc, int variant, float* host,
                               cudaStream_t stream)
{
    const int NB = ctx->progressBands;
    unsigned int expected[16];
    CK(cudaMemsetAsync(ctx->dBandDone, 0, 64, stream), "zero band counters");
    CK(cudaEventRecord(ctx->forkEvent, stream), "fork event");
    CK(cudaStreamWaitEvent(ctx->copyStream, ctx->forkEvent, 0), "copy stream wait");
    cudaError_t e = launch_fast(p, sc, variant, ctx->numSMs, stream, ctx->dBandDone, NB, expected);
    if (e != cudaSuccess) return fail(ctx, e, "kernel launch");
    CK(cudaEventRecord(ctx->tlKernelEnd, stream), "timeline event");
    ctx->tlBands = 0;
    const long long regionPix = (long long)p.numRows * p.width, slab = fast_slab_pixels();
    const long long mtiles = (regionPix + slab - 1) / slab, mpb = (mtiles + NB - 1) / NB;
    const size_t firstPix = p.packed ? 0 : (size_t)p.row0 * p.width;
    for (int b = NB - 1; b >= 0; --b)     // the kernel walks the image from its last macro-tile down: last band first
    {
        const long long p0 = (long long)b * mpb * slab, p1 = (long long)(b + 1) * mpb * slab < regionPix ? (long long)(b + 1) * mpb * slab : regionPix;
        if (p1 <= p0) continue;
        if (ctx->waitValue32((CUstream)ctx->copyStream, (CUdeviceptr)(ctx->dBandDone + b), expected[b], CU_STREAM_WAIT_VALUE_GEQ) != CUDA_SUCCESS)
            return fail_msg(ctx, "cuStreamWaitValue32 failed");
        const size_t off = (firstPix + (size_t)p0) * 4;
        CK(cudaMemcpyAsync(host + off, p.image + off, (size_t)(p1 - p0) * 16, cudaMemcpyDeviceToHost, ctx->copyStream), "D2H band");
        CK(cudaEventRecord(ctx->tlBand[ctx->tlBands++], ctx->copyStream), "timeline event");
    }
    CK(cudaEventRecord(ctx->bandEvent[0], ctx->copyStream), "copy event");
    CK(cudaStreamWaitEvent(stream, ctx->bandEvent[0], 0), "join copies");
    return 0;
}

// The same with one launch sequence per band of contiguous or packed rows, each on its own stream (earlier band = higher
// priority) followed by the band's copy: the D2H of band b overlaps the tracing of band b+1, and the persistent CTAs of
// band b+1 fill the SMs as band b's tail drains.
static int draw_row_bands(tpt_context* ctx, const DrawParams& p, const SceneDev& sc, int variant, float* host, cudaStream_t stream)
{
    const int NB = ctx->hostBands;
    CK(cudaEventRecord(ctx->forkEvent, stream), "fork event");
    for (int b = 0; b < NB; ++b)
    {
        const int rb0 = (int)((long long)p.numRows * b / NB), rb1 = (int)((long long)p.numRows * (b + 1) / NB);
        cudaStream_t bs = ctx->bandStream[b];
        CK(cudaStreamWaitEvent(bs, ctx->forkEvent, 0), "band wait");
        DrawParams pb = p;
        pb.row0 = p.row0 + rb0 * p.rowStep;
        pb.numRows = rb1 - rb0;
        pb.workCounter = p.workCounter + 4 * b;
        const size_t firstRow = p.packed ? (size_t)rb0 : (size_t)(p.row0 + rb0);   // rowStep == 1 when not packed
        if (p.packed) pb.image = p.image + firstRow * p.width * 4;
        cudaError_t e = launch_fast(pb, sc, variant, ctx->numSMs, bs);
        if (e != cudaSuccess) return fail(ctx, e, "kernel launch");
        const size_t off = firstRow * p.width * 4, bytes = (size_t)(rb1 - rb0) * p.width * 16;
        CK(cudaMemcpyAsync(host + off, p.image + off, bytes, cudaMemcpyDeviceToHost, bs), "D2H band");
        CK(cudaEventRecord(ctx->bandEvent[b], bs), "band event");
        CK(cudaStreamWaitEvent(stream, ctx->bandEvent[b], 0), "join band");
    }
    return 0;
}

// One launch sequence of tpt_draw: frames [p.frame0, p.frame0 + p.numFrames) of the region in `mode`.
static int draw_frames(tpt_context* ctx, DrawParams p, const SceneDev& sc, int mode, int variant, cudaStream_t stream)
{
    cudaError_t e;
    if (mode == TPT_MODE_EXACT)
    {
        if (p.numFrames > 1)
        {
            int r = ensure(ctx, (void**)&ctx->dScratch, &ctx->scratchCap, (size_t)p.numFrames * p.numRows * p.width * 16, "cudaMalloc scratch");
            if (r) return r;
            p.scratch = ctx->dScratch;
        }
        e = launch_exact(p, sc, ctx->exactLanes, ctx->numSMs, stream);
    }
    else if (mode == TPT_MODE_REFGPU) e = launch_refgpu_exact(p, sc, ctx->numSMs, stream);
    else if (mode == TPT_MODE_REFGPU_FAST) e = launch_refgpu_fast(p, sc, ctx->numSMs, stream);
    else e = launch_fast(p, sc, variant, ctx->numSMs, stream);
    return e == cudaSuccess ? 0 : fail(ctx, e, "kernel launch");
}

extern "C" {

int tpt_draw(tpt_context* ctx, int frameCount, int numFrames, int width, int height,
             int row0, int numRows, int rowStep, int packed,
             float* backbuffer, int bufferOnDevice, unsigned testFlags, int mode,
             long long* outRayCount, long long* outRaysPerFrame, void* cudaStreamArg)
{
    if (!ctx) return (int)cudaErrorInvalidValue;
    if (!ctx->haveScene) return fail_msg(ctx, "tpt_draw: no scene (call tpt_set_scene after UpdateTest)");
    if (!backbuffer || width <= 0 || height <= 0 || numFrames <= 0 || frameCount < 0 || numRows < 0 || rowStep <= 0 || row0 < 0)
        return fail_msg(ctx, "tpt_draw: bad arguments");
    if (mode != TPT_MODE_EXACT && mode != TPT_MODE_FAST && mode != TPT_MODE_REFGPU && mode != TPT_MODE_REFGPU_FAST)
        return fail_msg(ctx, "tpt_draw: unknown mode");
    // the parity modes reproduce the reference, which has no environment to be bit-identical to
    if (mode != TPT_MODE_FAST && ctx->env.have)
        return fail_msg(ctx, "tpt_draw: an environment is set, and only TPT_MODE_FAST draws use one (clear it with "
                             "tpt_set_environment(ctx, NULL, 0, 0, 0) for exact and reference-GPU draws)");
    if (mode != TPT_MODE_FAST && (ctx->tex.slots.have || ctx->emit.slots.have))
    {
        const bool albedo = ctx->tex.slots.have;
        return fail_msgf(ctx, "tpt_draw: %s are set, and only TPT_MODE_FAST draws use them (clear them with "
                              "%s(ctx, NULL, 0, 0, 0, NULL, 0, 0) for exact and reference-GPU draws)",
                         albedo ? "textures" : "emission textures", albedo ? "tpt_set_textures" : "tpt_set_emission_textures");
    }
    if (mode != TPT_MODE_FAST && (ctx->scene.layout.flags & kSceneMedia))
        return fail_msg(ctx, "tpt_draw: the scene has media, and only TPT_MODE_FAST draws use them (clear them with "
                             "tpt_set_media(ctx, NULL, 0) for exact and reference-GPU draws)");
    if (mode != TPT_MODE_FAST && (ctx->scene.layout.flags & kSceneFog))
        return fail_msg(ctx, "tpt_draw: the scene has fog, and only TPT_MODE_FAST draws use it (clear it with "
                             "tpt_set_fog(ctx, NULL) for exact and reference-GPU draws)");
    if (mode != TPT_MODE_FAST && ctx->maxDepth != kRefMaxDepth)
        return fail_msgf(ctx, "tpt_draw: \"max_depth\" is %d, and only TPT_MODE_FAST draws use it (set it back to 10 for "
                              "exact and reference-GPU draws)", ctx->maxDepth);
    // an empty shard (more ranks than rows, TraceRowJob(start, start)): nothing to trace, nothing to copy
    if (numRows == 0) return empty_call(ctx, outRayCount, outRaysPerFrame, numFrames);
    if (row0 + (long long)(numRows - 1) * rowStep >= height) return fail_msg(ctx, "tpt_draw: rows outside the image");
    cudaStream_t stream;
    SceneDev scene;
    if (int r = begin_call(ctx, cudaStreamArg, &stream, &scene)) return r;
    // only the slab queue's reference-form 6-CTA and 768-thread instances sample the environment, look up textures,
    // trace media and fog and take the call's depth cap
    const bool envSampling = (scene.layout.flags & kSceneEnvSampling) != 0;
    const bool textured = (scene.layout.flags & kSceneAnyTextures) != 0;
    if (envSampling && ctx->fastVariant >= 0 && !fast_variant_info(ctx->fastVariant).referenceQueue)
        return fail_msgf(ctx, "tpt_draw: \"environment_sampling\" is active (option on, a map with non-zero weight, light "
                              "sampling on), and fast_variant %d does not sample the environment: use -1 (auto), 3 or 9",
                         ctx->fastVariant);
    if (textured && ctx->fastVariant >= 0 && !fast_variant_info(ctx->fastVariant).referenceQueue)
    {
        const bool albedo = (scene.layout.flags & kSceneTextures) != 0;
        return fail_msgf(ctx, "tpt_draw: %s are set (%s), and fast_variant %d does not look them up: use -1 (auto), 3 or 9",
                         albedo ? "textures" : "emission textures", albedo ? "tpt_set_textures" : "tpt_set_emission_textures",
                         ctx->fastVariant);
    }
    if ((scene.layout.flags & kSceneMedia) && ctx->fastVariant >= 0 && !fast_variant_info(ctx->fastVariant).referenceQueue)
        return fail_msgf(ctx, "tpt_draw: the scene has media (tpt_set_media), and fast_variant %d does not trace them: use -1 "
                              "(auto), 3 or 9", ctx->fastVariant);
    if ((scene.layout.flags & kSceneFog) && ctx->fastVariant >= 0 && !fast_variant_info(ctx->fastVariant).referenceQueue)
        return fail_msgf(ctx, "tpt_draw: the scene has fog (tpt_set_fog), and fast_variant %d does not trace it: use -1 "
                              "(auto), 3 or 9", ctx->fastVariant);
    if ((scene.layout.flags & kSceneDepth) && ctx->fastVariant >= 0 && !fast_variant_info(ctx->fastVariant).referenceQueue)
        return fail_msgf(ctx, "tpt_draw: \"max_depth\" is %d, and fast_variant %d keeps the depth cap at 10: use -1 (auto), 3 "
                              "or 9", ctx->maxDepth, ctx->fastVariant);

    const RowRegion rows = {width, row0, numRows, rowStep, packed};
    const size_t bufBytes = (packed ? (size_t)numRows : (size_t)height) * width * 4 * sizeof(float);
    if (!bufferOnDevice && ctx->registerHost) register_host(ctx, backbuffer, bufBytes);
    const float prevWeight = prev_weight(frameCount, numFrames, testFlags);
    // Host-buffer draw whose `prev` has zero weight, into page-locked memory the GPU can address: the trace kernel's
    // coalesced 128-bit pixel stores go straight into the caller's buffer over PCIe while the other pixels are still
    // being traced — no staging image, no device-to-host copy after the kernel.
    bool zeroCopy = false;
    cudaPointerAttributes attr{};
    if (!bufferOnDevice && mode == TPT_MODE_FAST && ctx->hostZeroCopy && !(scene.layout.flags & kSceneRefForm) &&
        (ctx->fastVariant < 0 || fast_variant_info(ctx->fastVariant).writesFinalPixels))
    {
        zeroCopy = prevWeight == 0.0f && numFrames <= kMaxFramesPerDraw && cudaPointerGetAttributes(&attr, backbuffer) == cudaSuccess &&
                   attr.type == cudaMemoryTypeHost && attr.devicePointer;
        if (!zeroCopy) (void)cudaGetLastError();
    }
    const int variant = ctx->fastVariant >= 0 ? ctx->fastVariant
                                              : fast_auto_variant(scene, (long long)numRows * width, ctx->spp, numFrames, zeroCopy);

    // frames per launch: exact mode needs numFrames*numRows*width float4 of scratch when numFrames > 1
    int framesPerLaunch = numFrames;
    if (mode == TPT_MODE_EXACT && numFrames > 1)
    {
        const size_t perFrame = (size_t)numRows * width * 16;
        size_t fit = ctx->maxScratchBytes / perFrame;
        if (fit < 1) fit = 1;
        if ((size_t)framesPerLaunch > fit) framesPerLaunch = (int)fit;
    }
    if (mode == TPT_MODE_FAST && framesPerLaunch > kMaxFramesPerDraw) framesPerLaunch = kMaxFramesPerDraw;
    const bool lookahead = mode == TPT_MODE_EXACT && numFrames == 1 && (ctx->exactLookahead > 1 || ctx->exactLookahead == -1) &&
                           !(testFlags & TPT_FLAG_ANIMATE);
    const FastVariantInfo info = fast_variant_info(variant);
    const bool banded = mode == TPT_MODE_FAST && !bufferOnDevice && info.rowBands && ctx->hostBands > 1 &&
                        (rowStep == 1 || packed) && framesPerLaunch == numFrames && numRows >= 16 * ctx->hostBands;
    // the per-band completion counters are 32-bit (cuStreamWaitValue32): a band never holds more paths than the image
    const bool progress = banded && ctx->waitValue32 && ctx->hostProgress && info.progressCounters &&
                          (long long)numRows * width * ctx->spp * numFrames <= 0xFFFFFFFFLL;

    // `prev` is an input of the blend (Test.cpp:293). Exact mode always uploads it (NaN/Inf * 0 and the untouched alpha
    // are part of bit parity). Fast mode uploads it only when prev has a non-zero weight; otherwise the kernel writes
    // alpha = 0, which is what every reference shell's zero-initialised buffer holds (TestWin.cpp:73-74,
    // Renderer.mm:148-149, Emscripten/main.cpp:50-51). (REFGPU writes alpha = 1 and lerp(col, prev, 0) does not read prev:
    // same rule as the fast mode.) Only the rows this draw renders go back, unless bands deliver them: the caller's other
    // rows are not ours to touch (TraceRowJob writes rows [start,end) only, Test.cpp:278-297). A zero-copy draw stores
    // through the buffer's device alias.
    const bool uploadPrev = mode == TPT_MODE_EXACT || prevWeight != 0.0f;
    CallerBuffer image[] = {{"backbuffer", zeroCopy ? attr.devicePointer : backbuffer, bufferOnDevice || zeroCopy, 16, bufBytes,
                             kStageImage, (uploadPrev ? kCopyUp : 0) | (banded ? 0 : kCopyDown), &rows}};
    if (int r = stage_in(ctx, stream, image)) return r;

    if (int r = start_kernels(ctx, stream, numFrames)) return r;
    DrawParams p = image_params(ctx, width, height, row0, numRows, rowStep, packed, ctx->spp, testFlags);
    p.image = (float*)image[0].dev;
    p.workCounter = next_work_counter(ctx);
    // alpha is never written by the reference (Maths.h:38). When `prev` has zero weight the fast kernels keep the alpha
    // that is in the buffer, unless the staging image was not uploaded (host buffer) or the caller waived it.
    p.zeroAlpha = (ctx->fastAlphaZero || (!bufferOnDevice && !uploadPrev)) ? 1 : 0;     // (zero-copy: never reads host memory)
    for (int f = 0; f < numFrames; f += framesPerLaunch)     // banded: one pass
    {
        p.frame0 = frameCount + f;
        p.numFrames = numFrames - f < framesPerLaunch ? numFrames - f : framesPerLaunch;
        p.rayCounter = ctx->dRayCounters + (mode == TPT_MODE_EXACT ? f : 0);    // per-frame counts in exact mode
        const int r = lookahead  ? draw_exact_lookahead(ctx, p, scene, stream)
                      : progress ? draw_progress_bands(ctx, p, scene, variant, backbuffer, stream)
                      : banded   ? draw_row_bands(ctx, p, scene, variant, backbuffer, stream)
                                 : draw_frames(ctx, p, scene, mode, variant, stream);
        if (r) return r;
    }
    if (int r = finish_kernels(ctx, stream, numFrames, outRayCount || outRaysPerFrame)) return r;
    if (int r = stage_out(ctx, stream, image)) return r;
    // host-buffer draws are synchronous like DrawTest
    return finish_call(ctx, stream, numFrames, !bufferOnDevice, outRayCount, outRaysPerFrame);
}

// tpt_trace_rays (points = false: in6 holds rays {o, d}), tpt_trace_irradiance (points = true: in6 holds surface points
// {p, n}, ids their sphere ids or null) and tpt_trace_samples (sums = true: entries null or a list of n indices into the
// numIn inputs, out4 = sum4 and sq4 accumulated): the same checks, staging and launch of the slab queue on caller entries.
// Without sums, n == numIn and there is no list.
static int trace_caller_entries(tpt_context* ctx, const char* fn, const char* inName, bool points, bool sums, const float* in6,
                                const int* ids, int inOnDevice, long long numIn, const int* entries, long long n, int spp,
                                int frame, float* out4, float* sq4, int outOnDevice, long long* outRayCount,
                                void* cudaStreamArg)
{
    const char* outName = sums ? "sum4" : "out4";
    if (!ctx) return (int)cudaErrorInvalidValue;
    if (!ctx->haveScene) return fail_msgf(ctx, "%s: no scene (call tpt_set_scene first)", fn);
    if (!in6 || !out4) return fail_msgf(ctx, "%s: null %s or %s", fn, inName, outName);
    if (numIn < 0 || n < 0) return fail_msgf(ctx, "%s: n < 0", fn);
    if (spp < 1) return fail_msgf(ctx, "%s: spp < 1", fn);
    // the sample stream of (input i, sample s) is i * spp + s in 32 bits, and so is the input index
    if (numIn > (1LL << 32) / spp || numIn > 0xffffffffLL)
        return fail_msgf(ctx, "%s: %s * spp > 2^32 (32-bit sample streams)", fn, sums ? "numIn" : "n");
    if (ids && !points) return fail_msgf(ctx, "%s: ids are only taken with points", fn);
    if (!entries && n != numIn) return fail_msgf(ctx, "%s: without entries n must be numIn", fn);
    if (sums && (n > 0xffffffffLL || (n + fast_slab_pixels() - 1) / fast_slab_pixels() * spp > 0x7fffffffLL))
        return fail_msgf(ctx, "%s: n * spp too large (2^31 slabs of 64 entries x one sample)", fn);
    // an empty sums call: nothing to trace, no buffer is read (as tpt_draw_samples)
    if (sums && n == 0) return empty_call(ctx, outRayCount);
    // the sums accumulate: host sums go up and come back
    const int outCopy = sums ? kCopyUp | kCopyDown : kCopyDown;
    CallerBuffer bufs[] = {{inName, (void*)in6, inOnDevice != 0, 4, (size_t)numIn * 24, kStageRays, kCopyUp},
                           {"ids", (void*)ids, inOnDevice != 0, 4, (size_t)numIn * 4, kStageIds, kCopyUp},
                           {"entries", (void*)entries, inOnDevice != 0, 4, (size_t)n * 4, kStagePixels, kCopyUp},
                           {outName, out4, outOnDevice != 0, 16, (size_t)n * 16, kStageImage, outCopy},
                           {"sq4", sq4, outOnDevice != 0, 16, (size_t)n * 16, kStageSq4, kCopyUp | kCopyDown}};
    if (int r = check_buffers(ctx, fn, bufs)) return r;
    if (n == 0) return empty_call(ctx, outRayCount);
    cudaStream_t stream;
    SceneDev scene;
    if (int r = begin_call(ctx, cudaStreamArg, &stream, &scene)) return r;
    if (entries)
        if (int r = ensure_index_check(ctx)) return r;
    if (int r = stage_in(ctx, stream, bufs)) return r;
    if (int r = start_kernels(ctx, stream, 1)) return r;
    DrawParams p;
    memset(&p, 0, sizeof(p));
    p.spp = spp;
    p.frame0 = frame; p.numFrames = 1;     // flags 0: the one frame has weight 1, `prev` none
    p.image = (float*)bufs[3].dev;
    p.sq4 = (float*)bufs[4].dev;
    p.rayCounter = ctx->dRayCounters;
    p.workCounter = next_work_counter(ctx);
    p.rays = (const float*)bufs[0].dev;
    p.numRays = (uint32_t)n;
    p.pointStart = points ? 1 : 0;
    p.pointIds = (const int*)bufs[1].dev;
    p.sums = sums ? 1 : 0;
    p.entries = (const int*)bufs[2].dev;
    cudaError_t e = launch_fast_rays(p, scene, numIn, ctx->dBadPixel, ctx->numSMs, stream);
    if (e != cudaSuccess) return fail(ctx, e, "kernel launch");
    if (int r = end_caller_call(ctx, stream, bufs, entries != nullptr, !inOnDevice || !outOnDevice, outRayCount)) return r;
    if (entries && *ctx->hBadPixel != ~0ull)
        return fail_msgf(ctx, "%s: entries[%llu] = %d is outside the %lld inputs (nothing was traced)", fn,
                         *ctx->hBadPixel >> 32, (int)(uint32_t)*ctx->hBadPixel, numIn);
    return 0;
}

int tpt_trace_rays(tpt_context* ctx, const float* rays6, int raysOnDevice, long long n, int spp, int frame,
                   float* out4, int outOnDevice, long long* outRayCount, void* cudaStreamArg)
{
    return trace_caller_entries(ctx, "tpt_trace_rays", "rays6", false, false, rays6, nullptr, raysOnDevice, n, nullptr, n, spp,
                                frame, out4, nullptr, outOnDevice, outRayCount, cudaStreamArg);
}

int tpt_trace_irradiance(tpt_context* ctx, const float* points6, const int* ids, int pointsOnDevice, long long n,
                         int spp, int frame, float* out4, int outOnDevice, long long* outRayCount, void* cudaStreamArg)
{
    return trace_caller_entries(ctx, "tpt_trace_irradiance", "points6", true, false, points6, ids, pointsOnDevice, n, nullptr, n,
                                spp, frame, out4, nullptr, outOnDevice, outRayCount, cudaStreamArg);
}

int tpt_trace_samples(tpt_context* ctx, const float* in6, const int* ids, int points, long long numIn,
                      const int* entries, long long n, int spp, int frame,
                      float* sum4, float* sq4, int buffersOnDevice,
                      long long* outRayCount, void* cudaStreamArg)
{
    if (ctx && points != 0 && points != 1) return fail_msg(ctx, "tpt_trace_samples: points must be 0 or 1");
    return trace_caller_entries(ctx, "tpt_trace_samples", "in6", points != 0, true, in6, ids, buffersOnDevice, numIn, entries, n,
                                spp, frame, sum4, sq4, buffersOnDevice, outRayCount, cudaStreamArg);
}

int tpt_draw_aovs(tpt_context* ctx, int frameCount, int numFrames, int width, int height,
                  int row0, int numRows, int rowStep, int packed,
                  float* albedo4, float* normal4, int* ids, int buffersOnDevice, unsigned testFlags,
                  long long* outRayCount, void* cudaStreamArg)
{
    if (!ctx) return (int)cudaErrorInvalidValue;
    if (!ctx->haveScene) return fail_msg(ctx, "tpt_draw_aovs: no scene (call tpt_set_scene first)");
    if (width <= 0 || height <= 0 || numFrames <= 0 || frameCount < 0 || numRows < 0 || rowStep <= 0 || row0 < 0)
        return fail_msg(ctx, "tpt_draw_aovs: bad arguments");
    if (numFrames > kMaxFramesPerDraw) return fail_msg(ctx, "tpt_draw_aovs: numFrames > 256");
    if (!albedo4 && !normal4 && !ids) return fail_msg(ctx, "tpt_draw_aovs: albedo4, normal4 and ids are all null");
    const RowRegion rows = {width, row0, numRows, rowStep, packed};
    const size_t bufPix = (packed ? (size_t)numRows : (size_t)height) * width;
    // the float4 outputs are `prev` of the blend when it has weight; ids are not blended
    const int prev = prev_weight(frameCount, numFrames, testFlags) != 0.0f ? kCopyUp : 0;
    const bool dev = buffersOnDevice != 0;
    CallerBuffer bufs[] = {{"albedo4", albedo4, dev, 16, bufPix * 16, kStageAlbedo, prev | kCopyDown, &rows},
                           {"normal4", normal4, dev, 16, bufPix * 16, kStageNormal, prev | kCopyDown, &rows},
                           {"ids", ids, dev, 4, bufPix * 4, kStageIds, kCopyDown, &rows, 4}};
    if (int r = check_buffers(ctx, "tpt_draw_aovs", bufs)) return r;
    if (numRows == 0) return empty_call(ctx, outRayCount);
    if (row0 + (long long)(numRows - 1) * rowStep >= height) return fail_msg(ctx, "tpt_draw_aovs: rows outside the image");
    if ((long long)numRows * width > 0xffffffe0LL) return fail_msg(ctx, "tpt_draw_aovs: more than 2^32 - 32 pixels");
    cudaStream_t stream;
    SceneDev scene;
    if (int r = begin_call(ctx, cudaStreamArg, &stream, &scene)) return r;
    if (int r = stage_in(ctx, stream, bufs)) return r;
    if (int r = start_kernels(ctx, stream, 1)) return r;
    DrawParams p = image_params(ctx, width, height, row0, numRows, rowStep, packed, ctx->spp, testFlags);
    p.frame0 = frameCount; p.numFrames = numFrames;
    p.rayCounter = ctx->dRayCounters;
    p.workCounter = next_work_counter(ctx);
    cudaError_t e = launch_fast_aovs(p, scene, false, (float*)bufs[0].dev, (float*)bufs[1].dev, (int*)bufs[2].dev, ctx->numSMs, stream);
    if (e != cudaSuccess) return fail(ctx, e, "kernel launch");
    if (int r = finish_kernels(ctx, stream, 1, outRayCount != nullptr)) return r;
    if (int r = stage_out(ctx, stream, bufs)) return r;
    return finish_call(ctx, stream, 1, !buffersOnDevice, outRayCount, nullptr);
}

int tpt_trace_aovs(tpt_context* ctx, const float* rays6, int raysOnDevice, long long n,
                   float* albedo4, float* normal4, int* ids, int outOnDevice,
                   long long* outRayCount, void* cudaStreamArg)
{
    if (!ctx) return (int)cudaErrorInvalidValue;
    if (!ctx->haveScene) return fail_msg(ctx, "tpt_trace_aovs: no scene (call tpt_set_scene first)");
    if (!rays6) return fail_msg(ctx, "tpt_trace_aovs: null rays6");
    if (n < 0) return fail_msg(ctx, "tpt_trace_aovs: n < 0");
    if (n > 0xffffffffLL) return fail_msg(ctx, "tpt_trace_aovs: n > 2^32 - 1 (32-bit ray indices)");
    if (!albedo4 && !normal4 && !ids) return fail_msg(ctx, "tpt_trace_aovs: albedo4, normal4 and ids are all null");
    const bool dev = outOnDevice != 0;
    CallerBuffer bufs[] = {{"rays6", (void*)rays6, raysOnDevice != 0, 4, (size_t)n * 24, kStageRays, kCopyUp},
                           {"albedo4", albedo4, dev, 16, (size_t)n * 16, kStageAlbedo, kCopyDown},
                           {"normal4", normal4, dev, 16, (size_t)n * 16, kStageNormal, kCopyDown},
                           {"ids", ids, dev, 4, (size_t)n * 4, kStageIds, kCopyDown}};
    if (int r = check_buffers(ctx, "tpt_trace_aovs", bufs)) return r;
    if (n == 0) return empty_call(ctx, outRayCount);
    cudaStream_t stream;
    SceneDev scene;
    if (int r = begin_call(ctx, cudaStreamArg, &stream, &scene)) return r;
    if (int r = stage_in(ctx, stream, bufs)) return r;
    if (int r = start_kernels(ctx, stream, 1)) return r;
    DrawParams p;
    memset(&p, 0, sizeof(p));
    p.spp = 1;
    p.numFrames = 1;
    p.rayCounter = ctx->dRayCounters;
    p.workCounter = next_work_counter(ctx);
    p.rays = (const float*)bufs[0].dev;
    p.numRays = (uint32_t)n;
    cudaError_t e = launch_fast_aovs(p, scene, true, (float*)bufs[1].dev, (float*)bufs[2].dev, (int*)bufs[3].dev, ctx->numSMs, stream);
    if (e != cudaSuccess) return fail(ctx, e, "kernel launch");
    if (int r = finish_kernels(ctx, stream, 1, outRayCount != nullptr)) return r;
    if (int r = stage_out(ctx, stream, bufs)) return r;
    return finish_call(ctx, stream, 1, !raysOnDevice || !outOnDevice, outRayCount, nullptr);
}

int tpt_draw_samples(tpt_context* ctx, int frame, int width, int height,
                     const int* pixels, long long n, int spp,
                     float* sum4, float* sq4, int buffersOnDevice,
                     long long* outRayCount, void* cudaStreamArg)
{
    if (!ctx) return (int)cudaErrorInvalidValue;
    if (!ctx->haveScene) return fail_msg(ctx, "tpt_draw_samples: no scene (call tpt_set_scene first)");
    if (width <= 0 || height <= 0 || frame < 0) return fail_msg(ctx, "tpt_draw_samples: bad arguments");
    if (n < 0) return fail_msg(ctx, "tpt_draw_samples: n < 0");
    if (spp < 1) return fail_msg(ctx, "tpt_draw_samples: spp < 1");
    // the sample stream of (pixel p, sample s) is p * spp + s in 32 bits
    const long long numPix = (long long)width * height;
    if (numPix > (1LL << 32) / spp) return fail_msg(ctx, "tpt_draw_samples: width * height * spp > 2^32 (32-bit sample streams)");
    if (!sum4) return fail_msg(ctx, "tpt_draw_samples: null sum4");
    if (!pixels && n != numPix) return fail_msg(ctx, "tpt_draw_samples: without a pixel list n must be width * height");
    // an empty list: nothing to trace, no buffer is read
    if (n == 0) return empty_call(ctx, outRayCount);
    const long long slab = fast_slab_pixels();
    if (n > 0xffffffffLL || (n + slab - 1) / slab * spp > 0x7fffffffLL)
        return fail_msg(ctx, "tpt_draw_samples: n * spp too large (2^31 slabs of 64 entries x one sample)");
    // the outputs accumulate: host sums go up and come back
    const bool dev = buffersOnDevice != 0;
    CallerBuffer bufs[] = {{"pixels", (void*)pixels, dev, 4, (size_t)n * 4, kStagePixels, kCopyUp},
                           {"sum4", sum4, dev, 16, (size_t)n * 16, kStageImage, kCopyUp | kCopyDown},
                           {"sq4", sq4, dev, 16, (size_t)n * 16, kStageSq4, kCopyUp | kCopyDown}};
    if (int r = check_buffers(ctx, "tpt_draw_samples", bufs)) return r;
    cudaStream_t stream;
    SceneDev scene;
    if (int r = begin_call(ctx, cudaStreamArg, &stream, &scene)) return r;
    if (pixels)
        if (int r = ensure_index_check(ctx)) return r;
    if (int r = stage_in(ctx, stream, bufs)) return r;
    if (int r = start_kernels(ctx, stream, 1)) return r;
    DrawParams p = image_params(ctx, width, height, 0, height, 1, 0, spp, 0);
    p.frame0 = frame; p.numFrames = 1;     // flags 0: the one frame has weight 1, `prev` none
    p.image = (float*)bufs[1].dev;
    p.sq4 = (float*)bufs[2].dev;
    p.pixels = (const int*)bufs[0].dev;
    p.numRays = (uint32_t)n;
    p.rayCounter = ctx->dRayCounters;
    p.workCounter = next_work_counter(ctx);
    cudaError_t e = launch_fast_samples(p, scene, ctx->dBadPixel, ctx->numSMs, stream);
    if (e != cudaSuccess) return fail(ctx, e, "kernel launch");
    if (int r = end_caller_call(ctx, stream, bufs, pixels != nullptr, !buffersOnDevice, outRayCount)) return r;
    if (pixels && *ctx->hBadPixel != ~0ull)
        return fail_msgf(ctx, "tpt_draw_samples: pixels[%llu] = %d is outside the %d x %d image (nothing was traced)",
                         *ctx->hBadPixel >> 32, (int)(uint32_t)*ctx->hBadPixel, width, height);
    return 0;
}

int tpt_set_environment(tpt_context* ctx, const float* rgba, int width, int height, int onDevice)
{
    static const char* fn = "tpt_set_environment";
    if (!ctx) return (int)cudaErrorInvalidValue;
    // NULL: the calls issued from now on see the reference sky; those in flight keep reading their slot
    if (!rgba) { ctx->env.have = false; return 0; }
    if (width < 1 || height < 1) return fail_msgf(ctx, "%s: width and height must be >= 1 (got %d x %d)", fn, width, height);
    const long long n = (long long)width * height;
    if (n >= (1LL << 31)) return fail_msgf(ctx, "%s: width * height must be below 2^31 (got %lld)", fn, n);
    CK(cudaSetDevice(ctx->device), "cudaSetDevice");
    if (onDevice)
    {
        if ((uintptr_t)rgba & 15) return fail_msgf(ctx, "%s: device rgba is not 16-byte aligned", fn);
        if (int r = check_device_buffer(ctx, fn, rgba, "rgba")) return r;
        if (int r = ensure_index_check(ctx)) return r;
    }
    else
        for (long long i = 0; i < n; ++i)
            for (int c = 0; c < 3; ++c)
                if (!env_channel_ok(rgba[4 * i + c]))
                    return fail_msgf(ctx, "%s: texel %lld (x %lld, y %lld) has %s = %g: RGB must be finite and not negative",
                                     fn, i, i % width, i / width, c == 0 ? "R" : c == 1 ? "G" : "B", rgba[4 * i + c]);
    // The slot that is not current: the calls issued since the last tpt_set_environment read the other one.
    // The slot holds the texels, each cell's sampling probability in their alpha, and the alias tables behind them
    // (tpt_env_tables.h): 24 W H + 8 H bytes, built here on the host.
    const size_t bytes = env_slot_bytes(width, height);
    int slot = 0;
    if (int r = slot_begin_upload(ctx, ctx->env, bytes, "environment", &slot)) return r;
    Q4* dst = (Q4*)ctx->env.ptr[slot];
    cudaStream_t s = ctx->uploadStream;
    std::vector<float> host((bytes + 3) / 4);
    float* tex = host.data();
    if (onDevice)
    {
        // R, G and B of every texel packed into the slot's first 12 n bytes, then checked as 3 n int32 in [0, +Inf's bits)
        // by the caller-list check (entry = channel index), and copied back for the table build
        CK(cudaMemcpy2DAsync(dst, 12, rgba, 16, 12, (size_t)n, cudaMemcpyDefault, s), "pack environment RGB");
        CK(launch_list_check((const int*)dst, 3 * n, kEnvBitsLimit, ctx->dBadPixel, ctx->numSMs, s),
           "environment check launch");
        CK(cudaMemcpyAsync(ctx->hBadPixel, ctx->dBadPixel, sizeof(unsigned long long), cudaMemcpyDeviceToHost, s), "D2H environment check");
        CK(cudaMemcpy2DAsync(tex, 16, dst, 12, 12, (size_t)n, cudaMemcpyDeviceToHost, s), "D2H environment RGB");
        // A refused map leaves the current environment as it was.
        CK(cudaStreamSynchronize(s), "environment check sync");
        if (*ctx->hBadPixel != ~0ull)
        {
            const long long k = (long long)(*ctx->hBadPixel >> 32), i = k / 3;
            uint32_t bits = (uint32_t)*ctx->hBadPixel;
            float v;
            memcpy(&v, &bits, 4);
            return fail_msgf(ctx, "%s: texel %lld (x %lld, y %lld) has %s = %g: RGB must be finite and not negative", fn, i,
                             i % width, i / width, k % 3 == 0 ? "R" : k % 3 == 1 ? "G" : "B", v);
        }
    }
    else
        memcpy(tex, rgba, (size_t)n * 16);
    EnvAlias* rows = reinterpret_cast<EnvAlias*>(tex + 4 * n);
    const bool sampleable = env_build_tables(tex, width, height, rows, rows + height);
    CK(cudaMemcpyAsync(dst, tex, bytes, cudaMemcpyHostToDevice, s), "environment upload");
    if (int r = slot_finish_upload(ctx, ctx->env, slot, "environment")) return r;
    ctx->envSampleable = sampleable;
    ctx->envW = width;
    ctx->envH = height;
    return 0;
}

// tpt_set_textures and tpt_set_emission_textures: the checks, the upload into one set's slots and its sizes. `fn` heads
// the error texts, `what` names the set in those of CUDA failures. `tables`: the slot also carries the layers' sampling
// tables, built here on the host (the emission set, tpt_env_tables.h).
static int set_textures(tpt_context* ctx, TextureSlots& ts, const char* fn, const char* what, const float* rgba, int width,
                        int height, int layers, const int* sphereLayers, int numSpheres, int onDevice, bool tables)
{
    // NULL: the calls issued from now on see every sphere without this set; those in flight keep reading their slot
    if (!rgba) { ts.slots.have = false; return 0; }
    if (width < 1 || height < 1 || layers < 1)
        return fail_msgf(ctx, "%s: width, height and layers must be >= 1 (got %d x %d x %d)", fn, width, height, layers);
    const long long plane = (long long)width * height, n = plane * layers;
    if (n >= (1LL << 31)) return fail_msgf(ctx, "%s: width * height * layers must be below 2^31 (got %lld)", fn, n);
    if (numSpheres < 0) return fail_msgf(ctx, "%s: numSpheres must be >= 0 (got %d)", fn, numSpheres);
    if (numSpheres > 0 && !sphereLayers) return fail_msgf(ctx, "%s: sphereLayers is NULL for %d spheres", fn, numSpheres);
    for (int i = 0; i < numSpheres; ++i)
        if (sphereLayers[i] < -1 || sphereLayers[i] >= layers)
            return fail_msgf(ctx, "%s: sphereLayers[%d] = %d is outside [-1, %d)", fn, i, sphereLayers[i], layers);
    auto bad_texel = [&](long long i, int c, float v) {
        return fail_msgf(ctx, "%s: texel of layer %lld (x %lld, y %lld) has %s = %g: RGB must be finite and not negative", fn,
                         i / plane, i % width, i % plane / width, c == 0 ? "R" : c == 1 ? "G" : "B", v);
    };
    CK(cudaSetDevice(ctx->device), "cudaSetDevice");
    if (onDevice)
    {
        if ((uintptr_t)rgba & 15) return fail_msgf(ctx, "%s: device rgba is not 16-byte aligned", fn);
        if (int r = check_device_buffer(ctx, fn, rgba, "rgba")) return r;
        if (int r = ensure_index_check(ctx)) return r;
    }
    else
        for (long long i = 0; i < n; ++i)
            for (int c = 0; c < 3; ++c)
                if (!env_channel_ok(rgba[4 * i + c])) return bad_texel(i, c, rgba[4 * i + c]);
    // The slot that is not current: the calls issued since the set's last upload read the other one. It holds the
    // texels and the sphere table behind them: 16 W H L + 4 numSpheres bytes; with tables, the padding and the tables
    // behind those (emit_slot_bytes), uploaded from a host copy of the slot in which they are built.
    const size_t texBytes = (size_t)n * 16;
    const size_t bytes = tables ? emit_slot_bytes(width, height, layers, numSpheres) : texBytes + (size_t)numSpheres * 4;
    int slot = 0;
    if (int r = slot_begin_upload(ctx, ts.slots, bytes, what, &slot)) return r;
    unsigned char* dst = (unsigned char*)ts.slots.ptr[slot];
    cudaStream_t s = ctx->uploadStream;
    std::vector<float> host(tables ? bytes / 4 : 0);
    if (onDevice)
    {
        // As tpt_set_environment checks a device map: R, G and B packed into the slot, checked as int32 bits by the
        // caller-list check (entry = channel index), in chunks whose entry indices fit the check's 32 bits. Then the
        // texels themselves, alpha included (never read).
        const long long kChunk = 1LL << 30;
        for (long long c0 = 0; c0 < n; c0 += kChunk)
        {
            const long long m = n - c0 < kChunk ? n - c0 : kChunk;
            CK(cudaMemcpy2DAsync(dst, 12, rgba + 4 * c0, 16, 12, (size_t)m, cudaMemcpyDefault, s), "pack texture RGB");
            CK(launch_list_check((const int*)dst, 3 * m, kEnvBitsLimit, ctx->dBadPixel, ctx->numSMs, s), "texture check launch");
            CK(cudaMemcpyAsync(ctx->hBadPixel, ctx->dBadPixel, sizeof(unsigned long long), cudaMemcpyDeviceToHost, s),
               "D2H texture check");
            // A refused texel leaves the current textures as they were.
            CK(cudaStreamSynchronize(s), "texture check sync");
            if (*ctx->hBadPixel != ~0ull)
            {
                const long long k = (long long)(*ctx->hBadPixel >> 32);
                uint32_t bits = (uint32_t)*ctx->hBadPixel;
                float v;
                memcpy(&v, &bits, 4);
                return bad_texel(c0 + k / 3, (int)(k % 3), v);
            }
            // with tables: the checked chunk's RGB back for the build, as tpt_set_environment does
            if (tables)
            {
                CK(cudaMemcpy2DAsync(host.data() + 4 * c0, 16, dst, 12, 12, (size_t)m, cudaMemcpyDeviceToHost, s), "D2H texture RGB");
                CK(cudaStreamSynchronize(s), "texture RGB sync");
            }
        }
        if (!tables) CK(cudaMemcpyAsync(dst, rgba, texBytes, cudaMemcpyDeviceToDevice, s), "texture upload");
    }
    else if (tables)
        memcpy(host.data(), rgba, texBytes);
    else
        CK(cudaMemcpyAsync(dst, rgba, texBytes, cudaMemcpyHostToDevice, s), "texture upload");
    bool sampleable = false;
    if (tables)
    {
        if (numSpheres > 0) memcpy(host.data() + 4 * n, sphereLayers, (size_t)numSpheres * 4);
        EnvAlias* tab = reinterpret_cast<EnvAlias*>(reinterpret_cast<unsigned char*>(host.data()) +
                                                    emit_table_offset(width, height, layers, numSpheres));
        sampleable = emit_build_tables(host.data(), width, height, layers, tab);
        CK(cudaMemcpyAsync(dst, host.data(), bytes, cudaMemcpyHostToDevice, s), "texture upload");
    }
    else if (numSpheres > 0)
        CK(cudaMemcpyAsync(dst + texBytes, sphereLayers, (size_t)numSpheres * 4, cudaMemcpyHostToDevice, s), "sphere layer upload");
    if (int r = slot_finish_upload(ctx, ts.slots, slot, what)) return r;
    ts.tables = tables;
    ts.sampleable = sampleable;
    ts.w = width;
    ts.h = height;
    ts.layers = layers;
    ts.spheres = numSpheres;
    return 0;
}

int tpt_set_textures(tpt_context* ctx, const float* rgba, int width, int height, int layers,
                     const int* sphereLayers, int numSpheres, int onDevice)
{
    if (!ctx) return (int)cudaErrorInvalidValue;
    return set_textures(ctx, ctx->tex, "tpt_set_textures", "textures", rgba, width, height, layers, sphereLayers, numSpheres,
                        onDevice, false);
}

int tpt_set_emission_textures(tpt_context* ctx, const float* rgba, int width, int height, int layers,
                              const int* sphereLayers, int numSpheres, int onDevice)
{
    if (!ctx) return (int)cudaErrorInvalidValue;
    return set_textures(ctx, ctx->emit, "tpt_set_emission_textures", "emission textures", rgba, width, height, layers,
                        sphereLayers, numSpheres, onDevice, true);
}

int tpt_read_ray_count(tpt_context* ctx, void* cudaStreamArg, long long* outRays)
{
    if (!ctx || !outRays) return (int)cudaErrorInvalidValue;
    CK(cudaSetDevice(ctx->device), "cudaSetDevice");
    cudaStream_t stream = cudaStreamArg ? (cudaStream_t)cudaStreamArg : ctx->stream;
    unsigned long long h[2] = {0, 0};
    CK(cudaMemcpyAsync(h, ctx->dAccum, sizeof(h), cudaMemcpyDeviceToHost, stream), "D2H accum");
    CK(cudaMemsetAsync(ctx->dAccum, 0, sizeof(unsigned long long), stream), "reset accum");
    CK(cudaStreamSynchronize(stream), "stream sync");
    *outRays = (long long)h[0];
    return 0;
}

int tpt_last_kernel_ms(tpt_context* ctx, float* outMs)
{
    if (!ctx || !outMs) return (int)cudaErrorInvalidValue;
    if (!ctx->haveTiming) return fail_msg(ctx, "tpt_last_kernel_ms: no draw yet");
    CK(cudaEventSynchronize(ctx->evStop), "event sync");
    CK(cudaEventElapsedTime(outMs, ctx->evStart, ctx->evStop), "event elapsed");
    return 0;
}

int tpt_last_launch_count(tpt_context* ctx) { return ctx ? ctx->lastLaunches : 0; }
long long tpt_last_scene_upload_bytes(tpt_context* ctx) { return ctx ? ctx->lastSceneUploadBytes : 0; }

int tpt_tonemap_rgba8(tpt_context* ctx, const float* image, int imageOnDevice, int width, int height,
                      unsigned char* dst, int dstOnDevice, int transfer, int bgr, int flipY, void* cudaStreamArg)
{
    if (!ctx || !image || !dst || width <= 0 || height <= 0) return (int)cudaErrorInvalidValue;
    if (transfer < 0 || transfer > 2) return fail_msg(ctx, "tpt_tonemap_rgba8: transfer 0..2");
    CK(cudaSetDevice(ctx->device), "cudaSetDevice");
    cudaStream_t stream = cudaStreamArg ? (cudaStream_t)cudaStreamArg : ctx->stream;
    const size_t outBytes = (size_t)width * height * 4;
    CallerBuffer in[] = {{"image", (void*)image, imageOnDevice != 0, 16, (size_t)width * height * 16, kStageImage, kCopyUp}};
    if (int r = stage_in(ctx, stream, in)) return r;
    unsigned char* dOut = dst;
    if (!dstOnDevice)
    {
        int r = ensure(ctx, (void**)&ctx->dScratch, &ctx->scratchCap, outBytes, "cudaMalloc tonemap out");
        if (r) return r;
        dOut = (unsigned char*)ctx->dScratch;
    }
    const int n = width * height;
    k_tonemap_rgba8<<<(n + 255) / 256, 256, 0, stream>>>((const float4*)in[0].dev, width, height, (uchar4*)dOut, transfer, bgr ? 1 : 0, flipY ? 1 : 0);
    CK(cudaGetLastError(), "tonemap launch");
    if (!dstOnDevice)
    {
        CK(cudaMemcpyAsync(dst, dOut, outBytes, cudaMemcpyDeviceToHost, stream), "D2H tonemap");
        CK(cudaStreamSynchronize(stream), "stream sync");
    }
    return 0;
}

int tpt_tonemap_srgb8(tpt_context* ctx, const float* image, int imageOnDevice, int width, int height,
                      unsigned char* dst, int dstOnDevice, void* cudaStreamArg)
{
    return tpt_tonemap_rgba8(ctx, image, imageOnDevice, width, height, dst, dstOnDevice, 0, 0, 1, cudaStreamArg);
}

int tpt_mem_alloc(tpt_context* ctx, unsigned long long bytes, void** outDevPtr)
{
    if (!ctx || !outDevPtr || !bytes) return (int)cudaErrorInvalidValue;
    CK(cudaSetDevice(ctx->device), "cudaSetDevice");
    CK(cudaMalloc(outDevPtr, (size_t)bytes), "cudaMalloc");
    CK(cudaMemset(*outDevPtr, 0, (size_t)bytes), "cudaMemset");
    return 0;
}
int tpt_mem_free(tpt_context* ctx, void* devPtr)
{
    if (!ctx) return (int)cudaErrorInvalidValue;
    CK(cudaSetDevice(ctx->device), "cudaSetDevice");
    CK(cudaFree(devPtr), "cudaFree");
    return 0;
}
int tpt_mem_copy(tpt_context* ctx, void* dst, const void* src, unsigned long long bytes, int kind)
{
    if (!ctx || !dst || !src || kind < 1 || kind > 3) return (int)cudaErrorInvalidValue;
    CK(cudaSetDevice(ctx->device), "cudaSetDevice");
    CK(cudaStreamSynchronize(ctx->stream), "stream sync");
    CK(cudaMemcpy(dst, src, (size_t)bytes, kind == 1 ? cudaMemcpyHostToDevice : kind == 2 ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice), "cudaMemcpy");
    return 0;
}
int tpt_ipc_export(tpt_context* ctx, void* devPtr, void* outHandle64)
{
    if (!ctx || !devPtr || !outHandle64) return (int)cudaErrorInvalidValue;
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    CK(cudaSetDevice(ctx->device), "cudaSetDevice");
    cudaIpcMemHandle_t h;
    CK(cudaIpcGetMemHandle(&h, devPtr), "cudaIpcGetMemHandle");
    memcpy(outHandle64, &h, 64);
    return 0;
}
int tpt_ipc_open(tpt_context* ctx, const void* handle64, void** outDevPtr)
{
    if (!ctx || !handle64 || !outDevPtr) return (int)cudaErrorInvalidValue;
    CK(cudaSetDevice(ctx->device), "cudaSetDevice");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, 64);
    CK(cudaIpcOpenMemHandle(outDevPtr, h, cudaIpcMemLazyEnablePeerAccess), "cudaIpcOpenMemHandle");
    return 0;
}
int tpt_ipc_close(tpt_context* ctx, void* devPtr)
{
    if (!ctx || !devPtr) return (int)cudaErrorInvalidValue;
    CK(cudaSetDevice(ctx->device), "cudaSetDevice");
    CK(cudaIpcCloseMemHandle(devPtr), "cudaIpcCloseMemHandle");
    return 0;
}

int tpt_debug_timeline(tpt_context* ctx, float* outMs, int capacity)
{
    if (!ctx || !outMs || capacity < 1) return (int)cudaErrorInvalidValue;
    CK(cudaEventSynchronize(ctx->evStop), "event sync");
    int n = 0;
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, ctx->evStart, ctx->tlKernelEnd), "elapsed");
    outMs[n++] = ms;
    for (int b = 0; b < ctx->tlBands && n < capacity; ++b)
    {
        CK(cudaEventElapsedTime(&ms, ctx->evStart, ctx->tlBand[b]), "elapsed");
        outMs[n++] = ms;
    }
    if (n < capacity) { CK(cudaEventElapsedTime(&ms, ctx->evStart, ctx->evStop), "elapsed"); outMs[n++] = ms; }
    return -n;   // negative count = number of entries written
}

int tpt_debug_libm(tpt_context* ctx, int fn, const float* in, float* out, long long n)
{
    if (!ctx || !in || !out || n <= 0 || fn < 0 || fn > 3) return (int)cudaErrorInvalidValue;
    CK(cudaSetDevice(ctx->device), "cudaSetDevice");
    float *dIn = nullptr, *dOut = nullptr;
    CK(cudaMalloc(&dIn, (size_t)n * 4), "cudaMalloc");
    cudaError_t e = cudaMalloc(&dOut, (size_t)n * 4);
    if (e == cudaSuccess) e = cudaMemcpyAsync(dIn, in, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) e = launch_debug_libm(fn, dIn, dOut, n, ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(out, dOut, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    cudaFree(dIn); cudaFree(dOut);
    if (e != cudaSuccess) return fail(ctx, e, "tpt_debug_libm");
    return 0;
}

int tpt_debug_hit(tpt_context* ctx, int kform, const float* rays, int* outId, float* outT, long long n)
{
    if (!ctx || !rays || !outId || !outT || n <= 0 || kform < 0 || kform > 5) return (int)cudaErrorInvalidValue;
    if (!ctx->scene.blob) return fail_msg(ctx, "tpt_debug_hit: no scene");
    if (kform == 4 && (ctx->scene.count + 3) / 4 * 4 > kParamPairSpheres) return fail_msg(ctx, "tpt_debug_hit: kform 4 takes at most 64 padded spheres");
    if (kform == 5 && !ctx->scene.halfOk) return fail_msg(ctx, "tpt_debug_hit: the scene has no half-precision pass 1 (kform 5)");
    CK(cudaSetDevice(ctx->device), "cudaSetDevice");
    float *dRays = nullptr, *dT = nullptr;
    int* dId = nullptr;
    cudaError_t e = cudaMalloc(&dRays, (size_t)n * 24);
    if (e == cudaSuccess) e = cudaMalloc(&dT, (size_t)n * 4);
    if (e == cudaSuccess) e = cudaMalloc(&dId, (size_t)n * 4);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(ctx->stream, ctx->uploadDone[ctx->curBlob], 0);
    if (e == cudaSuccess) e = cudaMemcpyAsync(dRays, rays, (size_t)n * 24, cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) e = launch_debug_hit(ctx->scene, kform, dRays, dId, dT, n, ctx->numSMs, ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(outId, dId, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(outT, dT, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    cudaFree(dRays); cudaFree(dT); cudaFree(dId);
    if (e != cudaSuccess) return fail(ctx, e, "tpt_debug_hit");
    return 0;
}

int tpt_debug_last_kernels(tpt_context* ctx, char* buf, int cap)
{
    if (!ctx || !buf || cap < 1) return -(int)cudaErrorInvalidValue;
    if (cudaError_t e = cudaSetDevice(ctx->device)) return -fail(ctx, e, "cudaSetDevice");
    int len = 0;
    buf[0] = '\0';
    const int kept = t_lastKernels.n < KernelRecord::kCap ? t_lastKernels.n : KernelRecord::kCap;
    for (int i = 0; i < kept; ++i)
    {
        const char* name = nullptr;
        cudaError_t e = cudaFuncGetName(&name, t_lastKernels.fn[i]);
        if (e != cudaSuccess) return -fail(ctx, e, "tpt_debug_last_kernels");
        const int need = (int)strlen(name) + (i ? 1 : 0);
        if (len + need + 1 > cap) return -fail_msg(ctx, "tpt_debug_last_kernels: buffer too small");
        if (i) buf[len++] = '\n';
        memcpy(buf + len, name, strlen(name) + 1);
        len += (int)strlen(name);
    }
    return t_lastKernels.n;
}

} // extern "C"
