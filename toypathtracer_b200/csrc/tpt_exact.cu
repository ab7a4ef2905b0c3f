// Exact ("replay") mode kernels. THIS TRANSLATION UNIT MUST BE COMPILED WITH -fmad=false: the integrator is
// written with plain float operators and relies on the compiler never contracting a*b+c (SURVEY.md §9.4: one
// contraction forks the row's RNG stream). Division and sqrt use the IEEE intrinsics explicitly.
//
// Work decomposition: the reference seeds one XorShift32 stream per (frame,row) and carries it serially across
// the row (Cpp/Source/Test.cpp:278-297), so the independent unit is a CHAIN = (frame, row). LANES lanes of a
// warp cooperate on one chain: all of them carry the (identical) integrator state, the ray-vs-all-spheres
// sweep is split across the lanes (sphere i -> lane i % LANES, SoA from shared memory) and the nearest hit is
// shuffle-reduced. LANES = 32 when chains are scarce (one 4-spp frame = `height` chains), 1 when thousands
// of frames are batched (1024 spp at 720p = 184 320 chains).
#include "tpt_integrator.cuh"
#include "tpt_device_utils.cuh"
#include "tpt_launch.h"
#include "tpt_refgpu.cuh"

namespace tpt {

// The (frame, row) of a chain. Consecutive chains = the same row in consecutive frames: neighbouring lanes trace the same
// pixels with different RNG streams (coherent geometry, similar path lengths), and the expensive bottom rows are
// scheduled first. Every kernel uses this order.
struct Chain
{
    int ri, fi;          // row index within the draw, frame index within the draw
    int y, frame;        // image row, frame number (seeds the row's RNG stream)
    size_t imgRow;       // first pixel of the row in p.image
};
template <class Index>
__device__ __forceinline__ Chain decode_chain(const DrawParams& p, Index chain)
{
    Chain c;
    c.ri = (int)(chain / (Index)p.numFrames);
    c.fi = (int)(chain % (Index)p.numFrames);
    c.y = p.row0 + c.ri * p.rowStep;
    c.frame = p.frame0 + c.fi;
    c.imgRow = (size_t)(p.packed ? c.ri : c.y) * p.width;
    return c;
}

// LANES consecutive lanes of the warp share one ray (LANES = 1, 8, 16 or 32).
template <int EXACT, int LANES>
__device__ __forceinline__ GroupHitter<EXACT, LANES> group_hitter(int lane)
{
    GroupHitter<EXACT, LANES> h;
    h.sub = lane % LANES;
    h.mask = LANES == 32 ? 0xffffffffu : (((1u << (LANES & 31)) - 1u) << (lane - h.sub));
    return h;
}

// Test.cpp:293-295: prev*lerpFac + col*(1-lerpFac) per component; alpha is never written by the CPU path
__device__ __forceinline__ void blend(float4& prev, V3 col, float lerpFac)
{
    const float oneMinus = 1.0f - lerpFac;
    prev.x = prev.x * lerpFac + col.x * oneMinus;
    prev.y = prev.y * lerpFac + col.y * oneMinus;
    prev.z = prev.z * lerpFac + col.z * oneMinus;
}

// A finished pixel of chain c: blended into p.image when the draw has one frame, else stored in p.scratch for
// k_resolve_exact, which blends the frames in order.
__device__ __forceinline__ void store_pixel(const DrawParams& p, const Chain& c, int x, V3 col, float lerpFac)
{
    if (p.numFrames == 1)
    {
        float4* px = reinterpret_cast<float4*>(p.image + (c.imgRow + x) * 4);
        float4 prev = *px;
        blend(prev, col, lerpFac);
        *px = prev;
    }
    else
    {
        float4* px = reinterpret_cast<float4*>(p.scratch) + ((size_t)c.fi * p.numRows + c.ri) * p.width + x;
        *px = make_float4(col.x, col.y, col.z, 0.0f);
    }
}

template <int LANES>
__global__ void k_trace_exact(DrawParams p, const unsigned char* __restrict__ blob, SceneBlobLayout L,
                              int count, int nLights, uint32_t stagedBytes)
{
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ uint64_t bar;
    stage_blob(smem, blob, stagedBytes, &bar);
    SceneView sc = make_view(smem, blob, L, stagedBytes, count, nLights);

    const long long chain = ((long long)blockIdx.x * blockDim.x + threadIdx.x) / LANES;
    const long long totalChains = (long long)p.numRows * p.numFrames;
    if (chain >= totalChains) return;
    const Chain ch = decode_chain(p, chain);
    const GroupHitter<1, LANES> hitter = group_hitter<1, LANES>(threadIdx.x & 31);

    uint32_t state = row_seed(ch.y, ch.frame);
    unsigned rc = 0;
    const float lerpFac = lerp_fac(ch.frame, p.flags);
    for (int x = 0; x < p.width; ++x)
    {
        V3 col = pixel_exact(sc, p.cam, x, ch.y, p.spp, p.invWidth, p.invHeight, state, rc, hitter);
        if (hitter.sub == 0) store_pixel(p, ch, x, col, lerpFac);
    }
    if (hitter.sub == 0) atomicAdd(p.rayCounter + ch.fi, (unsigned long long)rc);
}

// One thread per chain, flat form: every loop iteration is one xchain_step() = one sphere sweep, so the lanes of a
// warp (the same row in 32 consecutive frames) stay converged on the sweep whatever their paths are doing.
template <int LANES>
__global__ void __launch_bounds__(128)
k_trace_exact_flat(DrawParams p, const unsigned char* __restrict__ blob, SceneBlobLayout L, int count, int nLights, uint32_t stagedBytes)
{
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ uint64_t bar;
    stage_blob(smem, blob, stagedBytes, &bar);
    SceneView sc = make_view(smem, blob, L, stagedBytes, count, nLights);
    const long long chain = ((long long)blockIdx.x * blockDim.x + threadIdx.x) / LANES;
    const long long totalChains = (long long)p.numRows * p.numFrames;
    if (chain >= totalChains) return;
    const Chain ch = decode_chain(p, chain);
    const float lerpFac = lerp_fac(ch.frame, p.flags);
    // LANES lanes share the chain: replicated state, split sweep (see k_trace_exact)
    const GroupHitter<1, LANES> hitter = group_hitter<1, LANES>(threadIdx.x & 31);
    unsigned rc = 0;
    XChain c;
    xchain_begin(c, p.cam, ch.y, ch.frame, p.invWidth, p.invHeight);
    while (c.x < p.width)
    {
        const int x = c.x;
        V3 col;
        if (xchain_step(sc, p.cam, c, ch.y, p.spp, p.width, p.invWidth, p.invHeight, rc, hitter, col) && hitter.sub == 0)
            store_pixel(p, ch, x, col, lerpFac);
    }
    if (hitter.sub == 0) atomicAdd(p.rayCounter + ch.fi, (unsigned long long)rc);
}

// Sequential progressive blend of the per-frame colours (Test.cpp:272-276,293-295), one thread per pixel,
// frames in order so the float sequence is the reference's.
__global__ void k_resolve_exact(DrawParams p)
{
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long n = (long long)p.numRows * p.width;
    if (idx >= n) return;
    const int ri = (int)(idx / p.width), x = (int)(idx % p.width);
    const int y = p.row0 + ri * p.rowStep;
    float4* px = reinterpret_cast<float4*>(p.image) + (size_t)(p.packed ? ri : y) * p.width + x;
    float4 prev = *px;
    const float4* s = reinterpret_cast<const float4*>(p.scratch) + idx;
    for (int fi = 0; fi < p.numFrames; ++fi, s += n)
    {
        const float lerpFac = lerp_fac(p.frame0 + fi, p.flags);
        float4 col = ld_stream_f4(reinterpret_cast<const float*>(s));
        blend(prev, v3(col.x, col.y, col.z), lerpFac);
    }
    *px = prev;
}


// ---- split kernel: one PATH warp + H SHADE warps per chain ----------------------------------------------------------------
// One 4-spp frame is only `height` chains, and a chain is a serial dependency through its RNG stream — but only through
// ray generation, the sweep and the scatter direction (see xpath_sample). Everything else (explicit light sampling with
// its shadow-ray sweeps — 44 % of all rays —, emission/attenuation, the back-to-front fold, the blend and the store) is
// taken off that critical path: warp 0 of the CTA walks the chain and pushes one 48-byte event per path vertex into a
// shared-memory ring (mbarrier full/empty pairs per slot); shade warp h consumes the samples k with k % H == h:
//   * the lights of a Lambert vertex are sampled by the two HALF-warps at once (light j on lanes 0-15, light j+1 on lanes
//     16-31, each half sweeping the spheres 16-wide and reducing its nearest hit with REDUX under its own mask),
//     contributions added in the reference's light order;
//   * finished samples go to a per-pixel slot; the warp that completes a pixel sums them in sample order (Test.cpp:289-291),
//     blends (Test.cpp:293-295) and stores the float4.
// Bit parity: tests/test_host_sim.py (the same xpath_sample/xshade_event on the host) and tests/test_gpu_exact.py.
constexpr int kRingDepth = 16;      // events per shade warp in flight
constexpr int kPixSlots = 16;       // pixels whose samples may be in flight (see the capacity argument in DESIGN.md)
constexpr int kSplitMaxSpp = 8;
enum { XE_BEGIN = 4, XE_QUIT = 5 };   // cluster kernel only: a chain starts / the path warp is done

// One event of xpath_sample(): a, b, c in q0..q2.xyz, the RNG state in q1.w, and in q0.w the tag: the type (XE_*) in the
// low 3 bits, above them the material id (XE_BEGIN: the chain index).
struct __align__(16) XEventSlot
{
    float4 q0, q1, q2;
    __device__ __forceinline__ int type() const { return __float_as_int(q0.w) & 7; }
    __device__ __forceinline__ int mid() const { return __float_as_int(q0.w) >> 3; }
};
__device__ __forceinline__ XEventSlot make_event(int type, int mid, V3 a, V3 b, V3 c, uint32_t rng)
{
    return {make_float4(a.x, a.y, a.z, __int_as_float(type | (mid << 3))), make_float4(b.x, b.y, b.z, __uint_as_float(rng)),
            make_float4(c.x, c.y, c.z, 0.0f)};
}
template <class LightFn>
__device__ __forceinline__ bool shade_event(const SceneView& sc, XShade& sh, const XEventSlot& e, LightFn&& lights, V3& result)
{
    return xshade_event(sc, sh, e.type(), e.mid(), v3(e.q0.x, e.q0.y, e.q0.z), v3(e.q1.x, e.q1.y, e.q1.z),
                        v3(e.q2.x, e.q2.y, e.q2.z), __float_as_uint(e.q1.w), lights, result);
}

// Event number `seq` of a ring: its slot, and the parity of that slot's barriers on this lap.
struct RingPos { uint32_t slot, phase; };
__device__ __forceinline__ RingPos ring_pos(uint32_t seq) { return {seq % kRingDepth, (seq / kRingDepth) & 1u}; }

// Returns seq[h] and increments it. The unrolled select keeps the array in registers for a runtime h.
template <int N>
__device__ __forceinline__ uint32_t next_seq(uint32_t (&seq)[N], int h)
{
    uint32_t sq = 0;
#pragma unroll
    for (int i = 0; i < N; ++i) if (i == h) sq = seq[i];
#pragma unroll
    for (int i = 0; i < N; ++i) if (i == h) seq[i] = sq + 1;
    return sq;
}

__device__ __forceinline__ void mbar_arrive(uint64_t* bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// lightE of a Lambert vertex on a shade warp (Test.cpp:96-133): the two half-warps (grp = lane / 16) sample and trace two
// lights at a time, and the contributions are added in the reference's light order (Test.cpp:96).
template <int SMODE>
__device__ __forceinline__ V3 shade_lights(const SceneView& sc, const GroupHitter<SMODE, 16>& hitter, int grp, int mid, V3 pos,
                                           V3 normal, V3 rdir, V3 albedo, uint32_t rng)
{
    V3 lightE = v3(0, 0, 0);
    int myJ = -1, kk = 0;
    uint32_t myRng = 0;
    auto run_batch = [&]() {
        V3 contrib = v3(0, 0, 0);
        bool reached = false;
        if (myJ >= 0)
        {
            const LightRec Lr = sc.lights[myJ];
            V3 l;
            sample_light<SMODE>(Lr, pos, normal, rdir, albedo, myRng, l, contrib);
            float ts;
            reached = hitter.hit(sc, pos, l, TPT_MIN_T, TPT_MAX_T, ts) == Lr.id;
        }
        __syncwarp();
#pragma unroll
        for (int g = 0; g < 2; ++g)
        {
            const bool r = __shfl_sync(0xffffffffu, reached ? 1 : 0, g * 16) != 0;
            const V3 cg = v3(__shfl_sync(0xffffffffu, contrib.x, g * 16), __shfl_sync(0xffffffffu, contrib.y, g * 16),
                             __shfl_sync(0xffffffffu, contrib.z, g * 16));
            if (r) lightE = lightE + cg;
        }
        myJ = -1;
    };
    for (int j = 0; j < sc.nLights; ++j)
    {
        if (sc.lights[j].id == mid) continue;                  // Test.cpp:100
        if ((kk & 1) == grp) { myJ = j; myRng = rng; }
        XorShift32(rng); XorShift32(rng);                      // eps1, eps2 of this light (Test.cpp:112)
        if ((++kk & 1) == 0) run_batch();
    }
    if (kk & 1) run_batch();
    return lightE;
}

// Hands sample s of the pixel in slot ps to the slot; the warp whose sample completes the pixel sums the samples in sample
// order (Test.cpp:289-291), scales by invSpp (Test.cpp:291) and stores the pixel. All 32 lanes call it.
__device__ __forceinline__ void finish_sample(float (*pixRes)[kSplitMaxSpp][3], unsigned* pixCnt, int ps, int s, int spp,
                                              float invSpp, V3 result, int lane, const DrawParams& p, const Chain& ch, int x,
                                              float lerpFac)
{
    unsigned old = 0;
    if (lane == 0)
    {
        pixRes[ps][s][0] = result.x; pixRes[ps][s][1] = result.y; pixRes[ps][s][2] = result.z;
        __threadfence_block();
        old = atomicInc(&pixCnt[ps], (unsigned)spp - 1u);      // wraps to 0 with the pixel's last sample
    }
    old = __shfl_sync(0xffffffffu, old, 0);
    if (old == (unsigned)spp - 1u && lane == 0)
    {
        __threadfence_block();
        V3 col = v3(0, 0, 0);
        for (int t = 0; t < spp; ++t)
            col = col + v3(((volatile float*)pixRes[ps][t])[0], ((volatile float*)pixRes[ps][t])[1], ((volatile float*)pixRes[ps][t])[2]);
        store_pixel(p, ch, x, col * invSpp, lerpFac);
    }
    __syncwarp();
}

constexpr int split_block_threads(int H) { return H <= 3 ? 128 : 32 * (1 + H); }   // 4-warp CTAs: one role per SM sub-partition

template <int H, int DRY = 0, int SMODE = 1>     // DRY: timing probes — 1 = shade warps only drain the rings, 2 = everything but the light sampling;
                                                 // SMODE: arithmetic flavour of the shade warps (1 = inlined: 882 Mray/s at 720p; 2 = shared out-of-line sqrt/div/libm: 780)
// SMODE 2 is held to 64 registers (8 CTAs per SM) like the other forms; ptxas would otherwise give it 72 to spill less
__global__ void __launch_bounds__(split_block_threads(H), SMODE == 2 ? 8 : 0)
k_trace_exact_split(DrawParams p, const unsigned char* __restrict__ blob, SceneBlobLayout L, int count, int nLights, uint32_t stagedBytes)
{
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ uint64_t bar;
    __shared__ uint64_t fullBar[H][kRingDepth], emptyBar[H][kRingDepth];
    __shared__ XEventSlot ring[H][kRingDepth];
    __shared__ float pixRes[kPixSlots][kSplitMaxSpp][3];
    __shared__ unsigned pixCnt[kPixSlots];
    stage_blob(smem, blob, stagedBytes, &bar);
    if (threadIdx.x == 0)
    {
        for (int h = 0; h < H; ++h)
            for (int i = 0; i < kRingDepth; ++i) { mbar_init(&fullBar[h][i], 1); mbar_init(&emptyBar[h][i], 1); }
        mbar_fence_init();
    }
    if (threadIdx.x < kPixSlots) pixCnt[threadIdx.x] = 0;
    __syncthreads();
    SceneView sc = make_view(smem, blob, L, stagedBytes, count, nLights);

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;     // (rotating the roles over the 4 sub-partitions: no effect, measured)
    const long long chain = blockIdx.x;
    const Chain ch = decode_chain(p, chain);
    const int spp = p.spp;
    const uint32_t totalSamples = (uint32_t)p.width * (uint32_t)spp;

    if (warp == 0)
    {
        // ---- PATH warp: the chain's RNG stream, sweeps split over the 32 lanes
        const GroupHitter<1, 32> hitter = group_hitter<1, 32>(lane);
        uint32_t rng = row_seed(ch.y, ch.frame);
        unsigned rc = 0;
        uint32_t seq[H];
#pragma unroll
        for (int h = 0; h < H; ++h) seq[h] = 0;
        uint32_t k = 0;
        for (int x = 0; x < p.width; ++x)
            for (int s = 0; s < spp; ++s, ++k)
            {
                const int h = H == 1 ? 0 : (int)(k % (uint32_t)H);
                auto emit = [&](int type, int mid, V3 a, V3 b, V3 c, uint32_t erng) {
                                 const RingPos r = ring_pos(next_seq(seq, h));
                                 mbar_wait_sleep(&emptyBar[h][r.slot], r.phase ^ 1u);      // slot free (passes at once on a fresh barrier)
                                 if (lane == 0)
                                 {
                                     ring[h][r.slot] = make_event(type, mid, a, b, c, erng);
                                     mbar_arrive(&fullBar[h][r.slot]);          // release: the stores above are visible to the waiter
                                 }
                             };
                xpath_sample(sc, p.cam, x, ch.y, p.invWidth, p.invHeight, rng, rc, hitter, emit);
            }
        if (lane == 0) atomicAdd(p.rayCounter + ch.fi, (unsigned long long)rc);
        return;
    }

    // ---- SHADE warp h: samples k = h, h + H, ...
    const int h = warp - 1;
    if (h >= H) return;                                          // padding warp of the 4-warp CTA
    const GroupHitter<SMODE, 16> hitter = group_hitter<SMODE, 16>(lane);   // half-warp = one light
    const float lerpFac = lerp_fac(ch.frame, p.flags);
    const float invSpp = M<SMODE>::div_(1.0f, (float)spp);
    uint32_t seq = 0;
    auto lights = [&](int mid, V3 pos, V3 normal, V3 rdir, V3 albedo, uint32_t rng) -> V3 {
        if (DRY == 2) return v3(0, 0, 0);                        // probe: shading without the light sampling
        return shade_lights<SMODE>(sc, hitter, lane >> 4, mid, pos, normal, rdir, albedo, rng);
    };

    for (uint32_t k = (uint32_t)h; k < totalSamples; k += (uint32_t)H)
    {
        const int x = (int)(k / (uint32_t)spp), s = (int)(k - (uint32_t)x * (uint32_t)spp);
        XShade sh;
        xshade_begin(sh);
        V3 result;
        for (;;)
        {
            const RingPos r = ring_pos(seq++);
            mbar_wait_sleep(&fullBar[h][r.slot], r.phase);
            const XEventSlot e = ring[h][r.slot];
            __syncwarp();
            if (lane == 0) mbar_arrive(&emptyBar[h][r.slot]);
            if (DRY == 1) { if (e.type() >= XE_END_SKY) { result = v3(0, 0, 0); break; } continue; }   // probe: path warp alone
            if (shade_event(sc, sh, e, lights, result)) break;
        }
        // hand the sample to its pixel; whoever completes the pixel finishes it
        finish_sample(pixRes, pixCnt, x % kPixSlots, s, spp, invSpp, result, lane, p, ch, x, lerpFac);
    }
}

// ---- cluster form of the split kernel: the two roles on DIFFERENT SMs ---------------------------------------------------------
// ncu on k_trace_exact_split: 17 % of the stall samples are `no_instructions`, i-cache hit rate 82 % (99.7 % for the path
// warp alone) — path code and shade code together (~54 KB) do not fit the instruction cache of an SM that hosts both
// roles, and the path warp, whose latency IS the frame time, pays for it. Here a thread-block CLUSTER of two CTAs, each
// sized to own its SM, splits the roles by SM: CTA 0 runs kCPathWarps path warps (each pulls chains from a global counter),
// CTA 1 runs the kCH shade warps of each of them. The event rings and the `full` barriers live in the shade CTA's shared
// memory and are written/arrived over DSMEM (st.shared::cluster / mbarrier.arrive.release.cluster), the `empty` barriers
// in the path CTA's; a chain starts with an XE_BEGIN event and the kernel ends with XE_QUIT.
constexpr int kCPathWarps = 10;
constexpr int kCH = 2;
constexpr int kCThreads = 32 * kCPathWarps * kCH;

struct ClusterShared
{
    uint64_t fullBar[kCPathWarps][kCH][kRingDepth];       // used in CTA 1 (waited on locally, arrived remotely)
    uint64_t emptyBar[kCPathWarps][kCH][kRingDepth];      // used in CTA 0
    XEventSlot ring[kCPathWarps][kCH][kRingDepth];        // CTA 1
    float pixRes[kCPathWarps][kPixSlots][kSplitMaxSpp][3];
    unsigned pixCnt[kCPathWarps][kPixSlots];
};

__device__ __forceinline__ uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ uint32_t map_to_cta(const void* localSmem, uint32_t rank)
{
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_u32(localSmem)), "r"(rank));
    return r;
}
__device__ __forceinline__ void cluster_sync_all()
{
    asm volatile("barrier.cluster.arrive.release.aligned;\n barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_remote(uint32_t clusterAddr)
{
    asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(clusterAddr) : "memory");
}
__device__ __forceinline__ void st_cluster_f4(uint32_t clusterAddr, float4 v)
{
    asm volatile("st.shared::cluster.v4.f32 [%0], {%1,%2,%3,%4};" ::"r"(clusterAddr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(kCThreads, 1)
k_trace_exact_cluster(DrawParams p, const unsigned char* __restrict__ blob, SceneBlobLayout L, int count, int nLights, uint32_t stagedBytes)
{
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ uint64_t bar;
    __shared__ ClusterShared cs;
    stage_blob(smem, blob, stagedBytes, &bar);
    for (int i = threadIdx.x; i < kCPathWarps * kCH * kRingDepth; i += blockDim.x)
    {
        mbar_init(&cs.fullBar[0][0][0] + i, 1);
        mbar_init(&cs.emptyBar[0][0][0] + i, 1);
    }
    if (threadIdx.x < kCPathWarps * kPixSlots) (&cs.pixCnt[0][0])[threadIdx.x] = 0;
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncthreads();
    cluster_sync_all();                                   // both CTAs' barriers exist before anyone touches them
    SceneView sc = make_view(smem, blob, L, stagedBytes, count, nLights);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t rank = cluster_ctarank();
    const long long totalChains = (long long)p.numRows * p.numFrames;
    const int spp = p.spp;

    if (rank == 0 && warp < kCPathWarps)
    {
        // ---- PATH warp `warp`
        const GroupHitter<1, 32> hitter = group_hitter<1, 32>(lane);
        uint32_t seq[kCH];
#pragma unroll
        for (int h = 0; h < kCH; ++h) seq[h] = 0;
        auto emit_to = [&](int h, int type, int mid, V3 a, V3 b, V3 c, uint32_t erng) {
            const RingPos r = ring_pos(next_seq(seq, h));
            mbar_wait_sleep<true>(&cs.emptyBar[warp][h][r.slot], r.phase ^ 1u);
            if (lane == 0)
            {
                const XEventSlot ev = make_event(type, mid, a, b, c, erng);
                const uint32_t e = map_to_cta(&cs.ring[warp][h][r.slot], 1);
                st_cluster_f4(e, ev.q0);
                st_cluster_f4(e + 16, ev.q1);
                st_cluster_f4(e + 32, ev.q2);
                mbar_arrive_remote(map_to_cta(&cs.fullBar[warp][h][r.slot], 1));
            }
        };
        const V3 zero = v3(0, 0, 0);
        for (;;)
        {
            unsigned chainU = 0;
            if (lane == 0) chainU = atomicAdd(p.workCounter, 1u);
            chainU = __shfl_sync(0xffffffffu, chainU, 0);
            if ((long long)chainU >= totalChains) break;
            const Chain ch = decode_chain(p, chainU);
#pragma unroll
            for (int h = 0; h < kCH; ++h) emit_to(h, XE_BEGIN, (int)chainU, zero, zero, zero, 0u);
            uint32_t rng = row_seed(ch.y, ch.frame);
            unsigned rc = 0;
            uint32_t k = 0;
            for (int x = 0; x < p.width; ++x)
                for (int s = 0; s < spp; ++s, ++k)
                {
                    const int h = (int)(k % (uint32_t)kCH);
                    xpath_sample(sc, p.cam, x, ch.y, p.invWidth, p.invHeight, rng, rc, hitter,
                                 [&](int type, int mid, V3 a, V3 b, V3 c, uint32_t erng) { emit_to(h, type, mid, a, b, c, erng); });
                }
            if (lane == 0) atomicAdd(p.rayCounter + ch.fi, (unsigned long long)rc);
        }
#pragma unroll
        for (int h = 0; h < kCH; ++h) emit_to(h, XE_QUIT, 0, zero, zero, zero, 0u);
    }
    else if (rank == 1)
    {
        // ---- SHADE warp: serves path warp pw, samples k with k % kCH == h
        const int pw = warp / kCH, h = warp % kCH;
        const GroupHitter<2, 16> hitter = group_hitter<2, 16>(lane);
        const float invSpp = M<2>::div_(1.0f, (float)spp);
        uint32_t seq = 0, k = 0, pixBase = 0, chainsSeen = 0;
        Chain ch = {};
        float lerpFac = 0.0f;
        XShade sh;
        xshade_begin(sh);
        auto lights = [&](int mid, V3 pos, V3 normal, V3 rdir, V3 albedo, uint32_t rng) -> V3 {
            return shade_lights<2>(sc, hitter, lane >> 4, mid, pos, normal, rdir, albedo, rng);
        };

        for (;;)
        {
            const RingPos r = ring_pos(seq++);
            mbar_wait_sleep<true>(&cs.fullBar[pw][h][r.slot], r.phase);
            const XEventSlot e = cs.ring[pw][h][r.slot];
            __syncwarp();
            if (lane == 0) mbar_arrive_remote(map_to_cta(&cs.emptyBar[pw][h][r.slot], 0));
            if (e.type() == XE_QUIT) break;
            if (e.type() == XE_BEGIN)
            {
                pixBase = chainsSeen++ * (uint32_t)p.width;   // pixel slots are indexed by a running pixel number across chains
                ch = decode_chain(p, (unsigned)e.mid());
                lerpFac = lerp_fac(ch.frame, p.flags);
                k = (uint32_t)h;
                xshade_begin(sh);
                continue;
            }
            V3 result;
            if (!shade_event(sc, sh, e, lights, result)) continue;
            // sample k of the chain finished
            const int x = (int)(k / (uint32_t)spp), s = (int)(k - (uint32_t)x * (uint32_t)spp);
            const int ps = (int)((pixBase + (uint32_t)x) % (uint32_t)kPixSlots);
            finish_sample(cs.pixRes[pw], cs.pixCnt[pw], ps, s, spp, invSpp, result, lane, p, ch, x, lerpFac);
            k += (uint32_t)kCH;
            xshade_begin(sh);
        }
    }
    // nobody leaves while the partner CTA may still address this CTA's shared memory
    __syncthreads();
    cluster_sync_all();
}

// Allows `dyn` bytes of dynamic shared memory for one of the trace kernels and launches it.
template <class Kernel>
static cudaError_t launch_chains(Kernel kern, long long grid, int block, size_t dyn, const DrawParams& p, const SceneDev& sc,
                                 cudaStream_t stream)
{
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn);
    if (e != cudaSuccess) return e;
    return launch_trace(kern, (unsigned)grid, block, dyn, stream, p, sc.blob, sc.layout, sc.count, sc.nLights, sc.stagedBytes);
}

static cudaError_t launch_exact_cluster(const DrawParams& p, const SceneDev& sc, int numSMs, cudaStream_t stream)
{
    const long long totalChains = (long long)p.numRows * p.numFrames;
    if (p.spp > kSplitMaxSpp || totalChains >= (1LL << 27)) return cudaErrorInvalidValue;   // the chain index travels in a tag
    cudaError_t e = cudaMemsetAsync(p.workCounter, 0, sizeof(unsigned int), stream);
    if (e != cudaSuccess) return e;
    long long clusters = numSMs / 2;
    const long long need = (totalChains + kCPathWarps - 1) / kCPathWarps;
    if (clusters > need) clusters = need;
    // one CTA per SM: ask for more than half of an SM's shared memory
    const size_t wantDyn = 118 * 1024;
    const size_t dyn = sc.stagedBytes > wantDyn ? sc.stagedBytes : wantDyn;
    return launch_chains(k_trace_exact_cluster, 2 * clusters, kCThreads, dyn, p, sc, stream);
}

// one CTA per chain; a pixel slot holds at most kSplitMaxSpp samples
template <int H, int DRY = 0, int SMODE = 1>
static cudaError_t launch_exact_split_t(const DrawParams& p, const SceneDev& sc, cudaStream_t stream)
{
    const long long totalChains = (long long)p.numRows * p.numFrames;
    if (p.spp > kSplitMaxSpp || totalChains > 0x7fffffffLL) return cudaErrorInvalidValue;
    return launch_chains(k_trace_exact_split<H, DRY, SMODE>, totalChains, split_block_threads(H), sc.stagedBytes, p, sc, stream);
}

template <int LANES>
static cudaError_t launch_exact_t(const DrawParams& p, const SceneDev& sc, cudaStream_t stream, int block)
{
    const long long threads = (long long)p.numRows * p.numFrames * LANES;
    return launch_chains(k_trace_exact<LANES>, (threads + block - 1) / block, block, sc.stagedBytes, p, sc, stream);
}

template <int LANES>
static cudaError_t launch_exact_flat_t(const DrawParams& p, const SceneDev& sc, cudaStream_t stream)
{
    const long long threads = (long long)p.numRows * p.numFrames * LANES;
    return launch_chains(k_trace_exact_flat<LANES>, (threads + 127) / 128, 128, sc.stagedBytes, p, sc, stream);
}

__global__ void k_debug_libm(int fn, const float* __restrict__ in, float* __restrict__ out, long long n)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float x = in[i];
    out[i] = fn == 0 ? M<true>::sin_(x) : (fn == 1 ? M<true>::cos_(x) : (fn == 2 ? M<true>::pow5_(x) : tptlibm::powf_glibc(x, 1.0f / 3.0f)));
}

cudaError_t launch_debug_libm(int fn, const float* dIn, float* dOut, long long n, cudaStream_t stream)
{
    k_debug_libm<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(fn, dIn, dOut, n);
    return cudaGetLastError();
}

cudaError_t launch_refgpu_exact(const DrawParams& p, const SceneDev& sc, int numSMs, cudaStream_t stream)
{
    return launch_refgpu_t<true>(p, sc, numSMs, stream);
}

cudaError_t launch_resolve_exact(const DrawParams& p, cudaStream_t stream)
{
    const long long n = (long long)p.numRows * p.width;
    note_launch();
    k_resolve_exact<<<(int)((n + 255) / 256), 256, 0, stream>>>(p);
    return cudaGetLastError();
}

cudaError_t launch_exact(const DrawParams& p, const SceneDev& sc, int lanes, int numSMs, cudaStream_t stream, bool resolve)
{
    const long long totalChains = (long long)p.numRows * p.numFrames;
    if (lanes <= 0)
    {
        // few chains: the split kernel (2 shade warps) hides the shading latency best; thousands of chains: 32 lanes per
        // chain, then 8; from ~100k chains one lane per chain in the flat form fills the GPU on its own
        lanes = totalChains >= 100000 ? 1 : (totalChains >= 20000 ? 8 : (totalChains <= 2400 && p.spp <= kSplitMaxSpp ? 65 : 32));
    }
    // nested form: smaller CTAs when there are few chains, so that they still spread over all SMs
    const long long threads = totalChains * lanes;
    const int block = threads >= numSMs * 256LL ? 128 : (threads >= numSMs * 64LL ? 64 : 32);
    cudaError_t e;
    switch (lanes)
    {
    case 1: e = launch_exact_flat_t<1>(p, sc, stream); break;
    case 2: e = launch_exact_t<1>(p, sc, stream, block); break;      // nested-loop form, one lane per chain (kept for comparison)
    case 8: e = launch_exact_t<8>(p, sc, stream, block); break;
    case 9: e = launch_exact_flat_t<8>(p, sc, stream); break;        // flat form with 8 lanes per chain: measured 2x SLOWER than
                                                                     // the nested form at 11 520 chains (221 vs 111 ms), comparison only
    case 32: e = launch_exact_t<32>(p, sc, stream, block); break;
    // split kernel: path warp + 1..4 shade warps per chain
    case 64: e = launch_exact_split_t<1>(p, sc, stream); break;
    case 65: e = launch_exact_split_t<2>(p, sc, stream); break;
    case 66: e = launch_exact_split_t<3>(p, sc, stream); break;
    case 67: e = launch_exact_split_t<4>(p, sc, stream); break;
    case 68: e = launch_exact_split_t<2, 2>(p, sc, stream); break;  // 68 / 69: timing probes (no light sampling / path warp
    case 69: e = launch_exact_split_t<2, 1>(p, sc, stream); break;  // alone); the image is NOT valid
    case 70: e = launch_exact_cluster(p, sc, numSMs, stream); break; // split kernel, roles on different SMs (2-CTA clusters)
    case 71: e = launch_exact_split_t<2, 0, 2>(p, sc, stream); break;   // comparison: shade warps calling shared out-of-line sqrt/div/libm
    default: return cudaErrorInvalidValue;
    }
    if (e != cudaSuccess) return e;
    if (p.numFrames > 1 && resolve) e = launch_resolve_exact(p, stream);
    return e;
}

} // namespace tpt
