"""The fast estimator replayed sample by sample: every draw of a sample's own XorShift32 stream, every vertex of its path
(Lambert, rough metal, glass, light-sampled shadow rays, the depth cap, the sky or an environment map) in float64, with
how far the kernel's float32 and MUFU arithmetic can be from it.

A fast sample is deterministic given its stream: each draw is an integer XorShift32 step, RandomFloat01 is exact, and every
sampler draws a fixed number of values (camera jitter 2 + lens 2, Lambert bounce 2, each light cone 2, rough metal 3 and
none at roughness 0, glass 1). So the float64 restatement of path_step below, fed the kernel's own draws in the kernel's
order, follows the kernel's path vertex by vertex; where every decision along it has a clear margin the kernel's value for
that one sample must match. replay() returns per sample: the value, the rays traced (shadow rays included), a
well-conditioned verdict, a value tolerance, the path (hit ids per traced ray), the draws consumed and feature flags.

Conditioning: mirror_chain._nearest carries the origin and direction uncertainty (eo, ed) of every ray through the sweep,
and the hit point and normal errors through pos = o + t d and (pos - s) * invRadius, as mirror_chain.chains does; on top of
that this module carries them through
  Lambert     nextDir = normalize(n + u): ill conditioned when |n + u| is small (the up-check below catches it);
  light cone  sw = normalize(centre - o), the Duff basis (its sign branch on sw.z), cosAMax, cosA, sinA (ill conditioned
              near sinA = 0 only through the square root's slope), the shadow ray's hit id (near the silhouette the sweep
              is ambiguous) and the sign of dot(l, nl) (within its error the ray's weight is below the tolerance);
  rough metal dot(out, n) > 0 against the error of out = reflect + roughness * unit-ball sample;
  glass       the sign of dn, the refraction discriminant, and u < reflProb against the error of reflProb;
and every new direction must leave (or, refracted, enter) the surface by more than its error.

MUFU bounds assumed (each a multiple of the documented figure, so that the float32 emulation of
test_sample_replay_oracle.py, which perturbs every MUFU result within these bounds, is a fair check of the verdict):
  rsqrt.approx.f32 (normalize)     relative 2^-22.9, PTX ISA; taken as mirror_chain.NORM_ERR = 2^-20 for the whole normalize
  sqrt.approx.f32                  relative 2^-21 (PTX ISA documents 2^-23 for the full range)
  __sincosf on [0, 2 pi)           absolute 2^-19 (CUDA C Programming Guide: 2^-21.41 on [-pi, pi]; the argument reduction
                                   x / 2 pi adds at most 2 pi * 2^-24 on [pi, 2 pi))
  __powf(u, 1/3) = ex2(lg2(u) / 3) relative 2^-18 (lg2.approx absolute 2^-22 times |lg2 u| <= 24 over 3, plus ex2.approx
                                   relative 2^-22; the Guide's ulp bound for __powf grows with |y log2 x| the same way)
  __fdividef                       relative 2^-22 (Guide: 2 ulp for |y| in [2^-126, 2^126])
  __frsqrt_rn                      correctly rounded, 2^-24
The value tolerance carries the same uncertainties through pend, the sky or map slope and the throughput products, plus
float32 rounding of every sum and product."""
from __future__ import annotations

import numpy as np

import mirror_chain as mc
import test_sweep_oracle as so
from toypathtracer_b200 import CAMERA_DTYPE

U = 2.0 ** -24
PI32 = float(np.float32(3.1415926))                     # TPT_PI
TWO_PI32 = 2.0 * PI32                                   # 2.0f * TPT_PI (exact)
INV_PI32 = float(np.float32(1.0) / np.float32(3.1415926))   # (1.0f / TPT_PI), folded in float32
NORM_REL = mc.NORM_ERR
SQRT_REL = 2.0 ** -21
SINCOS_ABS = 2.0 ** -19
POW_REL = 2.0 ** -18
FDIV_REL = 2.0 ** -22
MAX_DEPTH = 10
LAMBERT, METAL, GLASS = 0, 1, 2
FLAGS = ("cap", "shadow_hit", "shadow_occluded", "fresnel_reflect", "fresnel_refract", "tir", "metal_absorbed",
         "sky_after_3", "rough_metal")


# ---- streams (tpt_fast.cu:36-44, tpt_integrator.cuh:130-140), uint32 throughout -------------------------------------
def fmix32(h):
    h = np.asarray(h, np.uint32).copy()
    h ^= h >> np.uint32(16); h *= np.uint32(0x85EBCA6B); h ^= h >> np.uint32(13); h *= np.uint32(0xC2B2AE35)
    h ^= h >> np.uint32(16)
    return h


def pixel_seed(index, frame):
    index = np.asarray(index, np.uint64).astype(np.uint32)
    f = fmix32(np.asarray(np.uint32(frame) + np.uint32(0x7F4A7C15), np.uint32))
    return fmix32(index * np.uint32(0x9E3779B9) + f) | np.uint32(1)


def xorshift32(x):
    x = np.asarray(x, np.uint32).copy()
    x ^= x << np.uint32(13); x ^= x >> np.uint32(17); x ^= x << np.uint32(15)
    return x


def u01(x):
    """RandomFloat01 of a raw draw: exact."""
    return (np.asarray(x, np.uint32) & np.uint32(0xFFFFFF)).astype(np.float64) * 2.0 ** -24


def ray_seeds(index, spp, sample, frame):
    """Caller rays and points (tpt_trace_rays / irradiance / samples): pixel_seed(input * spp + s, frame); a list call
    uses the input's index, not the entry's position."""
    return pixel_seed(np.asarray(index, np.uint64) * spp + sample, frame)


def draw_seeds(x, y, width, spp, sample, frame):
    """Draws and pixel lists: pixel_seed((y * width + x) * spp + s, frame)."""
    return pixel_seed((np.asarray(y, np.uint64) * width + x) * spp + sample, frame)


def mega_seed(x, y, width, frame):
    """Variant 0: one stream per pixel and frame, pixel_seed(y * width + x, frame), carried across the pixel's samples."""
    return pixel_seed(np.asarray(y, np.uint64) * width + x, frame)


class Stream:
    """Per-sample XorShift32 states; draw(mask) advances the masked lanes and returns their raw values."""

    def __init__(self, state):
        self.state = np.asarray(state, np.uint32).copy()
        self.count = np.zeros(len(self.state), np.int64)

    def draw(self, idx):
        x = xorshift32(self.state[idx])
        self.state[idx] = x
        self.count[idx] += 1
        return x


# ---- arithmetic: float64 (the oracle) or emulated float32 with perturbed MUFU results -------------------------------
class Exact:
    emu = False

    def r(self, x):
        return np.asarray(x, np.float64)

    def rel(self, x, b):
        return np.asarray(x, np.float64)

    def abs_(self, x, b):
        return np.asarray(x, np.float64)


class Emulated(Exact):
    """Every op rounded to float32 (an FMA's product of float32 values is exact in float64, so a * b + c rounds once, up
    to a double rounding the bounds do not depend on); a MUFU result is its exact value times (1 + delta) or plus delta,
    delta uniform within the bound assumed above."""
    emu = True

    def __init__(self, seed):
        self.g = np.random.default_rng(seed)

    def r(self, x):
        return np.asarray(x, np.float64).astype(np.float32).astype(np.float64)

    def rel(self, x, b):
        return self.r(x * (1.0 + self.g.uniform(-b, b, np.shape(x))))

    def abs_(self, x, b):
        return self.r(x + self.g.uniform(-b, b, np.shape(x)))


def _dot(A, a, b):
    return A.r(A.r(A.r(a[..., 0] * b[..., 0]) + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2])


def _norm(A, v):
    """M<false>::normalize: v * rsqrt(dot(v, v))."""
    return A.r(v * A.rel(1.0 / np.sqrt(_dot(A, v, v)), NORM_REL)[..., None])


def _sqrt(A, x):
    return A.rel(np.sqrt(np.maximum(x, 0.0)), SQRT_REL)


def _sincos(A, a):
    return A.abs_(np.sin(a), SINCOS_ABS), A.abs_(np.cos(a), SINCOS_ABS)


def unit_vector(A, x1, x2):
    """RandomUnitVectorFromDraws<false>: z from the first draw, the angle from the second."""
    z = A.r(u01(x1) * 2.0 - 1.0)
    a = A.r(u01(x2) * TWO_PI32)
    r = _sqrt(A, A.r(1.0 - A.r(z * z)))
    s, c = _sincos(A, a)
    return np.stack([A.r(r * c), A.r(r * s), z], -1)


def in_unit_sphere(A, x1, x2, x3):
    """fast_in_unit_sphere: z, the angle, then the radius u^(1/3)."""
    z = A.r(1.0 - A.r(2.0 * u01(x1)))
    s, c = _sincos(A, A.r(TWO_PI32 * u01(x2)))
    rad = A.rel(u01(x3) ** (1.0 / 3.0), POW_REL)
    r = A.r(_sqrt(A, A.r(1.0 - A.r(z * z))) * rad)
    return np.stack([A.r(r * c), A.r(r * s), A.r(z * rad)], -1)


def in_unit_disk(A, x1, x2):
    r = _sqrt(A, u01(x1))
    s, c = _sincos(A, A.r(TWO_PI32 * u01(x2)))
    return A.r(r * c), A.r(r * s)


# ---- scenes --------------------------------------------------------------------------------------------------------
def mixed_corridor(count: int, layout: str, n_lights: int = 4, seed: int = 0):
    """mirror_chain.corridor's floor and ceiling (Lambert, radius 100, 3 apart) with `count - 2` small spheres between
    them: Lambert, rough metal (roughness 0.1 - 1) and glass (ri 1.2 - 2) in equal shares, and `n_lights` of the small
    Lambert ones emissive (the lights; every light is small, so other spheres, glass included, occlude it). No two
    spheres overlap. compact: |s| <= 8 (the expanded-form gate passes); spread: over x, z in [-40, 40] with one sphere
    at |s| > 20 (it fails). Returns (spheres, materials, light ids)."""
    assert count >= 3
    sph, mats, _ = mc.corridor(count, layout, seed)
    rng = np.random.default_rng(seed * 104729 + count * 2 + (layout == "spread"))
    c = sph["center"].astype(np.float64)
    r = sph["radius"].astype(np.float64).copy()
    k = count - 2
    # shrink small spheres until none overlaps another or the floor / ceiling (mc.corridor keeps |y| <= 1.45 - r)
    for _ in range(40):
        dd = np.linalg.norm(c[2:, None] - c[None, 2:], axis=2) + np.eye(k) * 1e9
        over = dd < (r[2:, None] + r[None, 2:]) * 1.05
        if not over.any():
            break
        r[2:][over.any(1)] *= 0.8
    keep = np.linalg.norm(c[2:, None] - c[None, 2:], axis=2) + np.eye(k) * 1e9 >= (r[2:, None] + r[None, 2:]) * 1.05
    assert keep.all(), "mixed_corridor: overlapping spheres"
    sph["radius"][2:] = r[2:]
    sph["invRadius"] = (np.float32(1) / sph["radius"]).astype(np.float32)
    typ = np.zeros(count, np.int32)
    typ[2:] = rng.permutation(np.arange(k) % 3)
    mats["type"] = typ
    mats["albedo"] = rng.integers(16, 60, (count, 3)) / 64.0
    mats["albedo"][:2] = rng.integers(40, 56, (2, 3)) / 64.0
    mats["emissive"] = 0.0
    mats["roughness"] = np.where(typ == METAL, rng.integers(1, 11, count) / 10.0, 0.0)
    mats["ri"] = np.where(typ == GLASS, rng.integers(12, 21, count) / 10.0, 0.0)
    lamb = np.nonzero(typ[2:] == LAMBERT)[0] + 2
    # lights: the small Lambert spheres nearest the camera's corridor section first, so that shadow rays cross the scene
    order = lamb[np.argsort(np.linalg.norm(c[lamb][:, [0, 2]] - mc.CAMERA_O[[0, 2]], axis=1))]
    em = np.sort(order[:n_lights]).astype(np.int32)
    mats["emissive"][em] = rng.integers(8, 41, (len(em), 3)) / 8.0
    return sph, mats, em


def candidate_rays(sph, n, seed):
    """Rays from around the camera position, aimed into the corridor (a third of them at a random small sphere, the rest
    with a direction of random elevation)."""
    rng = np.random.default_rng(seed)
    raw = np.asarray(sph).view(np.float32).reshape(-1, 5).astype(np.float64)
    o = mc.CAMERA_O + rng.normal(size=(n, 3)) * np.array([0.6, 0.4, 0.6])
    o[:, 1] = np.clip(o[:, 1], -1.2, 1.2)
    d = rng.normal(size=(n, 3))
    d[:, 1] *= 0.6
    aim = rng.random(n) < 0.35
    if len(raw) > 2:
        tgt = raw[2 + rng.integers(0, len(raw) - 2, int(aim.sum())), :3]
        d[aim] = tgt - o[aim] + rng.normal(size=(int(aim.sum()), 3)) * 0.1
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return np.concatenate([o, d], 1).astype(np.float32)


def inside_glass_rays(sph, mats, n, seed):
    """Rays that start inside the glass spheres (a ray that entered a sphere by refraction always leaves it again, so
    total internal reflection needs an origin inside): origins within half the radius of the centre, random directions."""
    rng = np.random.default_rng(seed)
    raw = np.asarray(sph).view(np.float32).reshape(-1, 5).astype(np.float64)
    glass = np.nonzero(mats["type"] == GLASS)[0]
    if not len(glass):
        return np.zeros((0, 6), np.float32)
    pick = glass[rng.integers(0, len(glass), n)]
    off = rng.normal(size=(n, 3)); off /= np.linalg.norm(off, axis=1, keepdims=True)
    o = raw[pick, :3] + off * raw[pick, 3:4] * rng.uniform(0.3, 0.9, (n, 1))
    d = rng.normal(size=(n, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
    return np.concatenate([o, d], 1).astype(np.float32)


def surface_points(sph, mats, em, n, seed, with_ids=True):
    """Points on the Lambert spheres (float32 {p, n}, outward normals) and the id of the sphere each lies on. Without
    ids, points on emissive spheres are left out (tpt_trace_irradiance: such a point must pass its sphere's id)."""
    rng = np.random.default_rng(seed)
    raw = np.asarray(sph).view(np.float32).reshape(-1, 5).astype(np.float64)
    ok = mats["type"] == LAMBERT
    if not with_ids:
        ok[em] = False
    cand = np.nonzero(ok)[0]
    pick = cand[rng.integers(0, len(cand), n)]
    nrm = rng.normal(size=(n, 3)); nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    big = raw[pick, 3] > 50
    xz = rng.uniform(-4, 4, (int(big.sum()), 2))
    cb, rb = raw[pick[big], :3], raw[pick[big], 3]
    sgn = np.where(cb[:, 1] < 0, 1.0, -1.0)
    nrm[big] = np.stack([xz[:, 0] - cb[:, 0], cb[:, 1] * 0 + sgn * np.sqrt(rb ** 2 - ((xz - cb[:, [0, 2]]) ** 2).sum(1)),
                         xz[:, 1] - cb[:, 2]], 1) / rb[:, None]
    p = raw[pick, :3] + nrm * raw[pick, 3:4]
    return np.concatenate([p, nrm], 1).astype(np.float32), pick.astype(np.int32)


def lens_camera(lens_radius=0.05):
    """A camera at mirror_chain.CAMERA_O looking down -z into the corridor, 60 degrees wide, focused 3 ahead."""
    cam = np.zeros(1, CAMERA_DTYPE)
    o = np.array(mc.CAMERA_O)
    focus, half = 3.0, np.tan(np.radians(30))
    cam["origin"] = o
    cam["lowerLeftCorner"] = o + focus * np.array([-half * 1.5, -half, -1.0])
    cam["horizontal"] = (2 * half * 1.5 * focus, 0, 0)
    cam["vertical"] = (0, 2 * half * focus, 0)
    cam["uu"] = (1, 0, 0); cam["vv"] = (0, 1, 0); cam["ww"] = (0, 0, 1)
    cam["lensRadius"] = lens_radius
    return cam


class Scene:
    """What the replay needs of a scene as set_scene stages it. mitsuba: metal roughness 0 and the constant sky;
    env: a lat-long map [h, w, 3] that replaces the sky."""

    def __init__(self, sph, mats, em, mitsuba=False, env=None, ls=True):
        self.sph, self.count = sph, len(sph)
        self.expanded = so.gate_passes(sph)
        centres, r2 = so.scene_arrays(sph)
        self.C, self.R2 = centres.astype(np.float64), r2.astype(np.float64)
        self.inv = sph["invRadius"].astype(np.float64)
        self.typ = mats["type"].astype(int)
        self.alb = mats["albedo"].astype(np.float64)
        self.emis = mats["emissive"].astype(np.float64)
        self.rough = np.where((self.typ == METAL) & bool(mitsuba), 0.0, mats["roughness"].astype(np.float64))
        self.ri = mats["ri"].astype(np.float64)
        self.mitsuba, self.env, self.ls = bool(mitsuba), env, bool(ls)
        self.em = np.asarray(em, np.int64) if ls else np.zeros(0, np.int64)   # light sampling off: no lights
        self.Lc = self.C[self.em] if len(self.em) else np.zeros((0, 3))
        self.Lr = sph["radius"].astype(np.float64)[self.em]
        self.LE = self.emis[self.em]

    def sky(self, d, ed):
        """The terminal value in unit directions d and how far the kernel's can be, its direction being within ed."""
        if self.env is not None:
            from test_gpu_environment import env_lookup, lookup_tolerance
            return env_lookup(self.env, d), lookup_tolerance(self.env, d, eps=np.maximum(ed, 4e-6))
        return mc.sky(d, self.mitsuba), (0.0 if self.mitsuba else mc.SKY_SLOPE) * ed + 2 * U


# ---- starts --------------------------------------------------------------------------------------------------------
def start_rays(rays):
    """Caller rays: the kernel normalises the direction on load (DIR_ERR)."""
    d = rays[:, 3:].astype(np.float64)
    n = len(rays)
    return dict(o=rays[:, :3].astype(np.float64), d=d / np.linalg.norm(d, axis=1, keepdims=True),
                eo=np.zeros(n), ed=np.full(n, mc.DIR_ERR))


def camera_rays(A, cam, w, h, x, y, stream, idx):
    """fast_camera_ray from the sample's stream: jitter u, v (2 draws), then the lens (2 draws)."""
    c = {k: cam[k][0].astype(np.float64) for k in cam.dtype.names}
    ju, jv = u01(stream.draw(idx)), u01(stream.draw(idx))
    iw, ih = float(np.float32(1) / np.float32(w)), float(np.float32(1) / np.float32(h))
    u = A.r(A.r(x + ju) * iw)
    v = A.r(A.r(y + jv) * ih)
    rx, ry = in_unit_disk(A, stream.draw(idx), stream.draw(idx))
    lr = float(c["lensRadius"])
    rx, ry = A.r(lr * rx), A.r(lr * ry)
    off = A.r(A.r(c["uu"] * rx[:, None]) + A.r(c["vv"] * ry[:, None]))
    o = A.r(c["origin"] + off)
    dv = A.r(A.r(A.r(A.r(c["lowerLeftCorner"] + A.r(u[:, None] * c["horizontal"])) + A.r(v[:, None] * c["vertical"]))
                 - c["origin"]) - off)
    mag = (np.abs(c["lowerLeftCorner"]) + np.abs(c["horizontal"]) + np.abs(c["vertical"]) + 2 * np.abs(c["origin"])).sum()
    eo = lr * (2 * SINCOS_ABS + 2 * SQRT_REL) + 8 * U * (np.abs(c["origin"]).sum() + lr)
    dl = np.linalg.norm(dv, axis=1)
    ed = 1.01 * (eo + 12 * U * (mag + lr)) / dl + NORM_REL
    return o, (_norm(A, dv) if A.emu else dv / dl[:, None]), np.full(len(x), eo), ed


# ---- the replay ----------------------------------------------------------------------------------------------------
def replay(scene: Scene, state, rays=None, points=None, point_ids=None, point_self=None, camera=None, A=None,
           max_steps=100000):
    """Replay one sample per entry. Start from caller `rays` (float32 [n, 6]), surface `points` (float32 [n, 6]; ids
    `point_ids` as passed to the kernel or None, and `point_self`, the sphere each point lies on) or `camera` = (cam,
    width, height, x, y) (camera rays drawn from the stream). `state`: the streams' seeds (uint32 [n]). A: Exact() (the
    oracle, default) or Emulated(seed). Returns a dict of arrays (see the module docstring); `stream` holds the states
    after the sample (variant 0 carries them to the pixel's next sample)."""
    A = A or Exact()
    st = Stream(state)
    n = len(st.state)
    sc = scene
    S, R2 = sc.C[None], sc.R2[None]
    nL = len(sc.em)
    all_ = np.arange(n)
    if rays is not None:
        s0 = start_rays(rays)
        o, d, eo, ed = s0["o"], s0["d"], s0["eo"], s0["ed"]
        if A.emu:
            d = _norm(A, rays[:, 3:].astype(np.float64))
    elif camera is not None:
        cam, w, h, x, y = camera
        o, d, eo, ed = camera_rays(A, cam, w, h, np.asarray(x, np.float64), np.asarray(y, np.float64), st, all_)
    else:
        o = points[:, :3].astype(np.float64)
        dn_ = points[:, 3:].astype(np.float64)
        d = _norm(A, dn_) if A.emu else dn_ / np.linalg.norm(dn_, axis=1, keepdims=True)
        eo, ed = np.zeros(n), np.full(n, mc.DIR_ERR)
    o, d = o.copy(), d.copy()
    self_id, eo_self = np.full(n, -1), np.zeros(n)
    thr, col = np.ones((n, 3)), np.zeros((n, 3))
    nextd, ednext, thrAlb, nl, enl = np.zeros((n, 3)), np.zeros(n), np.ones((n, 3)), np.zeros((n, 3)), np.zeros(n)
    mid, kind, depth = np.full(n, -1), np.zeros(n, int), np.zeros(n, int)
    pend, epend, dl_, edl_ = np.zeros(n), np.zeros(n), np.zeros(n), np.zeros(n)
    doE = np.ones(n, bool)
    active = np.ones(n, bool)
    well = np.ones(n, bool)
    tol, mag = np.zeros(n), np.zeros(n)
    nrays, nvert = np.zeros(n, int), np.zeros(n, int)
    flags = {k: np.zeros(n, bool) for k in FLAGS}
    trail = []

    def add(idx, v, e):
        col[idx] += v
        tol[idx] += e
        mag[idx] += np.abs(v).max(1)

    def lambert_next(idx, light_from):
        """The next light from light_from on (skipping the vertex's own sphere), its cone and shadow ray; or the bounce."""
        j = light_from.copy()
        if nL:
            skip = (j < nL) & (sc.em[np.minimum(j, nL - 1)] == mid[idx])
            j = j + skip
        has = j < nL
        li, jj = idx[has], j[has]
        if len(li):
            cone(li, jj)
        bi = idx[~has]
        if len(bi):
            d[bi], ed[bi], thr[bi], kind[bi] = nextd[bi], ednext[bi], thrAlb[bi], 0
            doE[bi] = not sc.ls
            depth[bi] += 1

    def cone(li, jj):
        """sample_light_cone from o[li] towards light jj: 2 draws (cosA, then phi)."""
        oo = o[li]
        pc = A.r(sc.Lc[jj] - oo)
        d2 = _dot(A, pc, pc)
        inv = A.r(1.0 / np.sqrt(d2))                       # __frsqrt_rn
        sw = A.r(pc * inv[:, None])
        sgn = np.where(np.signbit(sw[:, 2]), -1.0, 1.0)
        oa = A.rel(-1.0 / (sgn + sw[:, 2]), FDIV_REL)
        ob = A.r(A.r(sw[:, 0] * sw[:, 1]) * oa)
        su = np.stack([A.r(1.0 + A.r(A.r(sgn * sw[:, 0] * sw[:, 0]) * oa)), A.r(sgn * ob), -sgn * sw[:, 0]], 1)
        sv = np.stack([ob, A.r(sgn + A.r(A.r(sw[:, 1] * sw[:, 1]) * oa)), -sw[:, 1]], 1)
        R = sc.Lr[jj]
        x = A.r(1.0 - A.r(A.r(A.r(R * R) * inv) * inv))
        cam_ = _sqrt(A, x)
        e1, e2 = u01(st.draw(li)), u01(st.draw(li))
        cosA = A.r(A.r(1.0 - e1) + A.r(e1 * cam_))
        sinA = _sqrt(A, A.r(1.0 - A.r(cosA * cosA)))
        sp, cp = _sincos(A, A.r(TWO_PI32 * e2))
        l = A.r(A.r(su * A.r(cp * sinA)[:, None] + sv * A.r(sp * sinA)[:, None]) + sw * cosA[:, None])
        omega = A.r(TWO_PI32 * A.r(1.0 - cam_))
        dl = _dot(A, l, nl[li])
        m = np.maximum(dl, 0.0)
        pend[li] = A.r(A.r(m * omega) * INV_PI32)
        if not A.emu:
            dist = np.sqrt(d2)
            esw = 1.1 * eo[li] / dist + 4 * U
            well[li] &= np.abs(sw[:, 2]) > esw + 1e-6              # the basis' sign branch
            ebasis = 8 * esw + 4 * FDIV_REL + 16 * U
            q = R * R / d2
            ex = q * 2.2 * (eo[li] / dist + 2 * U) + 3 * U
            ecm = ex / (2 * np.maximum(cam_, 1e-30)) + SQRT_REL * cam_ + U
            ecA = e1 * ecm + 3 * U
            es2 = 2 * ecA + 2 * U
            with np.errstate(divide="ignore"):
                esA = np.minimum(np.where(sinA > 0, es2 / (2 * sinA), np.inf), np.sqrt(es2)) + SQRT_REL * sinA + U
            el = 1.5 * (ebasis * sinA + esA + sinA * (SINCOS_ABS + 2 * U * TWO_PI32)) + esw * cosA + ecA + 8 * U
            edl = el + enl[li] + 4 * U
            eom = TWO_PI32 * ecm + 2 * U * omega
            epend[li] = 1.01 * (edl * omega + m * eom) * INV_PI32 + 4 * U * pend[li]
            dl_[li], edl_[li] = dl, edl
            ed[li] = el
        d[li] = l
        kind[li] = jj + 1

    step = 0
    if points is not None:
        # begin_vertex: a white Lambert vertex at p facing n, the bounce drawn first, then the lights
        idx = all_
        nl[:] = d
        enl[:] = ed
        u = unit_vector(A, st.draw(idx), st.draw(idx))
        v = A.r(d + u)
        lv = np.linalg.norm(v, axis=1)
        nextd[:] = _norm(A, v) if A.emu else v / lv[:, None]
        ednext[:] = 1.01 * (mc.DIR_ERR + 2.0 ** -18) / lv + NORM_REL
        if not A.emu:
            up = (nextd * nl).sum(1)
            well &= up > ednext + mc.DIR_ERR + 1e-6
        thrAlb[:] = 1.0
        mid[:] = -1 if point_ids is None else point_ids
        self_id[:] = point_self
        raw = np.asarray(sc.sph).view(np.float32).reshape(-1, 5).astype(np.float64)
        off = np.abs(np.linalg.norm(o - raw[point_self, :3], axis=1) - raw[point_self, 3])
        eo_self[:] = off + 4 * U * np.abs(o).sum(1)
        lambert_next(idx, np.zeros(n, int))

    while active.any():
        step += 1
        assert step < max_steps
        idx = np.nonzero(active)[0]
        if A.emu:
            from test_mirror_chain_oracle import _sweep
            form = "expanded" if (sc.expanded and A.g.random() < 0.5) else "reference"
            K = (sc.C * sc.C).sum(1) - sc.R2
            hid, ht = _sweep(o[idx], d[idx], sc.C, sc.R2, A.r(K), form, A.g)
            h = dict(id=hid, t=ht, well=np.ones(len(idx), bool), dtr=np.zeros(len(idx)))
        else:
            h = mc._nearest(o[idx], d[idx], eo[idx], ed[idx], S, R2, sc.expanded, sc.count, self_id[idx], eo_self[idx])
        nrays[idx] += 1
        tr = np.full(n, -3)
        tr[idx] = h["id"]
        trail.append(tr)
        hid = h["id"]
        shadow = kind[idx] > 0
        # ---- shadow rays: credited when they reach their own light
        si = idx[shadow]
        if len(si):
            j = kind[si] - 1
            hit_own = hid[shadow] == sc.em[j]
            contrib = thrAlb[si] * sc.LE[j] * pend[si][:, None]
            if A.emu:
                add(si[hit_own], contrib[hit_own], 0.0)
            else:
                sure = dl_[si] > edl_[si]
                amb = ~sure & (dl_[si] >= -edl_[si])
                well[si] &= h["well"][shadow] | ~sure
                trail[-1][si[~sure]] = -4                 # this shadow ray's hit does not matter
                cred = sure & hit_own
                add(si[cred], contrib[cred], (np.abs(thrAlb[si] * sc.LE[j]).max(1) * epend[si])[cred])
                # within its error of zero the weight is below (dl + edl) omega / pi whether or not the ray hits
                tol[si[amb]] += (np.abs(thrAlb[si] * sc.LE[j]).max(1) * 2.02 * edl_[si] * A.r(
                    TWO_PI32 * (1 + 1e-9)) * INV_PI32)[amb]
                flags["shadow_hit"][si[cred]] = True
                flags["shadow_occluded"][si[sure & ~hit_own]] = True
            lambert_next(si, j + 1)
        # ---- path rays
        pi_, ph = idx[~shadow], {k: v[~shadow] for k, v in h.items()}
        if not A.emu:
            well[pi_] &= ph["well"]
        miss = ph["id"] < 0
        mi = pi_[miss]
        if len(mi):
            sv, es = sc.sky(d[mi], ed[mi])
            add(mi, thr[mi] * sv, np.abs(thr[mi]).max(1) * es)
            flags["sky_after_3"][mi[nvert[mi] >= 3]] = True
            active[mi] = False
        hi, hid = pi_[~miss], ph["id"][~miss]
        if not len(hi):
            continue
        nvert[hi] += 1
        t = ph["t"][~miss]
        oo, dd = o[hi], d[hi]
        pos = A.r(oo + A.r(dd * t[:, None]))
        nrm = A.r(A.r(pos - sc.C[hid]) * sc.inv[hid][:, None])
        nn = np.linalg.norm(nrm, axis=1)
        dn = _dot(A, dd, nrm)
        if not A.emu:
            dtr = ph["dtr"][~miss]
            cos = np.abs(dn) / nn
            # mirror_chain's hit-point error, plus the root's move when |d| is off 1 (the sweep takes |d| = 1; the
            # normalize's length error shifts nb by t |dd|, the root by t^2 |dd| / (r cos): _nearest's dt)
            epos = 1.1 * (eo[hi] + t * ed[hi]) / cos + dtr * (1 + ed[hi]) + 4 * U * (np.linalg.norm(oo, axis=1) + t) \
                + 1.1 * t * t * (NORM_REL + ed[hi] ** 2) * sc.inv[hid] / cos
            en = epos * sc.inv[hid] + 4 * U * nn
            well[hi] &= (cos > 0.02) & np.isfinite(epos)
            eself = dtr * (1 + ed[hi]) + 4 * U * (np.linalg.norm(oo, axis=1) + t) + epos * epos * sc.inv[hid] \
                + 1.1 * t * t * (NORM_REL + ed[hi] ** 2) * sc.inv[hid] / cos
        else:
            epos = en = eself = np.zeros(len(hi))
        typ = sc.typ[hid]
        E = sc.emis[hid]
        # the depth cap: the hit's emission ends the path
        cap = depth[hi] >= MAX_DEPTH
        ci = hi[cap]
        add(ci, thr[ci] * E[cap], 0.0)
        flags["cap"][ci] = True
        active[ci] = False

        def moved(sel, dnext, ednext_):
            """The path goes on from pos along dnext: the next ray, and the up-check (it leaves the surface, or enters it
            when refracted, by more than its error)."""
            k = hi[sel]
            if not A.emu:
                well[k] &= np.abs((dnext * nrm[sel]).sum(1)) > ednext_ * nn[sel] + en[sel] + 1e-6
            o[k], d[k], eo[k], ed[k] = pos[sel], dnext, epos[sel], ednext_
            self_id[k], eo_self[k] = hid[sel], eself[sel]
            depth[k] += 1

        # Lambert
        lam = ~cap & (typ == LAMBERT)
        if lam.any():
            k = hi[lam]
            with_e = doE[k] | (not sc.ls)
            add(k[with_e], (thr[k] * E[lam])[with_e], 0.0)
            u = unit_vector(A, st.draw(k), st.draw(k))
            v = A.r(nrm[lam] + u)
            lv = np.linalg.norm(v, axis=1)
            nd = _norm(A, v) if A.emu else v / lv[:, None]
            ednd = 1.01 * (en[lam] + 2.0 ** -18 + 8 * U) / lv + NORM_REL
            if not A.emu:
                well[k] &= (nd * nrm[lam]).sum(1) > ednd * nn[lam] + en[lam] + 1e-6
            if sc.ls:
                nextd[k], ednext[k] = nd, ednd
                thrAlb[k] = A.r(thr[k] * sc.alb[hid[lam]])
                facing = dn[lam] < 0
                nl[k] = np.where(facing[:, None], nrm[lam], -nrm[lam])
                enl[k] = en[lam]
                mid[k] = hid[lam]
                o[k], eo[k], self_id[k], eo_self[k] = pos[lam], epos[lam], hid[lam], eself[lam]
                lambert_next(k, np.zeros(len(k), int))
            else:
                thr[k] = A.r(thr[k] * sc.alb[hid[lam]])
                o[k], d[k], eo[k], ed[k] = pos[lam], nd, epos[lam], ednd
                self_id[k], eo_self[k] = hid[lam], eself[lam]
                depth[k] += 1
        # metal
        met = ~cap & (typ == METAL)
        if met.any():
            k = hi[met]
            nm, dm = nrm[met], dd[met]
            refl = A.r(dm - A.r(A.r(2.0 * dn[met])[:, None] * nm))
            rough = sc.rough[hid[met]]
            out = refl.copy()
            rr = rough != 0
            if rr.any():
                kr = k[rr]
                vec = in_unit_sphere(A, st.draw(kr), st.draw(kr), st.draw(kr))
                out[rr] = A.r(refl[rr] + A.r(rough[rr][:, None] * vec))
                flags["rough_metal"][kr] = True
            lo = np.linalg.norm(out, axis=1)
            outd = _norm(A, out) if A.emu else out / lo[:, None]
            up = _dot(A, outd, nm)
            ok = up > 0
            if not A.emu:
                nn_m, en_m = nn[met], en[met]
                er = ed[k] * np.maximum(1.0, np.abs(2 * nn_m * nn_m - 1)) + en_m * (2 * np.abs(dn[met]) + 2 * nn_m + 2 * en_m)
                er = er + 24 * U + rough * (2.0 ** -17 + 8 * U) + 4 * U * rough
                eout = 1.01 * er / lo + NORM_REL
                well[k] &= np.abs(up) > eout * nn_m + en_m + 1e-6
            else:
                eout = np.zeros(len(k))
            flags["metal_absorbed"][k[~ok]] = True
            add(k[~ok], (thr[k] * E[met])[~ok], 0.0)
            active[k[~ok]] = False
            go = ok & (doE[k] | (not sc.ls))
            add(k[go], (thr[k] * E[met])[go], 0.0)
            doE[k[ok]] = True
            thr[k[ok]] = A.r(thr[k[ok]] * sc.alb[hid[met][ok]])
            sel = np.zeros(len(hi), bool)
            sel[np.nonzero(met)[0][ok]] = True
            moved(sel, outd[ok], eout[ok])
        # glass
        gl = ~cap & (typ == GLASS)
        if gl.any():
            k = hi[gl]
            nm, dm, dng = nrm[gl], dd[gl], dn[gl]
            ri = sc.ri[hid[gl]]
            inside = dng > 0
            outw = np.where(inside[:, None], -nm, nm)
            nint = np.where(inside, ri, A.rel(1.0 / ri, FDIV_REL))
            cosine = np.where(inside, A.r(ri * dng), -dng)
            dt = _dot(A, dm, outw)
            disc = A.r(1.0 - A.r(A.r(nint * nint) * A.r(1.0 - A.r(dt * dt))))
            can = disc > 0
            sq = _sqrt(A, disc)
            refr = A.r(A.r(nint[:, None] * A.r(dm - A.r(outw * dt[:, None]))) - A.r(outw * sq[:, None]))
            r0 = A.rel((1.0 - ri) / (1.0 + ri), FDIV_REL)
            r0 = A.r(r0 * r0)
            x = A.r(1.0 - cosine)
            x2 = A.r(x * x)
            p5 = A.r(A.r(x2 * x2) * x)
            rp = np.where(can, A.r(r0 + A.r(A.r(1.0 - r0) * p5)), 1.0)
            uu = u01(st.draw(k))
            refl_ = uu < rp
            refl = A.r(dm - A.r(A.r(2.0 * dng)[:, None] * nm))
            vec = np.where(refl_[:, None], refl, refr)
            lv = np.linalg.norm(vec, axis=1)
            outd = _norm(A, vec) if A.emu else vec / np.maximum(lv, 1e-300)[:, None]
            if not A.emu:
                nn_g, en_g = nn[gl], en[gl]
                edt = ed[k] + en_g + 4 * U
                fd = np.where(inside, 0.0, 2 * FDIV_REL)
                edisc = (nint * nint) * (2 * np.abs(dt) * edt + fd * np.abs(1 - dt * dt)) + 6 * U
                ecos = np.where(inside, ri, 1.0) * edt + 2 * U
                erp = 5 * (1 - r0) * np.abs(x) ** 4 * ecos + 4 * r0 * (FDIV_REL + U) + 8 * U
                well[k] &= np.abs(dng) / nn_g > 1.1 * edt                  # inside / outside
                well[k] &= np.abs(disc) > edisc                             # refraction or total internal reflection
                well[k] &= ~can | (np.abs(uu - rp) > erp)                   # Fresnel choice
                er = ed[k] * np.maximum(1.0, np.abs(2 * nn_g * nn_g - 1)) + en_g * (2 * np.abs(dng) + 2 * nn_g + 2 * en_g) + 24 * U
                with np.errstate(divide="ignore", invalid="ignore"):
                    erf = nint * (ed[k] + 2 * en_g + 2 * edt) + en_g * sq + edisc / (2 * np.sqrt(np.maximum(disc, 1e-300))) \
                        + SQRT_REL * sq + 8 * U * (nint + 1)
                eout = 1.01 * np.where(refl_, er, erf) / lv + NORM_REL
            else:
                eout = np.zeros(len(k))
            flags["tir"][k[~can]] = True
            flags["fresnel_reflect"][k[can & refl_]] = True
            flags["fresnel_refract"][k[can & ~refl_]] = True
            go = doE[k] | (not sc.ls)
            add(k[go], (thr[k] * E[gl])[go], 0.0)
            doE[k] = True
            moved(gl, outd, eout)
    tol_v = tol + (4 * nrays + 12) * U * (mag + np.abs(col).max(1)) + 1e-9
    return dict(v=col, rays=nrays, well=well, tol=tol_v, flags=flags, draws=st.count, state=st.state,
                trail=np.stack(trail, 1) if trail else np.zeros((n, 0), int), nvert=nvert)


def describe(res, i):
    """One sample's path for a failure message: hit ids per traced ray (-1 sky), draws, flags."""
    ids = [int(x) for x in res["trail"][i] if x != -3]
    fl = [k for k in FLAGS if res["flags"][k][i]]
    return f"sample {i}: path {ids}, draws {int(res['draws'][i])}, flags {fl}, tol {res['tol'][i]:.3g}"


def flag_counts(res, sel=None):
    sel = res["well"] if sel is None else sel
    return {k: int((v & sel).sum()) for k, v in res["flags"].items()}
