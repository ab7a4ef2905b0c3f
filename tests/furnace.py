"""Scenes whose rendered answer is known without rendering them, and that answer in float64.

A — deterministic furnace: one receiver sphere (radius 0.25 at the origin, Lambert or Metal) under the constant sky of
    DO_MITSUBA_COMPARE (which also forces Metal roughness to 0), seen through a narrow pinhole camera, so that every
    pixel footprint lies on the receiver with incidence cos >= 0.8. Optionally K tiny lights (r = 0.01) are buried
    inside it, within 0.15 of its centre. The receiver is convex, so every bounce or mirror ray leaves it and sees the
    sky, and every shadow ray toward a buried light points into the surface (sw.n <= -0.25 from any surface point,
    cone half-angle <= 6 deg) and contributes exactly 0. Every sample is therefore exactly v = albedo * sky (float32),
    a sample traces exactly 2 + K rays (Lambert with light sampling) or 2 (Metal, or light sampling off), and a pixel
    after a draw is prev * W + v * (1 - W), W the product of the drawn frames' lerp factors.
B1 — light sampling: a Lambert receiver under the constant sky with outside lights (albedo 0, emission Le_i) whose cones
    are fully above every visible point's horizon and do not overlap. With or without light sampling the pixel's
    expectation is E = rho * (sky + sum_i (Le_i - sky) * Phi_i), Phi_i = (1/pi) * integral over cone_i of n.w dw
    = cos(beta_i) * sin^2(alpha_i).
B2 — cosine lobe: a Lambert receiver under the gradient sky, no lights. The sky is affine in d_y and the mean of the
    cosine lobe around n is (2/3) n, so E = rho * L_sky(d_y = (2/3) n_y).

Expectations are per pixel, integrated over the pixel footprint with Gauss-Legendre quadrature, from the same float32
scene and camera bytes the renderers get."""
from __future__ import annotations

import numpy as np

from toypathtracer_b200 import MATERIAL_DTYPE, SPHERE_DTYPE
from toypathtracer_b200.scenes import make_camera

_F = np.float32
RECEIVER_R = 0.25
MITSUBA_SKY = np.array([0.15, 0.21, 0.3], _F)        # Test.cpp:226-227
ALBEDO = (0.8, 0.6, 0.4)
LAMBERT, METAL, DIELECTRIC = 0, 1, 2


def furnace_camera(w: int, h: int, half_deg: float = 5.0) -> np.ndarray:
    """Pinhole camera at (0, 0.3, 1) looking at the receiver: the image's longer side spans 2 * half_deg degrees (the
    receiver's angular radius from there is 13.9 degrees, so up to half_deg = 9 every footprint stays on it)."""
    aspect = w / h
    half = np.tan(np.radians(half_deg)) / max(aspect, 1.0)
    return make_camera((0, 0.3, 1), (0, 0, 0), (0, 1, 0), 2 * np.degrees(np.arctan(half)), aspect, 0.0, 1.0)


def _scene(receiver_type, lights, roughness=0.0, ri=0.0):
    """lights: [(centre, radius, albedo, emission)]. Returns (spheres, materials, emissive ids)."""
    n = 1 + len(lights)
    sph = np.zeros(n, SPHERE_DTYPE)
    mats = np.zeros(n, MATERIAL_DTYPE)
    sph[0] = ((0, 0, 0), RECEIVER_R, 0)
    mats[0] = (receiver_type, ALBEDO if receiver_type != DIELECTRIC else (1, 1, 1), (0, 0, 0), roughness, ri)
    for i, (c, r, alb, e) in enumerate(lights, 1):
        sph[i] = (c, r, 0)
        mats[i] = (LAMBERT, alb, e, 0, 0)
    sph["invRadius"] = (_F(1) / sph["radius"]).astype(_F)
    em = np.arange(1, n, dtype=np.int32)
    return sph, mats, em


def furnace_scene(w: int, h: int, n_lights: int = 0, metal: bool = False, seed: int = 7):
    """Scene A: (spheres, materials, camera, emissive ids). The Metal receiver has roughness 0.5 on file; the constant
    sky's mode forces it to 0, which the deterministic answer depends on."""
    rng = np.random.default_rng(seed + n_lights)
    lights = []
    for _ in range(n_lights):
        d = rng.normal(size=3)
        c = d / np.linalg.norm(d) * 0.15 * rng.uniform(0.0, 1.0) ** (1 / 3)
        lights.append((tuple(c), 0.01, (0.5, 0.5, 0.5), tuple(rng.uniform(1.0, 20.0, 3))))
    sph, mats, em = _scene(METAL if metal else LAMBERT, lights, roughness=0.5 if metal else 0.0)
    return sph, mats, furnace_camera(w, h), em


def furnace_value(mats) -> np.ndarray:
    """The one value every sample of scene A returns: albedo * sky in float32."""
    return (mats["albedo"][0].astype(_F) * MITSUBA_SKY).astype(_F)


def lerp_factor(frame: int, flags: int) -> np.float32:
    """Test.cpp:272-276 in float32."""
    lf = _F(frame) / _F(frame + 1)
    if flags & 1:
        lf = _F(lf * _F(0.9))
    if not flags & 2:
        lf = _F(0)
    return lf


def frame_weights(frame0: int, nframes: int, flags: int):
    """(W, w[nframes]): the weight of `prev` and of each drawn frame's sample mean, in float64."""
    lf = np.array([float(lerp_factor(frame0 + f, flags)) for f in range(nframes)])
    w = np.empty(nframes)
    suffix = 1.0
    for f in range(nframes - 1, -1, -1):
        w[f] = (1.0 - lf[f]) * suffix
        suffix *= lf[f]
    return suffix, w


def furnace_expect(prev_rgb, v, frame0, nframes, flags, spp):
    """(expected RGB, tolerance) of scene A after one draw over `prev_rgb`. The tolerance is a quarter of the smallest
    change one lost or duplicated sample makes (v * w_f / spp for the lightest frame that counts), so a single such
    sample in a single pixel fails, while float32 summation of <= 512 samples stays two orders of magnitude below it."""
    W, w = frame_weights(frame0, nframes, flags)
    v = np.asarray(v, np.float64)
    exp = np.asarray(prev_rgb, np.float64) * W + v * (1.0 - W)
    tol = v * w[w > 0].min() / spp / 4 + 2.0 ** -22 * np.abs(exp)
    return exp, tol


def furnace_rays_per_sample(mats, n_lights: int, light_sampling: bool) -> int:
    return 2 + n_lights if (light_sampling and int(mats["type"][0]) == LAMBERT) else 2


# ---- B: analytic expectations ---------------------------------------------------------------------------------------
def b1_scene(w: int, h: int, n_lights: int = 3):
    """Scene B1: Lambert receiver, 1-3 outside lights (albedo 0) 35 degrees off the camera axis."""
    cam_dir = np.array([0.0, 0.3, 1.0]) / np.linalg.norm([0.0, 0.3, 1.0])
    specs = [((1, 0, 0), 35, 1.25, 0.30, (2.0, 1.5, 1.0)),
             ((-1, 0, 0), 35, 1.10, 0.25, (0.6, 1.2, 2.4)),
             ((0, 1, 0), 40, 1.60, 0.22, (3.0, 3.0, 3.0))]
    lights = []
    for axis, deg, dist, r, e in specs[:n_lights]:
        a = np.asarray(axis, float)
        a = a - a.dot(cam_dir) * cam_dir
        a /= np.linalg.norm(a)
        d = np.cos(np.radians(deg)) * cam_dir + np.sin(np.radians(deg)) * a
        lights.append((tuple(d * dist), r, (0, 0, 0), e))
    sph, mats, em = _scene(LAMBERT, lights)
    return sph, mats, furnace_camera(w, h), em


def b2_scene(w: int, h: int):
    """Scene B2: Lambert receiver under the gradient sky, no lights."""
    sph, mats, em = _scene(LAMBERT, [])
    return sph, mats, furnace_camera(w, h), em


def gradient_sky(dy):
    """Test.cpp:228-231 in float64, affine in d_y."""
    t = 0.5 * (np.asarray(dy, np.float64)[..., None] + 1.0)
    return ((1.0 - t) * np.ones(3) + t * np.array([0.5, 0.7, 1.0])) * 0.3


def _gl(n):
    x, wt = np.polynomial.legendre.leggauss(n)
    return 0.5 * (x + 1.0), 0.5 * wt


def footprint_hits(cam, w, h, nq=4):
    """Receiver hits over each pixel's footprint: (p[h, w, Q, 3], weights[Q], d[h, w, Q, 3]) with Q = nq^2 Gauss-Legendre nodes
    over the jitter square, rays built in float64 from the float32 camera (Maths.h:437-442, zero aperture)."""
    c = {k: cam[k][0].astype(np.float64) for k in ("origin", "lowerLeftCorner", "horizontal", "vertical")}
    xs, ws = _gl(nq)
    jx, jy = np.meshgrid(xs, xs, indexing="ij")
    wq = np.outer(ws, ws).ravel()
    u = (np.arange(w)[None, :, None] + jx.ravel()[None, None, :]) / w
    v = (np.arange(h)[:, None, None] + jy.ravel()[None, None, :]) / h
    u, v = np.broadcast_arrays(u, v)
    d = c["lowerLeftCorner"] + u[..., None] * c["horizontal"] + v[..., None] * c["vertical"] - c["origin"]
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    o = c["origin"]
    b = (d * o).sum(-1)
    disc = b * b - (o.dot(o) - RECEIVER_R ** 2)
    assert (disc > 0).all(), "a pixel footprint leaves the receiver"
    t = -b - np.sqrt(disc)
    p = o + t[..., None] * d
    return p, wq, d


def light_phi(p, n, centre, radius):
    """Phi = (1/pi) * integral over the light's cone of max(0, n.w) dw = cos(beta) sin^2(alpha), asserting that the cone
    lies wholly above the horizon (beta + alpha < 90 deg) so that the closed form is exact."""
    pc = np.asarray(centre, np.float64) - p
    d2 = (pc * pc).sum(-1)
    cosb = (pc * n).sum(-1) / np.sqrt(d2)
    sin2a = radius * radius / d2
    assert (cosb > np.sqrt(sin2a)).all(), "a light cone crosses a visible point's horizon"
    return cosb * sin2a


def b1_expect(sph, mats, cam, w, h, nq=4):
    """Per-pixel expectation [h, w, 3] of scene B1 (light sampling on or off)."""
    p, wq, _ = footprint_hits(cam, w, h, nq)
    n = p / RECEIVER_R
    rho = mats["albedo"][0].astype(np.float64)
    sky = MITSUBA_SKY.astype(np.float64)
    e = np.broadcast_to(sky, p.shape).copy()
    ls = list(range(1, len(sph)))
    for i in ls:                                          # the cones must not overlap: no shadow ray is occluded
        for j in ls:
            if i < j:
                ai, aj = sph["center"][i] - p, sph["center"][j] - p
                cos_ij = (ai * aj).sum(-1) / np.linalg.norm(ai, axis=-1) / np.linalg.norm(aj, axis=-1)
                alpha_i = np.arcsin(sph["radius"][i] / np.linalg.norm(ai, axis=-1))
                alpha_j = np.arcsin(sph["radius"][j] / np.linalg.norm(aj, axis=-1))
                assert (np.arccos(np.clip(cos_ij, -1, 1)) > alpha_i + alpha_j).all()
        phi = light_phi(p, n, sph["center"][i].astype(np.float64), float(sph["radius"][i]))
        e += (mats["emissive"][i].astype(np.float64) - sky) * phi[..., None]
    return rho * (e * wq[:, None]).sum(-2)


def b2_expect(sph, mats, cam, w, h, nq=4):
    """Per-pixel expectation [h, w, 3] of scene B2."""
    p, wq, _ = footprint_hits(cam, w, h, nq)
    ny = p[..., 1] / RECEIVER_R
    rho = mats["albedo"][0].astype(np.float64)
    return rho * (gradient_sky(2.0 / 3.0 * ny) * wq[:, None]).sum(-2)


def bins_by(e, nbins=4, key=None):
    """Pixel bins [h, w] -> 0..nbins-1 by quantiles of `key` [h, w] (default: the expectation's luminance)."""
    lum = e @ np.array([0.25, 0.5, 0.25]) if key is None else key
    edges = np.quantile(lum, np.linspace(0, 1, nbins + 1)[1:-1])
    return np.searchsorted(edges, lum)


def check_bins(batches, e, bins, k_se=5.0, rel_floor=1e-4):
    """batches[B, h, w, 3]: independent per-pixel means. Per bin and channel: |mean - E| <= max(k_se * se, rel_floor * E)
    with se from the spread of the batch means. Returns [(bin, mean, E, se)] for the report; raises on failure."""
    out = []
    for b in range(bins.max() + 1):
        m = bins == b
        bm = batches[:, m, :].mean(axis=1)                 # [B, 3]
        mean = bm.mean(axis=0)
        se = bm.std(axis=0, ddof=1) / np.sqrt(len(bm))
        eb = e[m].mean(axis=0)
        out.append((b, mean, eb, se))
        assert (np.abs(mean - eb) <= np.maximum(k_se * se, rel_floor * eb)).all(), (b, mean, eb, se, (mean - eb) / se)
    return out


# ---- B3: rough metal -------------------------------------------------------------------------------------------------
B3_HALF_DEG = 8.5           # incidence cos from 1 down to ~0.45 over the image


def b3_scene(w: int, h: int, roughness: float):
    """Scene B3: Metal receiver (roughness 0.2 / 0.6 / 1.0) under the gradient sky, no lights."""
    sph, mats, em = _scene(METAL, [], roughness=roughness)
    return sph, mats, furnace_camera(w, h, B3_HALF_DEG), em


def sky_affine():
    """(a, b) per channel with the gradient sky L(d_y) = a + b * d_y (Test.cpp:228-231)."""
    c = np.array([0.5, 0.7, 1.0])
    return 0.15 * (1.0 + c), 0.15 * (c - 1.0)


def rough_lobe_moments(cos_g, r, n=32):
    """For a mirror direction refl at angle g from n (cos_g = refl.n) and d = normalize(refl + r u), u uniform in the unit
    ball: (P, M_n, M_t) = (P[d.n > 0], E[d.n 1{d.n > 0}], E[d.t 1{d.n > 0}]), t the unit tangent of refl. The indicator
    only bounds u's component along n (u_n > -cos_g / (r s) at radius s), so it becomes an integration limit and the
    remaining integrand is smooth: Gauss-Legendre in s (split where the limit reaches -1), in u_n, trapezoid in azimuth."""
    cos_g = np.asarray(cos_g, np.float64)[:, None, None, None]
    sin_g = np.sqrt(np.maximum(1.0 - cos_g ** 2, 0.0))
    x, wx = _gl(n)
    phi = (np.arange(n) + 0.5) * (2 * np.pi / n)
    out = np.zeros((3,) + cos_g.shape[:1])
    s0 = np.clip(cos_g / r, 0.0, 1.0)                        # below s0 the whole ball keeps d.n > 0
    for lo_s, hi_s in ((np.zeros_like(s0), s0), (s0, np.ones_like(s0))):
        s = lo_s + (hi_s - lo_s) * x[None, :, None, None]
        ws = (hi_s - lo_s) * wx[None, :, None, None] * 3.0 * s ** 2
        lo = np.maximum(-1.0, -cos_g / (r * np.maximum(s, 1e-300)))
        un = lo + (1.0 - lo) * x[None, None, :, None]
        wn = (1.0 - lo) * wx[None, None, :, None] * 0.5
        ut = np.sqrt(np.maximum(1.0 - un ** 2, 0.0)) * np.cos(phi)[None, None, None, :]
        ub = np.sqrt(np.maximum(1.0 - un ** 2, 0.0)) * np.sin(phi)[None, None, None, :]
        dn, dt, db = cos_g + r * s * un, sin_g + r * s * ut, r * s * ub
        inv = 1.0 / np.sqrt(dn * dn + dt * dt + db * db)
        wgt = ws * wn / n
        out[0] += (wgt * np.ones_like(inv)).sum(axis=(1, 2, 3))
        out[1] += (wgt * dn * inv).sum(axis=(1, 2, 3))
        out[2] += (wgt * dt * inv).sum(axis=(1, 2, 3))
    return out


def b3_expect(sph, mats, cam, w, h, nq=4, n=32):
    """Per-pixel expectation [h, w, 3] of scene B3 and the incidence cos [h, w] to bin by:
    E = rho * (a * P + b * (M_n n_y + M_t t_y)), the lobe moments tabulated over the incidence and splined."""
    from scipy.interpolate import CubicSpline
    p, wq, d = footprint_hits(cam, w, h, nq)
    nrm = p / RECEIVER_R
    cg = -(d * nrm).sum(-1)
    refl = d + 2.0 * cg[..., None] * nrm
    tang = refl - cg[..., None] * nrm
    tn = np.linalg.norm(tang, axis=-1, keepdims=True)
    tang = np.where(tn > 1e-12, tang / np.maximum(tn, 1e-300), 0.0)
    grid = np.linspace(cg.min() - 1e-3, 1.0, 129)
    mom = rough_lobe_moments(grid, float(mats["roughness"][0]), n)
    P, Mn, Mt = (CubicSpline(grid, m)(cg) for m in mom)
    a, b = sky_affine()
    dy = Mn * nrm[..., 1] + Mt * tang[..., 1]
    e = a * P[..., None] + b * dy[..., None]
    rho = mats["albedo"][0].astype(np.float64)
    return rho * (e * wq[:, None]).sum(-2), (cg * wq).sum(-1)


# ---- B4: glass -------------------------------------------------------------------------------------------------------
def b4_scene(w: int, h: int):
    """Scene B4: glass receiver (ri 1.5) under the gradient sky, no lights."""
    sph, mats, em = _scene(DIELECTRIC, [], ri=1.5)
    return sph, mats, furnace_camera(w, h, B3_HALF_DEG), em


def schlick(cosine, ri, saturate):
    """Maths.h:327-332 (the CPU path: 1 - cosine may be negative, and its 5th power then is) or the GPU shader's
    saturating form (ComputeShader.hlsl: 1 - cosine clamped to [0, 1])."""
    r0 = ((1.0 - ri) / (1.0 + ri)) ** 2
    x = 1.0 - cosine
    if saturate:
        x = np.clip(x, 0.0, 1.0)
    return r0 + (1.0 - r0) * x ** 5


def _refract(v, n, nint):
    """Maths.h refract() in float64 (the discriminant is positive for every refraction inside a sphere)."""
    dt = (v * n).sum(-1, keepdims=True)
    disc = 1.0 - nint * nint * (1.0 - dt * dt)
    assert (disc > 0).all()
    return nint * (v - n * dt) - n * np.sqrt(disc)


def b4_expect(sph, mats, cam, w, h, rule="cpu", nq=4):
    """Per-pixel expectation [h, w, 3] of scene B4 and the incidence cos [h, w]. A sample reflects at the first hit with
    probability R1 = schlick(cos_i) and escapes, or refracts; inside a sphere every hit has the same angle, so it then
    leaves after k internal reflections with probability R2^k (1 - R2), R2 = schlick(ri cos_t) (Test.cpp:151-186). The
    depth limit keeps k <= 8 on the CPU path (rays of depth 0..10, kMaxDepth = 10) and k <= 7 in the GPU shader (at
    most 10 rays), which also saturates Schlick: rule "cpu" or "gpu". Attenuation is 1; a truncated path returns 0."""
    ri = float(mats["ri"][0])
    saturate, kmax = (False, 8) if rule == "cpu" else (True, 7)
    p, wq, d = footprint_hits(cam, w, h, nq)
    nrm = p / RECEIVER_R
    cos_i = -(d * nrm).sum(-1)
    a, b = sky_affine()
    sky = lambda v: a + b * v[..., 1:2]
    r1 = schlick(cos_i, ri, saturate)[..., None]
    e = r1 * sky(d + 2.0 * cos_i[..., None] * nrm)
    v = _refract(d, nrm, 1.0 / ri)
    pos = p
    weight = 1.0 - r1
    for k in range(kmax + 1):
        pos = pos - 2.0 * (pos * v).sum(-1, keepdims=True) * v          # the next hit of the chord
        nq_ = pos / RECEIVER_R
        cos_t = (v * nq_).sum(-1, keepdims=True)
        r2 = schlick(ri * cos_t, ri, saturate)
        e = e + weight * (1.0 - r2) * sky(_refract(v, -nq_, ri))
        weight = weight * r2
        v = v - 2.0 * cos_t * nq_
    return (e * wq[:, None]).sum(-2), (cos_i * wq).sum(-1)


# ---- B5: defocus -----------------------------------------------------------------------------------------------------
def b5_scene(w: int, h: int):
    """Scene B5: the Lambert receiver under the constant sky seen whole (36 degree field of view) through a lens of radius
    0.03 focused at 0.6, in front of the receiver's silhouette (at ~1.0): its edge is blurred over ~8 pixels at 128x128.
    Every sample is the receiver's albedo * sky or the sky."""
    sph, mats, em = _scene(LAMBERT, [])
    return sph, mats, make_camera((0, 0.3, 1), (0, 0, 0), (0, 1, 0), 36.0, w / h, 0.06, 0.6), em


def _lens_coverage(cam, su, tv, nphi):
    """Fraction of the lens disk whose ray through the focus-plane point of screen coordinates (su, tv) hits the
    receiver (Maths.h:437-442). For a fixed lens azimuth the lens points form a segment and the rays through one focus
    point form a fan, so the hitting part of the segment is where a quadratic in the lens radius rho is <= 0: the
    uniform-disk measure 2 rho d rho integrates in closed form; the azimuth is integrated by the trapezoid rule."""
    c = {k: cam[k][0].astype(np.float64) for k in ("origin", "lowerLeftCorner", "horizontal", "vertical", "uu", "vv")}
    R = float(cam["lensRadius"][0])
    q = c["lowerLeftCorner"] + su[..., None] * c["horizontal"] + tv[..., None] * c["vertical"]
    A = c["origin"] - q
    D = -q                                                  # receiver centre (origin) - q
    phi = (np.arange(nphi) + 0.5) * (2 * np.pi / nphi)
    B = R * (np.cos(phi)[:, None] * c["uu"] + np.sin(phi)[:, None] * c["vv"])      # [nphi, 3]
    A, D = A[..., None, :], D[..., None, :]
    DA, DB = np.cross(D, A), np.cross(D, B)
    r2 = RECEIVER_R ** 2
    qa = (DB * DB).sum(-1) - r2 * (B * B).sum(-1)
    qb = 2.0 * ((DA * DB).sum(-1) - r2 * (A * B).sum(-1))
    qc = (DA * DA).sum(-1) - r2 * (A * A).sum(-1)
    disc = qb * qb - 4.0 * qa * qc
    sq = np.sqrt(np.maximum(disc, 0.0))
    with np.errstate(divide="ignore", invalid="ignore"):
        x1 = (-qb - np.sign(qa) * sq) / (2.0 * qa)
        x2 = (-qb + np.sign(qa) * sq) / (2.0 * qa)
    lo, hi = np.minimum(x1, x2), np.maximum(x1, x2)
    seg = lambda a_, b_: np.clip(b_, 0, 1) ** 2 - np.clip(a_, 0, 1) ** 2
    inside = np.where(qa > 0, seg(lo, hi), 1.0 - seg(lo, hi))      # qa < 0: the quadratic is <= 0 outside its roots
    full = np.where(qc <= 0, 1.0, 0.0)                              # no real roots: the sign of the quadratic at rho = 0
    cov = np.where(disc > 0, inside, full)
    return cov.mean(-1)


def b5_expect(sph, mats, cam, w, h, nq=6, nphi=256):
    """Per-pixel expectation [h, w, 3] of scene B5 and the coverage [h, w]: E = cov * albedo * sky + (1 - cov) * sky,
    cov the float64 integral of "the ray hits the receiver" over the pixel (Gauss-Legendre) x the lens disk. Pixels
    more than two pixels away from any partly covered pixel on a coarse pass are exactly 0 or 1."""
    xs, ws = _gl(nq)
    coarse = _lens_coverage(cam, (np.arange(w)[None, :] + 0.5 + 0 * np.arange(h)[:, None]) / w,
                            (np.arange(h)[:, None] + 0.5 + 0 * np.arange(w)[None, :]) / h, 64)
    part = (coarse > 0) & (coarse < 1)
    for _ in range(3):
        part = part | np.roll(part, 1, 0) | np.roll(part, -1, 0) | np.roll(part, 1, 1) | np.roll(part, -1, 1)
    cov = np.round(coarse)
    yy, xx = np.nonzero(part)
    acc = np.zeros(len(yy))
    for i, (jx, wx) in enumerate(zip(xs, ws)):
        for jy, wy in zip(xs, ws):
            acc += wx * wy * _lens_coverage(cam, (xx + jx) / w, (yy + jy) / h, nphi)
    cov[yy, xx] = acc
    v = (mats["albedo"][0].astype(np.float64) * MITSUBA_SKY).astype(np.float64)
    sky = MITSUBA_SKY.astype(np.float64)
    return cov[..., None] * v + (1.0 - cov[..., None]) * sky, cov


# ---- the B scenes as test cases --------------------------------------------------------------------------------------
B_SCENES = ("b1_ls", "b1_nols", "b2", "b3_r02", "b3_r06", "b3_r10", "b4", "b5")
_b_cache = {}


def b_case(name: str, rule: str = "cpu"):
    """(spheres, materials, camera, emissives, w, h, E[h, w, 3], bins[h, w], mitsuba_compare, light_sampling) of a B
    scene: 64x64 in four bins of 1024 pixels (B5: 128x128, binned by lens coverage: sky, partial < 0.5, partial >= 0.5,
    receiver; the partial bins hold ~1 300 pixels each). rule: "cpu" for the CPU path's estimator, "gpu" for the GPU
    shader's (only B4 depends on it)."""
    key = (name, rule if name == "b4" else "cpu")
    if key not in _b_cache:
        w = h = 128 if name == "b5" else 64
        if name.startswith("b1"):
            s, m, c, em = b1_scene(w, h)
            e = b1_expect(s, m, c, w, h); bins = bins_by(e)
        elif name == "b2":
            s, m, c, em = b2_scene(w, h)
            e = b2_expect(s, m, c, w, h); bins = bins_by(e)
        elif name.startswith("b3"):
            s, m, c, em = b3_scene(w, h, int(name[-2:]) / 10)
            e, inc = b3_expect(s, m, c, w, h); bins = bins_by(e, key=inc)
        elif name == "b4":
            s, m, c, em = b4_scene(w, h)
            e, inc = b4_expect(s, m, c, w, h, rule); bins = bins_by(e, key=inc)
        else:
            s, m, c, em = b5_scene(w, h)
            e, cov = b5_expect(s, m, c, w, h); bins = np.digitize(cov, [1e-12, 0.5, 1 - 1e-12])
        _b_cache[key] = (s, m, c, em, w, h, e, bins, name in ("b1_ls", "b1_nols", "b5"), name != "b1_nols")
    return _b_cache[key]
