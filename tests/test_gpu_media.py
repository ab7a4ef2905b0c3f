"""Homogeneous media inside glass spheres (tpt_set_media, Context.set_media) on the GPU.

1. Inert media are the identity, bit for bit and ray for ray, through every fast call with light sampling on and off,
   on the 46- and 4096-sphere scenes: media on non-glass spheres only equal "fast_kform" 0 without media; media whose
   ids lie past the scene run the default kernel with the default bits; a pure absorber on glass draws no random number
   and changes no path decision (same ray counts), and at spp 1 no output channel grows.
2. Beer-Lambert: a clear absorbing glass sphere under a constant map, rays from its centre and along its axis from
   outside, against the float64 sum over the axial reflect/refract chain (the reference's schlick with the inside-face
   cosine ri dot(d, n), and the depth cap).
3. White furnace: sigma_a = 0 with scattering: the mean is L (1 - p_cap), p_cap from the float64 model of the estimator.
4. Absorbing and scattering together against an independent numpy Monte-Carlo of the same estimator.
5. The 46-sphere scene with a tinted scattering medium in its glass sphere: light sampling on and off agree per
   first-hit sphere, also with "environment_sampling" and constant albedo textures.
6. Routing, refusals, lifetime, ordering, unchanged AOVs and the upload size."""
import numpy as np
import pytest
import torch

import furnace as F
from test_gpu_textures import TEX_KERNELS, _const_layers, _draw, _every_call
from toypathtracer_b200 import MATERIAL_DTYPE, MODE_EXACT, MODE_FAST, MODE_REFGPU, MODE_REFGPU_FAST, SPHERE_DTYPE, TptError, scenes

pytestmark = pytest.mark.gpu

MAX_DEPTH = 10           # TPT_MAX_DEPTH
GLASS46 = 7              # the 46-sphere scene's glass sphere


@pytest.fixture
def mctx(gpu_ctx):
    yield gpu_ctx
    gpu_ctx.set_media(None)
    gpu_ctx.set_textures(None)
    gpu_ctx.set_environment(None)
    for k, v in (("fast_variant", -1), ("fast_kform", 2), ("light_sampling", 1), ("environment_sampling", 0)):
        gpu_ctx.set_option(k, v)
    gpu_ctx.set_spp(4)


def _media(n, rows):
    m = np.zeros((n, 5), np.float32)
    for i, rec in rows.items():
        m[i] = rec
    return m


def _same(got, ref):
    for k in ref:
        (ga, gr), (ra, rr) = got[k], ref[k]
        assert gr == rr, (k, gr, rr)
        ga, ra = np.asarray(ga), np.asarray(ra)
        assert ga.shape == ra.shape and ga.tobytes() == ra.tobytes(), (k, int((ga.view(np.uint32) != ra.view(np.uint32)).sum()))


# ---- 1. inert media -------------------------------------------------------------------------------------------------
SCENES = {"46": (lambda: scenes.reference_scene(64, 36), 64, 36, (-1, 3, 9)),
          "4096": (lambda: scenes.stress_scene(48, 27), 48, 27, (3, 9))}


@pytest.mark.parametrize("ls", [1, 0])
@pytest.mark.parametrize("which", sorted(SCENES))
def test_media_on_non_glass_spheres_equal_reference_form_without_media(mctx, which, ls):
    make, w, h, variants = SCENES[which]
    s, m, c, em = make()
    mctx.set_option("light_sampling", ls)
    mctx.set_option("fast_kform", 0)
    mctx.set_scene(s, m, c, em)
    ref = _every_call(mctx, w, h, c, s, variants)
    media = np.zeros((len(s), 5), np.float32)
    other = m["type"] != F.DIELECTRIC
    media[other] = (0.7, 0.2, 0.1, 3.0, 0.5)
    mctx.set_media(media)
    got = _every_call(mctx, w, h, c, s, variants)
    _same(got, ref)


@pytest.mark.parametrize("ls", [1, 0])
@pytest.mark.parametrize("which", sorted(SCENES))
def test_media_past_the_scene_run_the_default_kernel(mctx, which, ls):
    make, w, h, variants = SCENES[which]
    s, m, c, em = make()
    mctx.set_option("light_sampling", ls)
    mctx.set_scene(s, m, c, em)
    ref = _every_call(mctx, w, h, c, s, (-1,))
    _draw(mctx, w, h)
    kern = mctx.last_kernels()
    media = np.zeros((len(s) + 4, 5), np.float32)
    media[len(s):] = (1.0, 1.0, 1.0, 5.0, 0.3)
    media[: len(s), 4] = 0.9                      # g alone is no medium
    mctx.set_media(media)
    assert mctx.last_scene_upload_bytes() == 0    # the blob is the plain scene's: nothing to upload
    got = _every_call(mctx, w, h, c, s, (-1,))
    _draw(mctx, w, h)
    assert mctx.last_kernels() == kern
    _same(got, ref)


def _spp1_calls(ctx, w, h, cam, sph):
    """Outputs (one sample each) and ray counts of a one-frame draw and every caller-buffer call."""
    ctx.set_spp(1)
    res = {"draw": _draw(ctx, w, h)}
    rays = scenes.camera_rays(cam, w, h, seed=5)
    res["rays"] = ctx.trace_rays(rays, spp=1)
    rng = np.random.default_rng(9)
    ids = rng.integers(0, len(sph), 512).astype(np.int32)
    nrm = rng.normal(size=(512, 3))
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    pts = np.concatenate([sph["center"][ids] + sph["radius"][ids][:, None] * nrm, nrm], 1).astype(np.float32)
    res["irr"] = ctx.trace_irradiance(pts, ids, spp=1)
    (s4, q4), r = ctx.draw_samples(0, w, h, spp=1)
    res["dsamples"] = (np.concatenate([s4.cpu().numpy(), q4.cpu().numpy()]), r)
    (s4, q4), r = ctx.trace_samples(rays, spp=1)
    res["tsamples"] = (np.concatenate([s4, q4]), r)
    return res


@pytest.mark.parametrize("ls", [1, 0])
@pytest.mark.parametrize("which", sorted(SCENES))
def test_pure_absorber_draws_nothing_and_only_darkens(mctx, which, ls):
    make, w, h, _v = SCENES[which]
    s, m, c, em = make()
    mctx.set_option("light_sampling", ls)
    mctx.set_option("fast_kform", 0)
    mctx.set_scene(s, m, c, em)
    ref = _spp1_calls(mctx, w, h, c, s)
    glass = np.nonzero(m["type"] == F.DIELECTRIC)[0]
    assert glass.size
    media = np.zeros((len(s), 5), np.float32)
    media[glass] = (0.9, 0.3, 2.5, 0.0, 0.0)
    mctx.set_media(media)
    got = _spp1_calls(mctx, w, h, c, s)
    darker = 0
    for k in ref:
        (ga, gr), (ra, rr) = got[k], ref[k]
        assert gr == rr, (k, gr, rr)
        ga, ra = np.asarray(ga), np.asarray(ra)
        assert (ga <= ra).all(), (k, int((ga > ra).sum()))
        darker += int((ga < ra).sum())
    assert darker > 0                                     # the absorber is there


# ---- float64 models of the estimator in one glass sphere under a constant map --------------------------------------
def schlick(cosine, ri):
    r0 = ((1.0 - ri) / (1.0 + ri)) ** 2
    return r0 + (1.0 - r0) * (1.0 - cosine) ** 5


def axial_expect(sigma_a, radius, ri, from_centre):
    """Mean radiance (per unit map radiance) of a ray through the centre of a clear absorbing glass sphere: from the
    centre every hit is on the inside face at normal incidence (cosine = ri); from outside along the axis the first hit
    reflects with schlick(1, ri). A hit at depth >= MAX_DEPTH ends the path with nothing (the sphere emits nothing)."""
    sa = np.asarray(sigma_a, np.float64)
    r_in = schlick(ri * 1.0, ri)
    total = np.zeros(3)
    if from_centre:
        for k in range(MAX_DEPTH):                        # k-th inside hit at depth k, after r + 2 r k in the medium
            total += r_in ** k * (1 - r_in) * np.exp(-sa * (radius + 2 * radius * k))
        return total
    r_out = schlick(1.0, ri)
    total += r_out                                        # reflected at the outside face, depth 0
    for k in range(MAX_DEPTH - 1):                        # k-th inside hit at depth 1 + k, after 2 r (k + 1)
        total += (1 - r_out) * r_in ** k * (1 - r_in) * np.exp(-sa * 2 * radius * (k + 1))
    return total


def hg_dirs(d, g, xi1, xi2):
    if abs(g) >= 1e-3:
        s = (1 - g * g) / (1 - g + 2 * g * xi1)
        cos_t = np.clip((1 + g * g - s * s) / (2 * g), -1, 1)
    else:
        cos_t = 1 - 2 * xi1
    sin_t = np.sqrt(np.maximum(1 - cos_t ** 2, 0))
    phi = 2 * np.pi * xi2
    sgn = np.where(d[:, 2] >= 0, 1.0, -1.0)
    a = -1.0 / (sgn + d[:, 2])
    b = d[:, 0] * d[:, 1] * a
    su = np.stack([1 + sgn * d[:, 0] ** 2 * a, sgn * b, -sgn * d[:, 0]], 1)
    sv = np.stack([b, sgn + d[:, 1] ** 2 * a, -d[:, 1]], 1)
    out = su * (sin_t * np.cos(phi))[:, None] + sv * (sin_t * np.sin(phi))[:, None] + d * cos_t[:, None]
    return out / np.linalg.norm(out, axis=1, keepdims=True)


def mc_model(n, sigma_a, sigma_s, g, radius, ri, seed):
    """float64 Monte-Carlo of the estimator for paths that start at the centre of a glass sphere (centre 0) under a
    constant unit map: per-path RGB values and whether the path ended at the depth cap."""
    rng = np.random.default_rng(seed)
    sa = np.asarray(sigma_a, np.float64)
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    o = np.zeros((n, 3))
    thr = np.ones((n, 3))
    depth = np.zeros(n, np.int64)
    val = np.zeros((n, 3))
    capped = np.zeros(n, bool)
    act = np.ones(n, bool)
    while act.any():
        i = np.nonzero(act)[0]
        oi, di = o[i], d[i]
        b = (oi * di).sum(1)
        c = (oi * oi).sum(1) - radius * radius
        t = -b + np.sqrt(np.maximum(b * b - c, 0))          # the inside face
        ts = -np.log(1 - rng.random(i.size)) / sigma_s if sigma_s > 0 else np.full(i.size, np.inf)
        sc = ts < t
        # scatter events
        j = i[sc]
        cap = depth[j] >= MAX_DEPTH
        capped[j[cap]] = True
        act[j[cap]] = False
        j = j[~cap]
        tsj = ts[sc][~cap]
        thr[j] *= np.exp(-sa[None, :] * tsj[:, None])
        o[j] += d[j] * tsj[:, None]
        d[j] = hg_dirs(d[j], g, rng.random(j.size), rng.random(j.size))
        depth[j] += 1
        # hits on the inside face
        k = i[~sc]
        tk = t[~sc]
        thr[k] *= np.exp(-sa[None, :] * tk[:, None])
        cap = depth[k] >= MAX_DEPTH
        capped[k[cap]] = True
        act[k[cap]] = False
        k, tk = k[~cap], tk[~cap]
        p = o[k] + d[k] * tk[:, None]
        nrm = p / radius
        dn = (d[k] * nrm).sum(1)                            # > 0: inside
        discr = 1 - ri * ri * (1 - dn * dn)
        refl_p = np.where(discr > 0, schlick(ri * dn, ri), 1.0)
        refl = rng.random(k.size) < refl_p
        out = k[~refl]
        val[out] = thr[out]
        act[out] = False
        r = k[refl]
        nr = nrm[refl]
        d[r] = d[r] - 2 * (d[r] * nr).sum(1)[:, None] * nr
        d[r] /= np.linalg.norm(d[r], axis=1, keepdims=True)
        o[r] = p[refl]
        depth[r] += 1
    return val, capped


def glass_scene(radius=1.0, ri=1.5):
    sph = np.zeros(1, SPHERE_DTYPE)
    mats = np.zeros(1, MATERIAL_DTYPE)
    sph[0] = ((0.0, 0.0, 0.0), radius, 1.0 / radius)
    mats[0] = (F.DIELECTRIC, (1, 1, 1), (0, 0, 0), 0.0, ri)
    return sph, mats, F.furnace_camera(8, 8), np.zeros(0, np.int32)


def _centre_rays(n, seed):
    d = np.random.default_rng(seed).normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return np.concatenate([np.zeros((n, 3)), d], 1).astype(np.float32)


def _per_sample_stats(ctx, rays, spp, frames):
    """Mean and standard error of the per-sample radiance over rays x spp x frames samples (trace_samples' sums)."""
    s = np.zeros(4)
    q = np.zeros(4)
    for f in range(frames):
        (s4, q4), _ = ctx.trace_samples(rays, spp=spp, frame=f)
        s += s4.astype(np.float64).sum(0)
        q += q4.astype(np.float64).sum(0)
    n = s[3]
    mean = s[:3] / n
    var = q[:3] / n - mean ** 2
    return mean, np.sqrt(np.maximum(var, 0) / n), n


L_ENV = np.float32([0.8, 1.3, 0.5])


@pytest.mark.parametrize("ls", [1, 0])
def test_beer_lambert_along_the_axis(mctx, ls):
    radius, ri = 1.0, 1.5
    sa = (0.15, 0.6, 1.8)
    mctx.set_option("light_sampling", ls)
    mctx.set_scene(*glass_scene(radius, ri))
    mctx.set_environment(np.broadcast_to(L_ENV, (4, 8, 3)).copy())
    mctx.set_media(np.float32([[*sa, 0.0, 0.0]]))
    n = 4096
    centre = _centre_rays(n, 3)
    axis = np.tile(np.float32([0, 0, 4.0, 0, 0, -1.0]), (n, 1))
    axis[: n // 2] = (4.0, 0, 0, -1.0, 0, 0)
    for rays, from_centre in ((centre, True), (axis, False)):
        want = L_ENV * axial_expect(sa, radius, ri, from_centre)
        mean, se, ns = _per_sample_stats(mctx, rays, 16, 1)
        assert ns >= 2 ** 16
        assert (np.abs(mean - want) <= 5 * se + 1e-6 * want).all(), (from_centre, mean, want, se)


@pytest.mark.parametrize("sigma_s", [0.5, 4.0])
@pytest.mark.parametrize("g", [-0.6, 0.0, 0.8])
def test_white_furnace_loses_only_the_depth_cap(mctx, sigma_s, g):
    radius, ri = 1.0, 1.5
    mctx.set_scene(*glass_scene(radius, ri))
    mctx.set_environment(np.broadcast_to(L_ENV, (4, 8, 3)).copy())
    mctx.set_media(np.float32([[0.0, 0.0, 0.0, sigma_s, g]]))
    val, capped = mc_model(200_000, (0, 0, 0), sigma_s, g, radius, ri, seed=int(sigma_s * 10 + g * 100) & 0xffff)
    p_cap = capped.mean()
    p_se = np.sqrt(p_cap * (1 - p_cap) / capped.size)
    assert np.array_equal(val[~capped], np.ones((int((~capped).sum()), 3)))   # sigma_a = 0: an escaping path carries L
    mean, se, _ = _per_sample_stats(mctx, _centre_rays(4096, 5), 16, 1)
    want = L_ENV * (1 - p_cap)
    tol = 5 * np.sqrt(se ** 2 + (L_ENV * p_se) ** 2)
    print(f"sigma_s {sigma_s} g {g}: p_cap {p_cap:.5f} +- {p_se:.5f}, kernel {mean / L_ENV}")
    assert (np.abs(mean - want) <= tol).all(), (sigma_s, g, p_cap, mean / L_ENV, se)
    if sigma_s == 4.0:
        assert p_cap > 0.1                                # the dense medium loses much of its energy to the cap


@pytest.mark.parametrize("ls", [1, 0])
def test_absorbing_and_scattering_match_the_numpy_model(mctx, ls):
    radius, ri = 1.0, 1.5
    sa, ss, g = (0.1, 0.35, 0.9), 1.5, 0.4
    mctx.set_option("light_sampling", ls)
    mctx.set_scene(*glass_scene(radius, ri))
    mctx.set_environment(np.broadcast_to(L_ENV, (4, 8, 3)).copy())
    mctx.set_media(np.float32([[*sa, ss, g]]))
    val, _ = mc_model(200_000, sa, ss, g, radius, ri, seed=11)
    want = L_ENV * val.mean(0)
    want_se = L_ENV * val.std(0) / np.sqrt(val.shape[0])
    mean, se, _ = _per_sample_stats(mctx, _centre_rays(4096, 7), 16, 1)
    assert (np.abs(mean - want) <= 5 * np.sqrt(se ** 2 + want_se ** 2)).all(), (mean, want, se, want_se)
    # the absorption is real: darker than the furnace with the same scattering
    assert (mean < 0.9 * L_ENV).all()


# ---- replay: single samples in float64 from their own streams ----------------------------------------------------------
REPLAY_SPHERES = [((0.0, 0.0, 0.0), 1.0, 1.5), ((2.3, 0.4, -0.3), 0.8, 1.3), ((-1.4, 1.7, 0.5), 0.6, 1.7)]
REPLAY_MEDIA = np.float32([[0.3, 0.1, 0.05, 1.2, 0.5],        # absorbing and scattering, forward
                           [0.8, 0.4, 0.2, 0.0, 0.0],         # absorbing only
                           [0.0, 0.0, 0.0, 2.5, -0.4]])       # scattering only, backward
TMIN = 0.001                                                  # TPT_MIN_T


def replay_scene():
    n = len(REPLAY_SPHERES)
    sph = np.zeros(n, SPHERE_DTYPE)
    mats = np.zeros(n, MATERIAL_DTYPE)
    for i, (c, r, ri) in enumerate(REPLAY_SPHERES):
        sph[i] = (c, r, 1.0 / r)
        mats[i] = (F.DIELECTRIC, (1, 1, 1), (0, 0, 0), 0.0, ri)
    sph["invRadius"] = (np.float32(1) / sph["radius"]).astype(np.float32)
    return sph, mats, F.furnace_camera(8, 8), np.zeros(0, np.int32)


def replay_one(ray, seed, sph):
    """float64 replay of one caller-ray sample through REPLAY_SPHERES with REPLAY_MEDIA under a constant unit map, fed
    the sample's own draws in the kernel's order: (value RGB, rays traced, well-conditioned, value tolerance). `err`
    bounds how far the kernel's float32 and MUFU path (__logf, __expf, __fdividef, __sincosf, rsqrt) can be from this one
    in position and direction; it grows at every interface and scatter event, and a decision whose margin is within a
    multiple of it makes the sample ill-conditioned (ties of t_s against t included)."""
    import sample_replay as sr
    st = sr.Stream(np.array([seed], np.uint32))
    draw = lambda: float(sr.u01(st.draw(np.array([0]))[0]))  # noqa: E731
    cen = sph["center"].astype(np.float64)
    rad = sph["radius"].astype(np.float64)
    o = ray[:3].astype(np.float64)
    d = ray[3:].astype(np.float64)
    d /= np.linalg.norm(d)
    thr, depth, rays, err, length = np.ones(3), 0, 0, 1e-6, 0.0
    ok = True
    k_margin = 16.0
    while True:
        rays += 1
        best, bid, ts_all = np.inf, -1, []
        for k in range(len(rad)):
            oc = o - cen[k]
            b = oc @ d
            disc = b * b - (oc @ oc - rad[k] ** 2)
            if disc <= 0:
                ok &= disc < -k_margin * err * rad[k]
                continue
            ok &= disc > k_margin * err * rad[k]
            for t in (-b - np.sqrt(disc), -b + np.sqrt(disc)):
                ok &= abs(t - TMIN) > 1e-5                # (a root at the ray's own surface lies at t ~ 0)
                if t > TMIN:
                    ts_all.append(t)
                    if t < best:
                        best, bid = t, k
                    break
        if bid < 0:
            return thr, rays, ok, 1e-6 + (k_margin * err * 4 + 1e-5) * np.abs(thr)
        ts_all.sort()
        if len(ts_all) > 1:
            ok &= ts_all[1] - ts_all[0] > k_margin * err
        t = best
        pos = o + d * t
        nrm = (pos - cen[bid]) / rad[bid]
        dn = d @ nrm
        ok &= abs(dn) > k_margin * err
        ri = REPLAY_SPHERES[bid][2]
        sa, ss, g = REPLAY_MEDIA[bid, :3].astype(np.float64), float(REPLAY_MEDIA[bid, 3]), float(REPLAY_MEDIA[bid, 4])
        if dn > 0:
            if ss > 0:
                t_s = -np.log(1 - draw()) / ss
                ok &= abs(t_s - t) > k_margin * err * max(t, 1.0)
                if t_s < t:
                    if depth >= MAX_DEPTH:
                        return np.zeros(3), rays, ok, np.full(3, 1e-6)
                    thr = thr * np.exp(-sa * t_s)
                    length += t_s
                    o = o + d * t_s
                    xi1, xi2 = draw(), draw()
                    ok &= abs(d[2]) > k_margin * err                       # the Duff basis' sign branch
                    d = hg_dirs(d[None, :], g, np.array([xi1]), np.array([xi2]))[0]
                    depth += 1
                    err = err * 1.5 + 1e-5
                    continue
            thr = thr * np.exp(-sa * t)
            length += t
        if depth >= MAX_DEPTH:
            return np.zeros(3), rays, ok, np.full(3, 1e-6)
        if dn > 0:
            out_n, nint, cosine = -nrm, ri, ri * dn
        else:
            out_n, nint, cosine = nrm, 1.0 / ri, -dn
        dt = d @ out_n
        discr = 1.0 - nint * nint * (1.0 - dt * dt)
        ok &= abs(discr) > k_margin * err
        refl_p = schlick(cosine, ri) if discr > 0 else 1.0
        u = draw()
        ok &= abs(u - refl_p) > k_margin * err
        if u < refl_p:
            d = d - 2 * (d @ nrm) * nrm
        else:
            d = nint * (d - out_n * dt) - out_n * np.sqrt(discr)
        d /= np.linalg.norm(d)
        o = pos
        depth += 1
        err = err * 1.5 + 1e-5


@pytest.mark.parametrize("ls", [1, 0])
def test_samples_replay_in_float64(mctx, ls):
    """At spp 1 each caller ray is one sample: its value and ray count (trace_samples with a one-entry list) must be
    the replay's wherever every decision along the path has a clear margin; at least 95 % must have one."""
    import sample_replay as sr
    mctx.set_option("light_sampling", ls)
    sph, mats, cam, em = replay_scene()
    mctx.set_scene(sph, mats, cam, em)
    mctx.set_environment(np.ones((4, 8, 3), np.float32))
    mctx.set_media(REPLAY_MEDIA)
    rng = np.random.default_rng(21 + ls)
    n_out, n_in = 300, 300
    aim = sph["center"][rng.integers(0, len(sph), n_out)] + rng.normal(scale=0.4, size=(n_out, 3))
    orig = rng.normal(size=(n_out, 3))
    orig = 6.0 * orig / np.linalg.norm(orig, axis=1, keepdims=True)
    outside = np.concatenate([orig, aim - orig], 1).astype(np.float32)
    rays = np.concatenate([outside, sr.inside_glass_rays(sph, mats, n_in, seed=5 + ls)])
    frame = 3
    (s4, _q4), _ = mctx.trace_samples(rays, spp=1, frame=frame)
    good, bad = 0, []
    seeds = sr.ray_seeds(np.arange(len(rays)), 1, 0, frame)
    for i in range(len(rays)):
        val, nr, ok, tol = replay_one(rays[i], seeds[i], sph)
        if not ok:
            continue
        good += 1
        (one, _), kr = mctx.trace_samples(rays, entries=np.array([i], np.int32), spp=1, frame=frame)
        if kr != nr or s4[i, 3] != 1 or (np.abs(s4[i, :3] - val) > tol).any() or one[0].tobytes() != s4[i].tobytes():
            bad.append((i, kr, nr, s4[i].tolist(), val.tolist()))
    print(f"replay: {good} of {len(rays)} samples well-conditioned, {len(bad)} differ")
    assert not bad, bad[:8]
    assert good >= 0.95 * len(rays), good


# ---- 5. the 46-sphere scene ------------------------------------------------------------------------------------------
def _per_sphere_frames(ctx, rays, ids, frames, spp):
    """[frames, spheres, 3] per-frame means by first-hit sphere."""
    ns = int(ids.max()) + 1
    out = np.zeros((frames, ns, 3))
    cnt = np.bincount(ids, minlength=ns)
    for f in range(frames):
        img, _ = ctx.trace_rays(rays, spp=spp, frame=f)
        for ch in range(3):
            out[f, :, ch] = np.bincount(ids, weights=img[:, ch].astype(np.float64), minlength=ns) / np.maximum(cnt, 1)
    return out, cnt


@pytest.mark.parametrize("extras", ["plain", "env_tex"])
def test_scene46_light_sampling_on_and_off_agree(mctx, extras):
    w, h = 160, 90
    s, m, c, em = scenes.reference_scene(w, h)
    media = np.zeros((len(s), 5), np.float32)
    media[GLASS46] = (0.8, 0.3, 0.1, 2.0, 0.6)
    rays = scenes.camera_rays(c, w, h, seed=2)
    res = {}
    for ls in (1, 0):
        mctx.set_option("light_sampling", ls)
        mctx.set_scene(s, m, c, em)
        if extras == "env_tex":
            mctx.set_environment(np.random.default_rng(6).uniform(0.0, 1.5, (16, 32, 3)).astype(np.float32))
            mctx.set_option("environment_sampling", 1)
            mctx.set_textures(_const_layers(0.8), np.zeros(len(s), np.int32))
        mctx.set_media(media)
        (_a, _n, ids), _ = mctx.trace_aovs(rays)
        keep = ids >= 0
        frames, cnt = _per_sphere_frames(mctx, rays[keep], ids[keep], 24, 8)
        res[ls] = frames
    on, off = res[1], res[0]
    m_on, m_off = on.mean(0), off.mean(0)
    se = np.sqrt(on.var(0, ddof=1) / on.shape[0] + off.var(0, ddof=1) / off.shape[0])
    big = cnt >= 100
    assert big[GLASS46]
    bad = (np.abs(m_on - m_off) > 5 * se + 1e-3 * np.abs(m_off)) & big[:, None]
    assert not bad.any(), [(int(i), m_on[i], m_off[i], se[i]) for i in np.nonzero(bad.any(1))[0]]


# ---- 6. routing, refusals, lifetime -----------------------------------------------------------------------------------
def _kinds(ctx):
    return [k for k in ctx.last_kernels() if k.startswith("k_fast") and not k.startswith("k_fast_aov")]


def _reference_form_only(kinds, inst):
    """Every trace kernel is a slab-queue instance `inst` (e.g. "<128, 6, 0>") of the family that carries the medium
    step (draw_samples' k_fast_samples instances have a fourth template argument)."""
    return bool(kinds) and all(k.startswith(("k_fast_queue", "k_fast_rays", "k_fast_samples")) and inst[:-1] in k
                               for k in kinds)


@pytest.mark.parametrize("which,inst", [("46", "<128, 6, 0>"), ("4096", "<768, 1, 0>")])
def test_media_route_to_the_reference_form_instances(mctx, which, inst):
    make, w, h, _v = SCENES[which]
    s, m, c, em = make()
    mctx.set_scene(s, m, c, em)
    _draw(mctx, w, h)
    default = mctx.last_kernels()
    media = np.zeros((len(s), 5), np.float32)
    media[np.nonzero(m["type"] == F.DIELECTRIC)[0][0]] = (0.2, 0.2, 0.2, 1.0, 0.0)
    mctx.set_media(media)
    for v in (-1, 3, 9):
        mctx.set_option("fast_variant", v)
        _draw(mctx, w, h)
        k = _kinds(mctx)
        assert _reference_form_only(k, inst) and all(x.startswith(TEX_KERNELS) for x in k), (v, k)
    mctx.set_option("fast_variant", -1)
    host = np.zeros((h, w, 4), np.float32)
    mctx.draw(0, 1, w, h, host, mode=MODE_FAST)
    assert _reference_form_only(_kinds(mctx), inst), mctx.last_kernels()
    rays = scenes.camera_rays(c, w, h)
    pts = np.concatenate([np.zeros((8, 3)), np.tile([0, 1, 0], (8, 1))], 1).astype(np.float32)
    for call in (lambda: mctx.trace_rays(rays, spp=2), lambda: mctx.draw_samples(0, w, h, spp=2),
                 lambda: mctx.trace_samples(rays, spp=2), lambda: mctx.trace_irradiance(pts, spp=2)):
        call()
        assert _reference_form_only(_kinds(mctx), inst), mctx.last_kernels()
    mctx.set_media(None)                                  # removal: the default kernel again
    _draw(mctx, w, h)
    assert mctx.last_kernels() == default


def test_refusals_keep_the_media(mctx):
    w, h = 64, 36
    s, m, c, em = scenes.reference_scene(w, h)
    mctx.set_scene(s, m, c, em)
    media = _media(len(s), {GLASS46: (0.5, 0.5, 0.5, 2.0, 0.3)})
    mctx.set_media(media)
    mctx.set_spp(1)
    ref, rr = _draw(mctx, w, h)
    L = mctx._L
    for bad, text in (((GLASS46, 3, -1.0), "tpt_set_media: sphere 7 has sigma_s = -1"),
                      ((2, 0, -0.0), "tpt_set_media: sphere 2 has sigma_a.r = -0"),
                      ((5, 1, np.inf), "tpt_set_media: sphere 5 has sigma_a.g = inf"),
                      ((0, 4, 1.0), "tpt_set_media: sphere 0 has g = 1"),
                      ((1, 4, np.nan), "tpt_set_media: sphere 1 has g = nan")):
        b = media.copy()
        b[bad[0], bad[1]] = bad[2]
        assert L.tpt_set_media(mctx._h, b.ctypes.data, len(b)) != 0
        assert L.tpt_last_error(mctx._h).decode() == text
    assert L.tpt_set_media(mctx._h, media.ctypes.data, -1) != 0
    assert "numSpheres" in L.tpt_last_error(mctx._h).decode()
    got, gr = _draw(mctx, w, h)
    assert gr == rr and got.tobytes() == ref.tobytes()    # the media stayed
    for v in (0, 1, 2, 4, 5, 6, 7, 8):
        mctx.set_option("fast_variant", v)
        with pytest.raises(TptError, match=f"the scene has media \\(tpt_set_media\\), and fast_variant {v}"):
            _draw(mctx, w, h)
    mctx.set_option("fast_variant", -1)
    for mode in (MODE_EXACT, MODE_REFGPU, MODE_REFGPU_FAST):
        with pytest.raises(TptError, match="the scene has media, and only TPT_MODE_FAST"):
            _draw(mctx, w, h, mode=mode)
    mctx.set_media(None)
    _draw(mctx, w, h, mode=MODE_EXACT)                    # allowed again


def test_media_survive_set_scene_and_upload_sizes(mctx):
    w, h = 64, 36
    s, m, c, em = scenes.reference_scene(w, h)
    mctx.set_option("scene_upload_always", 1)
    mctx.set_scene(s, m, c, em)
    assert mctx.last_scene_upload_bytes() == 2720
    mctx.set_spp(1)
    plain, _ = _draw(mctx, w, h)
    media = _media(len(s), {GLASS46: (0.3, 0.6, 0.9, 3.0, -0.2)})
    mctx.set_media(media)
    n = len(s)
    section = (n + 1) * 16 + -(-(n + 1) * 4 // 16) * 16
    assert mctx.last_scene_upload_bytes() == 2720 + section
    with_media, r1 = _draw(mctx, w, h)
    assert with_media.tobytes() != plain.tobytes()
    mctx.set_scene(s, m, c, em)                           # kept across tpt_set_scene
    assert mctx.last_scene_upload_bytes() == 2720 + section
    again, r2 = _draw(mctx, w, h)
    assert r1 == r2 and again.tobytes() == with_media.tobytes()
    mctx.set_option("scene_upload_always", 0)
    # before any scene: stored, applied by the first tpt_set_scene
    from toypathtracer_b200 import Context
    fresh = Context(0)
    try:
        fresh.set_media(media)
        fresh.set_scene(s, m, c, em)
        fresh.set_spp(1)
        first, r3 = _draw(fresh, w, h)
        assert r3 == r1 and first.tobytes() == with_media.tobytes()
    finally:
        fresh.close()


def test_draw_issued_before_set_media_keeps_the_old_media(mctx):
    w, h = 1280, 720
    s, m, c, em = scenes.reference_scene(w, h)
    mctx.set_option("fast_kform", 0)
    mctx.set_scene(s, m, c, em)
    mctx.set_spp(1)                                       # one sample per pixel: a draw is bitwise reproducible
    ref, _ = _draw(mctx, w, h)
    buf = torch.zeros((h, w, 4), dtype=torch.float32, device="cuda")
    mctx.draw(0, 1, w, h, buf, mode=MODE_FAST, want_rays=False)     # asynchronous: still in flight
    mctx.set_media(_media(len(s), {GLASS46: (5.0, 5.0, 5.0, 8.0, 0.0)}))
    torch.cuda.synchronize()
    assert buf.cpu().numpy().tobytes() == ref.tobytes()
    after, _ = _draw(mctx, w, h)
    assert after.tobytes() != ref.tobytes()


def test_aovs_do_not_change(mctx):
    w, h = 64, 36
    s, m, c, em = scenes.reference_scene(w, h)
    mctx.set_scene(s, m, c, em)
    rays = scenes.camera_rays(c, w, h, seed=1)
    (a0, n0, i0), r0 = mctx.trace_aovs(rays)
    mctx.set_media(_media(len(s), {GLASS46: (1.0, 0.5, 0.2, 4.0, 0.7)}))
    (a1, n1, i1), r1 = mctx.trace_aovs(rays)
    assert r0 == r1 and a0.tobytes() == a1.tobytes() and n0.tobytes() == n1.tobytes() and i0.tobytes() == i1.tobytes()
