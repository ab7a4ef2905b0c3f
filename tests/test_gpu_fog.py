"""Homogeneous fog between the spheres (tpt_set_fog, Context.set_fog) on the GPU.

1. Zero-sigma fog and removed fog are the identity, bit for bit, ray for ray and kernel for kernel, through every fast call.
2. A pure absorber draws nothing extra: the same ray counts as the no-fog reference-form instance, and no pixel grows.
3. Beer-Lambert: an emitter under a black map seen through absorbing fog from origins inside and outside the ball,
   including rays that leave the ball before the emitter, against Le exp(-sigma_a L) with L in float64.
4. White furnace: a lossless glass sphere in the ball under a constant unit map, sigma_a = 0: every sample is exactly 1.
5. The 46-sphere scene with fog around both emitters: light sampling on and off agree within standard errors, also with
   media, textures, "environment_sampling" and "emission_texture_sampling".
6. A float64 replay of single samples fed their own draws in the documented order, through fog vertices (g -0.5, 0, 0.7),
   shadow transmittance and Lambert shadow rays through fog, light sampling on and off, exact ray counts, at the default
   depth cap and at "max_depth" 2.
7. trace_samples agrees with trace_rays and trace_irradiance, and draw_samples with the draw, sample for sample.
8. Routing to the texture instances only, refusals, tpt_set_scene keeping the fog, a draw in flight keeping the old fog,
   upload sizes and unchanged AOVs."""
import numpy as np
import pytest
import torch

import furnace as F
import sample_replay as sr
from test_gpu_media import _centre_rays, _per_sphere_frames, _reference_form_only, _same, _spp1_calls, glass_scene
from test_gpu_textures import TEX_KERNELS, _const_layers, _draw, _every_call
from toypathtracer_b200 import MATERIAL_DTYPE, MODE_EXACT, MODE_FAST, MODE_REFGPU, MODE_REFGPU_FAST, SPHERE_DTYPE, TptError, scenes

pytestmark = pytest.mark.gpu

TMIN, MAX_T = 0.001, 1.0e7               # TPT_MIN_T, TPT_MAX_T
LIGHTS46 = (8, 45)                       # the 46-sphere scene's emitters
GLASS46 = 7
# a ball around the camera and both lights of the 46-sphere scene
FOG46 = dict(centre=(0.0, 0.0, -1.5), radius=6.0)


@pytest.fixture
def fctx(gpu_ctx):
    yield gpu_ctx
    gpu_ctx.set_fog(None)
    gpu_ctx.set_media(None)
    gpu_ctx.set_textures(None)
    gpu_ctx.set_emission_textures(None)
    gpu_ctx.set_environment(None)
    for k, v in (("fast_variant", -1), ("fast_kform", 2), ("light_sampling", 1), ("environment_sampling", 0),
                 ("emission_texture_sampling", 0), ("max_depth", 10), ("scene_upload_always", 0)):
        gpu_ctx.set_option(k, v)
    gpu_ctx.set_spp(4)


# ---- 1. inert fog --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ls", [1, 0])
def test_zero_sigma_and_removed_fog_are_the_identity(fctx, ls):
    w, h = 64, 36
    s, m, c, em = scenes.reference_scene(w, h)
    fctx.set_option("light_sampling", ls)
    fctx.set_scene(s, m, c, em)
    ref = _every_call(fctx, w, h, c, s, (-1, 3, 9))
    _draw(fctx, w, h)
    kern = fctx.last_kernels()
    fctx.set_fog(**FOG46, sigma_a=0.0, sigma_s=0.0, g=0.5)
    assert fctx.last_scene_upload_bytes() == 0            # the plain scene's blob: nothing to upload
    _same(_every_call(fctx, w, h, c, s, (-1, 3, 9)), ref)
    _draw(fctx, w, h)
    assert fctx.last_kernels() == kern
    fctx.set_fog(**FOG46, sigma_a=0.2, sigma_s=0.3)
    fctx.set_fog(None)
    _same(_every_call(fctx, w, h, c, s, (-1, 3, 9)), ref)
    _draw(fctx, w, h)
    assert fctx.last_kernels() == kern


# ---- 2. a pure absorber ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ls", [1, 0])
def test_pure_absorber_draws_nothing_and_only_darkens(fctx, ls):
    w, h = 64, 36
    s, m, c, em = scenes.reference_scene(w, h)
    fctx.set_option("light_sampling", ls)
    fctx.set_option("fast_kform", 0)
    fctx.set_scene(s, m, c, em)
    ref = _spp1_calls(fctx, w, h, c, s)
    fctx.set_fog(**FOG46, sigma_a=(0.05, 0.1, 0.2), sigma_s=0.0, g=0.3)
    got = _spp1_calls(fctx, w, h, c, s)
    darker = 0
    for k in ref:
        (ga, gr), (ra, rr) = got[k], ref[k]
        assert gr == rr, (k, gr, rr)
        ga, ra = np.asarray(ga), np.asarray(ra)
        assert (ga <= ra).all(), (k, int((ga > ra).sum()))
        darker += int((ga < ra).sum())
    assert darker > 0


# ---- 3. Beer-Lambert -------------------------------------------------------------------------------------------------
def chord64(o, d, t, c, R):
    """float64 fog length of the segments o + s d, s in [0, t] (d unit), in the ball {c, R}."""
    p = o - c
    b = (p * d).sum(1)
    hh = p - b[:, None] * d
    disc = R * R - (hh * hh).sum(1)
    q = np.sqrt(np.maximum(disc, 0))
    a = np.maximum(-b - q, 0)
    return np.where(disc > 0, np.maximum(np.minimum(q - b, t) - a, 0), 0.0), a


def one_sphere(centre, radius, mtype, albedo, emissive, ri=1.5):
    sph = np.zeros(1, SPHERE_DTYPE)
    mats = np.zeros(1, MATERIAL_DTYPE)
    sph[0] = (centre, radius, 1.0 / radius)
    mats[0] = (mtype, albedo, emissive, 0.0, ri)
    return sph, mats, F.furnace_camera(8, 8), np.zeros(0, np.int32)


@pytest.mark.parametrize("ls", [1, 0])
def test_beer_lambert_towards_an_emitter(fctx, ls):
    """A black emitter-only Lambert sphere (albedo 0, Le) at (0, 0, -5) under a black map; fog ball {(0, 0, 0), 3}.
    Rays aimed at the emitter's centre from origins inside the ball, outside it on the far side (crossing it), and
    beside it (passing outside it, or leaving it before the emitter): the value is Le exp(-sigma_a L) exactly up to
    float32 rounding."""
    le = np.float32([2.0, 3.0, 4.0])
    sa = np.float32([0.05, 0.2, 0.6])
    centre = np.array([0.0, 0.0, -5.0])
    fctx.set_option("light_sampling", ls)
    fctx.set_scene(*one_sphere(centre, 1.0, F.LAMBERT, (0, 0, 0), le))
    fctx.set_environment(np.zeros((4, 8, 3), np.float32))
    fctx.set_fog((0.0, 0.0, 0.0), 3.0, sa, 0.0)
    rng = np.random.default_rng(5)
    n = 3000
    inside = rng.normal(size=(n, 3))
    inside *= (rng.uniform(0, 2.9, n) / np.linalg.norm(inside, axis=1))[:, None]
    far = np.stack([rng.uniform(-1, 1, n), rng.uniform(-1, 1, n), rng.uniform(4, 9, n)], 1)
    side = np.stack([rng.uniform(-6, 6, n), rng.uniform(-6, 6, n), rng.uniform(-2, 4, n)], 1)
    o = np.concatenate([inside, far, side])
    d = centre - o
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    rays = np.concatenate([o, d], 1).astype(np.float32)
    o64, d64 = rays[:, :3].astype(np.float64), rays[:, 3:].astype(np.float64)
    d64 /= np.linalg.norm(d64, axis=1, keepdims=True)
    p = o64 - centre
    b = (p * d64).sum(1)
    t = -b - np.sqrt(b * b - (p * p).sum(1) + 1.0)
    L, _ = chord64(o64, d64, t, np.zeros(3), 3.0)
    # every kind occurs: fully inside, crossing, leaving before the emitter, never entering
    assert (L == 0).sum() > 100 and ((L > 0) & (L < t - 1e-3)).sum() > 1000
    want = le[None, :] * np.exp(-sa[None, :].astype(np.float64) * L[:, None])
    got, _ = fctx.trace_rays(rays, spp=2)
    err = np.abs(got[:, :3] - want)
    tol = 2e-5 * want + 2e-4 * le * sa * (1 + t[:, None]) * want / le
    assert (err <= tol + 1e-6).all(), (int((err > tol + 1e-6).any(1).sum()), float((err / want).max()))


# ---- 4. white furnace -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ls", [1, 0])
@pytest.mark.parametrize("sigma_s,g,centre,radius", [(0.5, 0.0, (0.3, 0.0, 0.0), 3.0), (1.5, -0.5, (0.3, 0.0, 0.0), 3.0),
                                                     (1.0, 0.8, (0.3, 0.0, 0.0), 3.0), (2.0, 0.3, (0.0, 0.0, 0.0), 1.3)])
def test_white_furnace_every_sample_is_one(fctx, sigma_s, g, centre, radius, ls):
    """Every sample escapes with throughput 1. The thin shell of fog around the glass (radius 1.3) puts many scatter
    points within TPT_MIN_T of the glass: the rays that leave them start at 0 and cannot skip its surface."""
    fctx.set_option("light_sampling", ls)
    fctx.set_option("max_depth", 256)
    fctx.set_scene(*glass_scene(1.0, 1.5))
    fctx.set_environment(np.ones((4, 8, 3), np.float32))
    rng = np.random.default_rng(int(sigma_s * 10) + ls)
    n = 4096
    # origins outside the glass (off-centre inside it, total internal reflection can trap a path until the cap) and
    # its centre
    o = rng.normal(size=(n, 3))
    o *= (rng.uniform(1.05, 6, n) / np.linalg.norm(o, axis=1))[:, None]
    d = rng.normal(size=(n, 3))
    rays = np.concatenate([o, d / np.linalg.norm(d, axis=1, keepdims=True)], 1).astype(np.float32)
    rays = np.concatenate([rays, _centre_rays(256, 4)])
    fctx.set_fog(None)
    _, plain = fctx.trace_samples(rays, spp=8)
    fctx.set_fog(centre, radius, 0.0, sigma_s, g)
    (s4, q4), traced = fctx.trace_samples(rays, spp=8)
    assert (s4[:, 3] == 8).all()
    assert (s4[:, :3] == s4[:, 3:4]).all(), s4[(s4[:, :3] != s4[:, 3:4]).any(1)][:4]
    assert (q4[:, :3] == s4[:, 3:4]).all()
    # the fog scattered: more rays than without it
    assert traced > plain


# ---- 5. the 46-sphere scene: light sampling on and off agree ------------------------------------------------------------
@pytest.mark.parametrize("extras", ["plain", "all"])
def test_scene46_light_sampling_on_and_off_agree(fctx, extras):
    w, h = 160, 90
    s, m, c, em = scenes.reference_scene(w, h)
    rays = scenes.camera_rays(c, w, h, seed=2)
    res = {}
    for ls in (1, 0):
        fctx.set_option("light_sampling", ls)
        fctx.set_scene(s, m, c, em)
        if extras == "all":
            media = np.zeros((len(s), 5), np.float32)
            media[GLASS46] = (0.4, 0.2, 0.1, 1.0, 0.3)
            fctx.set_media(media)
            fctx.set_environment(np.random.default_rng(6).uniform(0.0, 1.5, (16, 32, 3)).astype(np.float32))
            fctx.set_option("environment_sampling", 1)
            fctx.set_textures(_const_layers(0.8), np.zeros(len(s), np.int32))
            emit = np.random.default_rng(8).uniform(0.5, 1.5, (1, 8, 16, 3)).astype(np.float32)
            layers = np.full(len(s), -1, np.int32)
            layers[list(LIGHTS46)] = 0
            fctx.set_emission_textures(emit, layers)
            fctx.set_option("emission_texture_sampling", 1)
        fctx.set_fog(**FOG46, sigma_a=(0.01, 0.02, 0.03), sigma_s=0.08, g=0.4)
        (_a, _n, ids), _ = fctx.trace_aovs(rays)
        keep = ids >= 0
        frames, cnt = _per_sphere_frames(fctx, rays[keep], ids[keep], 24, 8)
        res[ls] = frames
    on, off = res[1], res[0]
    m_on, m_off = on.mean(0), off.mean(0)
    se = np.sqrt(on.var(0, ddof=1) / on.shape[0] + off.var(0, ddof=1) / off.shape[0])
    big = cnt >= 100
    bad = (np.abs(m_on - m_off) > 5 * se + 1e-3 * np.abs(m_off)) & big[:, None]
    assert not bad.any(), [(int(i), m_on[i], m_off[i], se[i]) for i in np.nonzero(bad.any(1))[0]]
    # the fog glows: light sampling makes the estimate no noisier overall
    assert se[big].mean() > 0


# ---- 6. float64 replay of single samples ----------------------------------------------------------------------------
REPLAY = [((0.0, -101.0, -2.0), 100.0, (0.6, 0.6, 0.6), (0, 0, 0)),     # floor
          ((0.0, 0.0, -3.0), 1.0, (0.7, 0.5, 0.3), (0, 0, 0)),
          ((2.0, 0.2, -2.0), 0.6, (0.4, 0.8, 0.5), (0, 0, 0)),
          ((-1.5, 1.6, -2.5), 0.5, (0.0, 0.0, 0.0), (6.0, 5.0, 3.0)),    # light 0
          ((1.0, 2.0, -4.0), 0.4, (0.0, 0.0, 0.0), (3.0, 4.0, 8.0))]     # light 1
REPLAY_FOG = ((0.0, 0.5, -2.5), 3.5)
REPLAY_SIGMA_A = np.array([0.08, 0.15, 0.25])
REPLAY_SIGMA_S = 0.35
ENV = 0.25


def replay_scene():
    n = len(REPLAY)
    sph = np.zeros(n, SPHERE_DTYPE)
    mats = np.zeros(n, MATERIAL_DTYPE)
    for i, (c, r, alb, e) in enumerate(REPLAY):
        sph[i] = (c, r, 1.0 / r)
        mats[i] = (F.LAMBERT, alb, e, 0.0, 1.0)
    sph["invRadius"] = (np.float32(1) / sph["radius"]).astype(np.float32)
    return sph, mats, F.furnace_camera(8, 8), np.array([3, 4], np.int32)


def hg_phase(cos_t, g):
    g = float(np.float32(g))
    if abs(g) < 1e-3:
        return float(np.float32(1.0 / (4 * np.pi)))
    return (1 - g * g) / (4 * np.pi * (1 + g * g - 2 * g * cos_t) ** 1.5)


def hg_dir(d, g, xi1, xi2):
    g = float(np.float32(g))
    if abs(g) >= 1e-3:
        s = (1 - g * g) / (1 - g + 2 * g * xi1)
        cos_t = min(max((1 + g * g - s * s) / (2 * g), -1.0), 1.0)
    else:
        cos_t = 1 - 2 * xi1
    sin_t = np.sqrt(max(1 - cos_t * cos_t, 0.0))
    su, sv = duff(d)
    phi = sr.TWO_PI32 * xi2
    out = su * sin_t * np.cos(phi) + sv * sin_t * np.sin(phi) + d * cos_t
    return out / np.linalg.norm(out)


def duff(w):
    sgn = -1.0 if np.signbit(w[2]) else 1.0
    a = -1.0 / (sgn + w[2])
    b = w[0] * w[1] * a
    return (np.array([1 + sgn * w[0] * w[0] * a, sgn * b, -sgn * w[0]]), np.array([b, sgn + w[1] * w[1] * a, -w[1]]))


class Replay:
    """One sample of the fast estimator in float64, fed its own stream; `ok` false where a decision's margin is within a
    multiple of `err`, the bound on how far the kernel's float32 path can have drifted."""

    def __init__(self, sph, mats, seed, ls, g, max_depth):
        self.C = sph["center"].astype(np.float64)
        self.R = sph["radius"].astype(np.float64)
        self.alb = mats["albedo"].astype(np.float64)
        self.le = mats["emissive"].astype(np.float64)
        self.lights = [3, 4]
        self.fc, self.fr = np.array(REPLAY_FOG[0]), REPLAY_FOG[1]
        self.st = sr.Stream(np.array([seed], np.uint32))
        self.ls, self.g, self.max_depth = ls, g, max_depth
        self.ok, self.err, self.rays, self.mag = True, 1e-6, 0, 0.0
        self.col = np.zeros(3)

    def draw(self):
        return float(sr.u01(self.st.draw(np.array([0]))[0]))

    def margin(self, x, scale=1.0):
        self.ok &= abs(x) > 16 * self.err * scale

    def nearest(self, o, d, tmin=TMIN):
        self.rays += 1
        best, bid, roots = MAX_T, -1, []
        for k in range(len(self.R)):
            oc = o - self.C[k]
            b = oc @ d
            hh = oc - b * d
            disc = self.R[k] ** 2 - hh @ hh
            self.margin(disc, self.R[k] * (1 + np.sqrt(oc @ oc)))
            if disc <= 0:
                continue
            for t in (-b - np.sqrt(disc), -b + np.sqrt(disc)):
                self.margin(t - tmin, 1e3)
                if t > tmin:
                    roots.append(t)
                    if t < best:
                        best, bid = t, k
                    break
        roots.sort()
        if len(roots) > 1:
            self.margin(roots[1] - roots[0], 1 + roots[0])
        return best, bid

    def fog_len(self, o, d, t):
        p = o - self.fc
        b = p @ d
        hh = p - b * d
        disc = self.fr ** 2 - hh @ hh
        self.margin(disc, self.fr * (1 + np.sqrt(p @ p)))
        if disc <= 0:
            return 0.0, 0.0
        q = np.sqrt(disc)
        a = max(-b - q, 0.0)
        self.margin(-b - q, 1 + abs(b))
        if t < MAX_T:
            self.margin(q - b - t, 1 + t)
        return max(min(q - b, t) - a, 0.0), a

    def add(self, v):
        self.col += v
        self.mag += np.abs(v).max()

    def shadow(self, o, l, j, w, thr, tmin=TMIN):
        """Light j's shadow ray from o along l with weight w: adds thr Le_j w T when it reaches the light."""
        t, hid = self.nearest(o, l, tmin)
        k = self.lights[j]
        if hid != k:
            return
        x = o + l * t
        face = l @ (x - self.C[k])
        self.margin(face, self.R[k])
        tr = np.ones(3)
        if face <= 0:
            L, _ = self.fog_len(o, l, t)
            tr = np.exp(-(REPLAY_SIGMA_A + REPLAY_SIGMA_S) * L)
        self.add(thr * self.le[k] * w * tr)

    def cone(self, o, k, nl, fog):
        pc = self.C[k] - o
        d2 = pc @ pc
        sw = pc / np.sqrt(d2)
        self.margin(sw[2], 1 + 1 / np.sqrt(d2))
        su, sv = duff(sw)
        cam = np.sqrt(1 - self.R[k] ** 2 / d2)
        e1, e2 = self.draw(), self.draw()
        cos_a = 1 - e1 + e1 * cam
        sin_a = np.sqrt(max(1 - cos_a * cos_a, 0.0))
        phi = sr.TWO_PI32 * e2
        l = su * np.cos(phi) * sin_a + sv * np.sin(phi) * sin_a + sw * cos_a
        omega = sr.TWO_PI32 * (1 - cam)
        if fog:
            return l, omega * hg_phase(l @ nl, self.g)
        dl = l @ nl
        self.margin(dl)
        return l, max(dl, 0.0) * omega * sr.INV_PI32

    def run(self, o, d):
        d = d / np.linalg.norm(d)
        thr, depth, do_e = np.ones(3), 0, True
        tmin = TMIN                    # 0 for the rays that leave a fog scatter point
        sa, ss = REPLAY_SIGMA_A, REPLAY_SIGMA_S
        while True:
            t, hid = self.nearest(o, d, tmin)
            tmin = TMIN
            air = True
            if hid >= 0:
                pos = o + d * t
                nrm = (pos - self.C[hid]) / self.R[hid]
                dn = d @ nrm
                self.margin(dn)
                air = dn <= 0
            scattered = False
            if air:
                L, tin = self.fog_len(o, d, t)
                if L > 0:
                    ts = -np.log(1 - self.draw()) / ss
                    self.margin(ts - L, 1 + L)
                    if ts < L:
                        scattered = True
                        if depth >= self.max_depth:
                            return
                        thr = thr * np.exp(-sa * ts)
                        o = o + d * (tin + ts)
                        xi1, xi2 = self.draw(), self.draw()
                        self.margin(d[2])
                        nd = hg_dir(d, self.g, xi1, xi2)
                        if self.ls:
                            for j, k in enumerate(self.lights):
                                l, w = self.cone(o, k, d, True)
                                self.shadow(o, l, j, w, thr, 0.0)
                            do_e = False
                        else:
                            do_e = True
                        d = nd
                        depth += 1
                        tmin = 0.0
                        self.err = self.err * 1.5 + 1e-5
                        continue
                    thr = thr * np.exp(-sa * L)
            if hid < 0:
                self.add(thr * ENV)
                return
            if depth >= self.max_depth:
                self.add(thr * self.le[hid])
                return
            if not self.ls or do_e:
                self.add(thr * self.le[hid])
            x1, x2 = self.st.draw(np.array([0]))[0], self.st.draw(np.array([0]))[0]
            u = sr.unit_vector(sr.Exact(), np.array([x1]), np.array([x2]))[0]
            tgt = nrm + u
            self.margin(np.linalg.norm(tgt), 10)
            nd = tgt / np.linalg.norm(tgt)
            alb = thr * self.alb[hid]
            if self.ls:
                nl = nrm if nrm @ d < 0 else -nrm
                for j, k in enumerate(self.lights):
                    if k == hid:
                        continue
                    l, w = self.cone(pos, k, nl, False)
                    self.shadow(pos, l, j, w, alb)
                do_e = False
            thr, o, d = alb, pos, nd
            depth += 1
            self.err = self.err * 1.5 + 1e-5


def _replay_rays(sph, n, seed):
    rng = np.random.default_rng(seed)
    c = np.array(REPLAY_FOG[0])
    # origins inside the fog ball (above the floor) and outside it, aimed at the spheres or anywhere
    inside = c + rng.normal(size=(n, 3)) * 1.2
    inside[:, 1] = np.maximum(inside[:, 1], -0.8)
    outside = c + np.array([0.0, 1.0, 9.0]) + rng.normal(size=(n, 3))
    o = np.concatenate([inside, outside])
    aim = sph["center"][rng.integers(1, len(sph), 2 * n)] + rng.normal(scale=0.5, size=(2 * n, 3))
    d = np.where((rng.random(2 * n) < 0.7)[:, None], aim - o, rng.normal(size=(2 * n, 3)))
    return np.concatenate([o, d], 1).astype(np.float32)


@pytest.mark.parametrize("max_depth", [10, 2])
@pytest.mark.parametrize("g", [-0.5, 0.0, 0.7])
@pytest.mark.parametrize("ls", [1, 0])
def test_samples_replay_in_float64(fctx, ls, g, max_depth):
    """At spp 1 each caller ray is one sample: its value and its ray count (trace_samples with a one-entry list) must
    be the replay's wherever every decision has a clear margin (the margins are wide: about half of the samples keep
    them), and most of those must carry light."""
    fctx.set_option("light_sampling", ls)
    fctx.set_option("max_depth", max_depth)
    sph, mats, cam, em = replay_scene()
    fctx.set_scene(sph, mats, cam, em)
    fctx.set_environment(np.full((4, 8, 3), ENV, np.float32))
    fctx.set_fog(REPLAY_FOG[0], REPLAY_FOG[1], REPLAY_SIGMA_A.astype(np.float32), REPLAY_SIGMA_S, g)
    rays = _replay_rays(sph, 150, seed=31 + ls)
    frame = 2
    (s4, _q4), _ = fctx.trace_samples(rays, spp=1, frame=frame)
    seeds = sr.ray_seeds(np.arange(len(rays)), 1, 0, frame)
    good, bad, lit = 0, [], 0
    for i in range(len(rays)):
        r = Replay(sph, mats, seeds[i], ls, g, max_depth)
        r.run(rays[i, :3].astype(np.float64), rays[i, 3:].astype(np.float64))
        if not r.ok:
            continue
        good += 1
        lit += int(r.mag > 0)
        (one, _), kr = fctx.trace_samples(rays, entries=np.array([i], np.int32), spp=1, frame=frame)
        tol = 1e-6 + 2e-3 * r.mag
        if kr != r.rays or s4[i, 3] != 1 or (np.abs(s4[i, :3] - r.col) > tol).any() or one[0].tobytes() != s4[i].tobytes():
            bad.append((i, kr, r.rays, s4[i, :3].tolist(), r.col.tolist()))
    print(f"replay ls {ls} g {g} cap {max_depth}: {good} of {len(rays)} well-conditioned, {len(bad)} differ")
    assert not bad, bad[:6]
    assert good >= 0.3 * len(rays) and lit >= 0.5 * good, (good, lit)


# ---- 7. the sample calls agree with the mean calls ------------------------------------------------------------------
@pytest.mark.parametrize("ls", [1, 0])
def test_sample_calls_agree_with_the_mean_calls(fctx, ls):
    w, h = 64, 36
    s, m, c, em = scenes.reference_scene(w, h)
    fctx.set_option("light_sampling", ls)
    fctx.set_scene(s, m, c, em)
    fctx.set_fog(**FOG46, sigma_a=(0.02, 0.04, 0.06), sigma_s=0.2, g=0.5)
    rays = scenes.camera_rays(c, w, h, seed=3)
    mean, r1 = fctx.trace_rays(rays, spp=1, frame=4)
    (s4, q4), r2 = fctx.trace_samples(rays, spp=1, frame=4)
    assert r1 == r2 and (s4[:, 3] == 1).all() and s4[:, :3].tobytes() == np.ascontiguousarray(mean[:, :3]).tobytes()
    assert (q4[:, :3] == s4[:, :3] ** 2).all()
    rng = np.random.default_rng(4)
    ids = rng.integers(0, len(s), 600).astype(np.int32)
    nrm = rng.normal(size=(600, 3))
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    pts = np.concatenate([s["center"][ids] + s["radius"][ids][:, None] * nrm, nrm], 1).astype(np.float32)
    irr, r3 = fctx.trace_irradiance(pts, ids, spp=1, frame=1)
    (p4, _), r4 = fctx.trace_samples(pts, ids=ids, points=True, spp=1, frame=1)
    assert r3 == r4 and p4[:, :3].tobytes() == np.ascontiguousarray(irr[:, :3]).tobytes()
    img, r5 = _draw(fctx, w, h, spp=1, frame=2)
    (d4, _dq), r6 = fctx.draw_samples(2, w, h, spp=1)
    d4 = d4.cpu().numpy().reshape(h, w, 4)
    assert r5 == r6 and d4[..., :3].tobytes() == np.ascontiguousarray(img[..., :3]).tobytes()


# ---- 8. routing, refusals, lifetime ----------------------------------------------------------------------------------
def _kinds(ctx):
    return [k for k in ctx.last_kernels() if k.startswith("k_fast") and not k.startswith("k_fast_aov")]


@pytest.mark.parametrize("which,inst", [("46", "<128, 6, 0>"), ("4096", "<768, 1, 0>")])
def test_fog_routes_to_the_texture_instances(fctx, which, inst):
    w, h = (64, 36) if which == "46" else (48, 27)
    s, m, c, em = scenes.reference_scene(w, h) if which == "46" else scenes.stress_scene(w, h)
    fctx.set_scene(s, m, c, em)
    _draw(fctx, w, h)
    default = fctx.last_kernels()
    fctx.set_fog(**FOG46, sigma_a=0.05, sigma_s=0.1)
    for v in (-1, 3, 9):
        fctx.set_option("fast_variant", v)
        _draw(fctx, w, h)
        k = _kinds(fctx)
        assert _reference_form_only(k, inst) and all(x.startswith(TEX_KERNELS) for x in k), (v, k)
    fctx.set_option("fast_variant", -1)
    host = np.zeros((h, w, 4), np.float32)
    fctx.draw(0, 1, w, h, host, mode=MODE_FAST)
    assert _reference_form_only(_kinds(fctx), inst), fctx.last_kernels()
    rays = scenes.camera_rays(c, w, h)
    pts = np.concatenate([np.zeros((8, 3)), np.tile([0, 1, 0], (8, 1))], 1).astype(np.float32)
    for call in (lambda: fctx.trace_rays(rays, spp=2), lambda: fctx.draw_samples(0, w, h, spp=2),
                 lambda: fctx.trace_samples(rays, spp=2), lambda: fctx.trace_irradiance(pts, spp=2)):
        call()
        assert _reference_form_only(_kinds(fctx), inst), fctx.last_kernels()
    fctx.set_fog(None)
    _draw(fctx, w, h)
    assert fctx.last_kernels() == default


def test_refusals_keep_the_fog(fctx):
    w, h = 64, 36
    s, m, c, em = scenes.reference_scene(w, h)
    fctx.set_scene(s, m, c, em)
    fctx.set_fog(**FOG46, sigma_a=0.05, sigma_s=0.3, g=0.2)
    fctx.set_spp(1)
    ref, rr = _draw(fctx, w, h)
    L = fctx._L
    good = np.float32([0.0, 0.0, -1.5, 6.0, 0.05, 0.05, 0.05, 0.3, 0.2])
    for f, v, text in ((0, np.nan, "centre.x = nan"), (2, np.inf, "centre.z = inf"), (3, -1.0, "radius = -1"),
                       (3, 0.0, "radius = 0"), (3, np.inf, "radius = inf"), (4, -0.0, "sigma_a.r = -0"),
                       (6, np.nan, "sigma_a.b = nan"), (7, -2.0, "sigma_s = -2"), (8, 1.0, "g = 1"),
                       (8, -1.0, "g = -1"), (8, np.nan, "g = nan")):
        b = good.copy()
        b[f] = v
        assert L.tpt_set_fog(fctx._h, b.ctypes.data) != 0
        assert L.tpt_last_error(fctx._h).decode() == "tpt_set_fog: " + text
    got, gr = _draw(fctx, w, h)
    assert gr == rr and got.tobytes() == ref.tobytes()
    for v in (0, 1, 2, 4, 5, 6, 7, 8):
        fctx.set_option("fast_variant", v)
        with pytest.raises(TptError, match=f"the scene has fog \\(tpt_set_fog\\), and fast_variant {v} does not trace it"):
            _draw(fctx, w, h)
    fctx.set_option("fast_variant", -1)
    for mode in (MODE_EXACT, MODE_REFGPU, MODE_REFGPU_FAST):
        with pytest.raises(TptError, match="the scene has fog, and only TPT_MODE_FAST"):
            _draw(fctx, w, h, mode=mode)
    # with media as well, the media's refusal comes first and keeps its text
    media = np.zeros((len(s), 5), np.float32)
    media[GLASS46] = (0.1, 0.1, 0.1, 1.0, 0.0)
    fctx.set_media(media)
    with pytest.raises(TptError, match="the scene has media, and only TPT_MODE_FAST"):
        _draw(fctx, w, h, mode=MODE_EXACT)
    fctx.set_media(None)
    fctx.set_fog(None)
    _draw(fctx, w, h, mode=MODE_EXACT)


def test_fog_survives_set_scene_and_upload_sizes(fctx):
    w, h = 64, 36
    s, m, c, em = scenes.reference_scene(w, h)
    fctx.set_option("scene_upload_always", 1)
    fctx.set_scene(s, m, c, em)
    assert fctx.last_scene_upload_bytes() == 2720
    fctx.set_spp(1)
    plain, _ = _draw(fctx, w, h)
    fctx.set_fog(**FOG46, sigma_a=(0.02, 0.03, 0.04), sigma_s=0.25, g=-0.3)
    assert fctx.last_scene_upload_bytes() == 2720 + 48
    with_fog, r1 = _draw(fctx, w, h)
    assert with_fog.tobytes() != plain.tobytes()
    fctx.set_scene(s, m, c, em)
    assert fctx.last_scene_upload_bytes() == 2720 + 48
    again, r2 = _draw(fctx, w, h)
    assert r1 == r2 and again.tobytes() == with_fog.tobytes()
    fctx.set_option("scene_upload_always", 0)
    fctx.set_fog(**FOG46, sigma_a=(0.02, 0.03, 0.04), sigma_s=0.25, g=-0.3)
    assert fctx.last_scene_upload_bytes() == 0            # identical bytes are not uploaded again
    from toypathtracer_b200 import Context
    fresh = Context(0)
    try:
        fresh.set_fog(**FOG46, sigma_a=(0.02, 0.03, 0.04), sigma_s=0.25, g=-0.3)
        fresh.set_scene(s, m, c, em)
        fresh.set_spp(1)
        first, r3 = _draw(fresh, w, h)
        assert r3 == r1 and first.tobytes() == with_fog.tobytes()
    finally:
        fresh.close()


def test_draw_issued_before_set_fog_keeps_the_old_fog(fctx):
    w, h = 1280, 720
    s, m, c, em = scenes.reference_scene(w, h)
    fctx.set_option("fast_kform", 0)
    fctx.set_scene(s, m, c, em)
    fctx.set_spp(1)
    ref, _ = _draw(fctx, w, h)
    buf = torch.zeros((h, w, 4), dtype=torch.float32, device="cuda")
    fctx.draw(0, 1, w, h, buf, mode=MODE_FAST, want_rays=False)
    fctx.set_fog(**FOG46, sigma_a=1.0, sigma_s=2.0)
    torch.cuda.synchronize()
    assert buf.cpu().numpy().tobytes() == ref.tobytes()
    after, _ = _draw(fctx, w, h)
    assert after.tobytes() != ref.tobytes()


def test_aovs_do_not_change(fctx):
    w, h = 64, 36
    s, m, c, em = scenes.reference_scene(w, h)
    fctx.set_scene(s, m, c, em)
    rays = scenes.camera_rays(c, w, h, seed=1)
    (a0, n0, i0), r0 = fctx.trace_aovs(rays)
    fctx.set_fog(**FOG46, sigma_a=0.5, sigma_s=1.0, g=0.7)
    (a1, n1, i1), r1 = fctx.trace_aovs(rays)
    assert r0 == r1 and a0.tobytes() == a1.tobytes() and n0.tobytes() == n1.tobytes() and i0.tobytes() == i1.tobytes()
