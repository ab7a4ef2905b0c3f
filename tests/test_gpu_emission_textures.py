"""Sphere emission textures (tpt_set_emission_textures, Context.set_emission_textures) on the GPU.

1. Direct hits: caller rays aimed at black-albedo Lambert emitters return emissive x T(n), T the float64 bilinear
   lat-long model at the hit's normal, at the seam, both poles, on 1 x 1 and 7 x 24 layers and for a one-hot texel;
   spheres with layer -1 or ids past the table keep their emission.
2. Shadow rays, closed form: the irradiance under an emitter whose texture is A on its lower half and B on its upper half
   matches a float64 quadrature of the integral of Le(x(w)) cos(theta) over the emitter's visible cap, with light
   sampling on (the cone's shadow ray, looked up where it meets the light) and off (bounce hits only).
3. A constant texture c is, bit for bit and ray for ray, the untextured scene with emission fl32(e x c), through every
   fast call, with light sampling on and off, under a sampled map, on the 4096-sphere scene, with a constant albedo
   texture at once, and in a mirror corridor whose paths end at the depth cap, are absorbed by Metal or fail in glass
   on emitters.
4. On the 46-sphere scene, light sampling on and off converge to the same image under checker emission textures.
5. No change where they are not set: cleared equals never set; AOVs ignore them; layers on spheres without emission, or
   no layer at all, leave albedo-textured calls' bits alone.
6. Routing, refusals and lifetime."""
import ctypes
import re

import numpy as np
import pytest
import torch

import furnace as F
from conftest import bits_differ, rel_l2
from test_gpu_environment import env_lookup, lat_long_dir, lookup_tolerance
from test_gpu_textures import _const_layers, _draw, _every_call, _texture_kernels_only
from toypathtracer_b200 import (MATERIAL_DTYPE, MODE_EXACT, MODE_FAST, MODE_REFGPU, MODE_REFGPU_FAST, SPHERE_DTYPE,
                                TptError, scenes)

pytestmark = pytest.mark.gpu


@pytest.fixture
def ectx(gpu_ctx):
    yield gpu_ctx
    gpu_ctx.set_emission_textures(None)
    gpu_ctx.set_textures(None)
    gpu_ctx.set_environment(None)
    for k, v in (("fast_variant", -1), ("fast_kform", 2), ("mitsuba_compare", 0), ("light_sampling", 1),
                 ("environment_sampling", 0)):
        gpu_ctx.set_option(k, v)
    gpu_ctx.set_spp(4)


def _scene(centres, radii, types, albedo, emission, rough=0.0, ri=1.5, lights=True):
    sph = np.zeros(len(centres), SPHERE_DTYPE)
    mats = np.zeros(len(centres), MATERIAL_DTYPE)
    for i, (c, r) in enumerate(zip(centres, radii)):
        sph[i] = (c, r, 0.0)
        mats[i] = (types[i], albedo[i], emission[i], rough, ri)
    sph["invRadius"] = (np.float32(1) / sph["radius"]).astype(np.float32)
    em = np.nonzero((mats["emissive"] != 0).any(1))[0].astype(np.int32) if lights else np.zeros(0, np.int32)
    return sph, mats, F.furnace_camera(8, 8), em


# ---- 1. direct hits ----------------------------------------------------------------------------------------------
CENTRES = np.array([[0.0, 0.0, -6.0], [4.0, 0.0, -6.0], [-4.0, 0.0, -6.0], [0.0, 4.0, -6.0]])
EMIT = np.float32([[2.0, 1.5, 0.5], [0.7, 1.1, 3.0], [1.0, 2.0, 3.0], [4.0, 0.5, 1.0]])
LAYER_OF = np.array([1, 0, -1], np.int32)      # sphere 3 lies past the table: untextured


def direct_scene():
    n = len(CENTRES)
    return _scene(CENTRES, [1.0] * n, [F.LAMBERT] * n, [(0, 0, 0)] * n, EMIT)


def _aimed(sphere, normals):
    c = CENTRES[sphere]
    n = np.asarray(normals, np.float64)
    return np.concatenate([c + 2.5 * n, -n], 1).astype(np.float32)


def _normals(w, h, rng):
    d = rng.normal(size=(300, 3))
    dirs = [d / np.linalg.norm(d, axis=1, keepdims=True)]
    vs = rng.uniform(0, h, 6)
    for u in (0.0, 1e-4, 0.5, w - 0.5, w - 1e-4, w):                   # the phi = +-pi seam, both sides
        dirs.append(lat_long_dir(np.full(6, u), vs, w, h))
    us = rng.uniform(0, w, 6)
    for v in (0.0, 1e-4, 0.5, h - 0.5, h - 1e-4, h):                   # both poles
        dirs.append(lat_long_dir(us, np.full(6, v), w, h))
    ii, jj = np.meshgrid(np.arange(w) + 0.5, np.arange(h) + 0.5)
    dirs.append(lat_long_dir(ii.ravel(), jj.ravel(), w, h))
    return np.concatenate(dirs)


@pytest.mark.parametrize("ls", [1, 0])
@pytest.mark.parametrize("size", [(64, 16), (1, 1), (7, 24)])
def test_direct_hit_is_emission_times_lookup(ectx, size, ls):
    """Black albedo: nothing after the first hit adds anything, so trace_rays returns the hit's emission exactly."""
    w, h = size
    rng = np.random.default_rng(w * 100 + h + ls)
    layers = rng.uniform(0.0, 2.0, (2, h, w, 3)).astype(np.float32)
    ectx.set_option("light_sampling", ls)
    ectx.set_option("fast_kform", 0)         # the AOV kernel sweeps in the form the textured trace_rays runs: same normal
    ectx.set_scene(*direct_scene())
    ectx.set_emission_textures(layers, LAYER_OF)
    for sphere in range(len(CENTRES)):
        rays = _aimed(sphere, _normals(w, h, rng))
        (_alb, nrm, ids), _ = ectx.trace_aovs(rays)
        assert (ids == sphere).all(), (sphere, np.unique(ids))
        out, _ = ectx.trace_rays(rays, spp=2)
        layer = LAYER_OF[sphere] if sphere < len(LAYER_OF) else -1
        if layer < 0:
            assert (out[:, :3] == EMIT[sphere]).all(), sphere
            continue
        n = nrm[:, :3].astype(np.float64)             # path_step's normal, (pos - centre) / r in float32
        want = EMIT[sphere].astype(np.float64) * env_lookup(layers[layer], n)
        tol = lookup_tolerance(layers[layer], n, eps=1e-5)[:, None] * EMIT[sphere] + 2.0 ** -21 * np.abs(want) + 1e-7
        bad = (np.abs(out[:, :3] - want) > tol).any(1)
        assert not bad.any(), (size, sphere, int(bad.sum()), n[bad][:3], out[bad][:3], want[bad][:3])
        if w == h == 1:
            assert (out[:, :3] == (EMIT[sphere] * layers[layer, 0, 0]).astype(np.float32)).all()


def test_one_hot_texel_orientation_and_row_order(ectx):
    w, h = 8, 4
    layer = np.zeros((1, h, w, 3), np.float32)
    layer[0, 1, 2] = (1.0, 2.0, 3.0)
    ectx.set_scene(*direct_scene())
    ectx.set_emission_textures(layer, [0])
    ii, jj = np.meshgrid(np.arange(w) + 0.5, np.arange(h) + 0.5)
    out, _ = ectx.trace_rays(_aimed(0, lat_long_dir(ii.ravel(), jj.ravel(), w, h)), spp=1)
    np.testing.assert_allclose(out[:, :3].reshape(h, w, 3), EMIT[0] * layer[0], atol=1e-4)


# ---- 2. shadow rays in closed form ----------------------------------------------------------------------------------
LIGHT_C, LIGHT_R, LIGHT_E = np.array([0.0, 3.0, 0.0]), 1.0, np.float32([1.0, 1.0, 1.0])
GROUND_R = 100.0
TEX_A, TEX_B = np.float32([3.0, 2.0, 1.0]), np.float32([0.1, 0.2, 0.4])


def _half_texture(w=16, h=8):
    t = np.empty((1, h, w, 3), np.float32)
    t[0, : h // 2] = TEX_B                 # rows at the +y pole: the light's upper half
    t[0, h // 2:] = TEX_A                  # its lower half, which faces the receiver
    return t


def _cap_integral(p, nrm, tex, nq=800):
    """Float64 midpoint quadrature over the cone from p to the light of Le(x(w)) cos(theta) dw, x(w) the near hit,
    Le = LIGHT_E x T(normal at x), theta against the receiver's normal nrm."""
    axis = LIGHT_C - p
    dist = np.linalg.norm(axis)
    axis /= dist
    cmax = np.sqrt(1.0 - (LIGHT_R / dist) ** 2)
    u = np.cross(axis, [1.0, 0.0, 0.0] if abs(axis[0]) < 0.9 else [0.0, 0.0, 1.0])
    u /= np.linalg.norm(u)
    v = np.cross(axis, u)
    ca = cmax + (1.0 - cmax) * (np.arange(nq) + 0.5) / nq
    ph = 2.0 * np.pi * (np.arange(nq) + 0.5) / nq
    CA, PH = np.meshgrid(ca, ph, indexing="ij")
    sa = np.sqrt(1.0 - CA ** 2)
    d = (CA[..., None] * axis + sa[..., None] * (np.cos(PH)[..., None] * u + np.sin(PH)[..., None] * v)).reshape(-1, 3)
    oc = p - LIGHT_C
    b = d @ oc
    t = -b - np.sqrt(np.maximum(b * b - oc @ oc + LIGHT_R ** 2, 0.0))
    n = (p + t[:, None] * d - LIGHT_C) / LIGHT_R
    le = LIGHT_E.astype(np.float64) * env_lookup(tex[0], n)
    cos = np.maximum(d @ nrm, 0.0)
    dw = (1.0 - cmax) * 2.0 * np.pi / (nq * nq)
    return (le * cos[:, None]).sum(0) * dw


@pytest.mark.parametrize("ls", [1, 0])
def test_irradiance_under_a_textured_light_is_the_cap_integral(ectx, ls):
    """With the lookup at -n or at the sampled direction the receiver would see B (about 1/10 of A) instead of A."""
    sph, mats, cam, em = _scene([LIGHT_C, (0.0, -GROUND_R, 0.0)], [LIGHT_R, GROUND_R], [F.LAMBERT, F.LAMBERT],
                                [(0, 0, 0), (1, 1, 1)], [LIGHT_E, (0, 0, 0)])
    tex = _half_texture()
    ectx.set_option("light_sampling", ls)
    ectx.set_scene(sph, mats, cam, em)
    ectx.set_environment(np.zeros((4, 8, 3), np.float32))
    ectx.set_emission_textures(tex, [0, -1])
    copies = 1 << 15
    for x in (0.0, 1.3, 2.6):
        y = GROUND_R * np.cos(np.arcsin(x / GROUND_R)) - GROUND_R
        pt = np.concatenate([[x, y, 0.0], np.array([x, y + GROUND_R, 0.0]) / GROUND_R]).astype(np.float32)
        p, n = pt[:3].astype(np.float64), pt[3:].astype(np.float64)       # the point and normal as the kernel gets them
        want = _cap_integral(p, n, tex)
        pts = np.tile(pt, (copies, 1))
        out, _ = ectx.trace_irradiance(pts, np.ones(copies, np.int32), spp=16 if ls else 64)
        e = out[:, :3].astype(np.float64)
        mean, se = e.mean(0), e.std(0) / np.sqrt(copies)
        assert (np.abs(mean - want) < 5.0 * se + 1e-6 * want).all(), (ls, x, mean, want, se)
        b_only = _cap_integral(p, n, np.broadcast_to(TEX_B, tex.shape))
        assert (np.abs(b_only - want) > 50.0 * se).all(), (x, b_only, want, se)     # the test can tell A from B


# ---- 3. a constant texture is the scaled emission, bit for bit --------------------------------------------------
C_EMIT = np.float32([0.7, 1.3, 0.45])
C_ALB = np.float32([0.7, 0.55, 0.3])


def _emissive_vs_scaled(ctx, scene, w, h, variants=(-1, 3, 9), albedo=False):
    s, m, c, em = scene
    assert (m["emissive"] != 0).any()
    ctx.set_option("fast_kform", 0)
    ctx.set_scene(s, m, c, em)
    if albedo:
        ctx.set_textures(_const_layers(C_ALB), np.zeros(len(s), np.int32))
    ctx.set_emission_textures(_const_layers(C_EMIT), np.zeros(len(s), np.int32))
    got = _every_call(ctx, w, h, c, s, variants)
    ctx.set_emission_textures(None)
    m2 = m.copy()
    m2["emissive"] = (m["emissive"].astype(np.float32) * C_EMIT).astype(np.float32)
    ctx.set_scene(s, m2, c, em)
    ref = _every_call(ctx, w, h, c, s, variants)
    for k in ref:
        (ga, gr), (ra, rr) = got[k], ref[k]
        assert gr == rr, (k, gr, rr)
        ga, ra = np.asarray(ga), np.asarray(ra)
        assert ga.dtype == ra.dtype and ga.shape == ra.shape, k
        assert ga.tobytes() == ra.tobytes(), (k, int((ga.view(np.uint32) != ra.view(np.uint32)).sum()))
    ctx.set_textures(None)


@pytest.mark.parametrize("ls", [1, 0])
def test_constant_texture_is_the_scaled_emission_bitwise(ectx, ls):
    ectx.set_option("light_sampling", ls)
    _emissive_vs_scaled(ectx, scenes.reference_scene(64, 36), 64, 36)


def test_constant_texture_under_a_sampled_map_bitwise(ectx):
    ectx.set_environment(np.random.default_rng(6).uniform(0.0, 3.0, (16, 32, 3)).astype(np.float32))
    ectx.set_option("environment_sampling", 1)
    _emissive_vs_scaled(ectx, scenes.reference_scene(64, 36), 64, 36)


def test_constant_texture_on_a_big_scene_bitwise(ectx):
    _emissive_vs_scaled(ectx, scenes.stress_scene(48, 27), 48, 27, variants=(3, 9))
    ectx.set_emission_textures(_const_layers(C_EMIT), [0])
    _draw(ectx, 48, 27)
    assert ectx.last_kernels() == ["k_fast_queue<768, 1, 0>"], ectx.last_kernels()


def test_constant_albedo_and_emission_textures_together_bitwise(ectx):
    """Both products at once: the albedo-textured scene with emission textures against the same with emission scaled."""
    _emissive_vs_scaled(ectx, scenes.reference_scene(64, 36), 64, 36, albedo=True)


def corridor_scene(w=48, h=27):
    """Two facing emissive mirrors (rough Metal, radius 1000, 2 apart) around the camera, an emissive glass ball and an
    emissive Lambert ball between them: most camera paths bounce between the mirrors until the depth cap, on an
    emitter; rough reflections that go under the surface end there (Metal absorbed), and the glass ball's failed
    scatters end on it."""
    R = 1000.0
    centres = [(0.0, 0.0, -R - 1.0), (0.0, 0.0, R + 1.0), (0.3, 0.0, -0.4), (-0.3, 0.1, 0.4)]
    radii = [R, R, 0.15, 0.12]
    types = [F.METAL, F.METAL, F.DIELECTRIC, F.LAMBERT]
    albedo = [(0.9, 0.85, 0.8), (0.8, 0.9, 0.85), (1, 1, 1), (0.5, 0.5, 0.5)]
    emission = [(0.2, 0.1, 0.05), (0.05, 0.1, 0.2), (0.3, 0.2, 0.1), (2.0, 1.0, 0.5)]
    sph, mats, _c, em = _scene(centres, radii, types, albedo, emission, rough=0.15, ri=1.5)
    cam = scenes.make_camera((0.0, 0.0, 0.0), (0.05, 0.02, -1.0), (0, 1, 0), 30.0, w / h, 0.0, 1.0)
    return sph, mats, cam, em


@pytest.mark.parametrize("ls", [1, 0])
def test_constant_texture_in_a_mirror_corridor_bitwise(ectx, ls):
    ectx.set_option("light_sampling", ls)
    _emissive_vs_scaled(ectx, corridor_scene(), 48, 27, variants=(-1,))


def test_corridor_paths_reach_the_depth_cap():
    """Most corridor paths reach the cap: a float64 mirror walk (roughness 0) of the camera rays stays between the
    mirrors for TPT_MAX_DEPTH = 10 bounces."""
    sph, _m, cam, _em = corridor_scene()
    rays = scenes.camera_rays(cam, 48, 27).astype(np.float64)
    o, d = rays[:, :3], rays[:, 3:]
    alive = np.ones(len(o), bool)
    for _ in range(10):
        best_t = np.full(len(o), np.inf)
        best_i = np.full(len(o), -1)
        for i in range(2):
            c, r = sph["center"][i].astype(np.float64), float(sph["radius"][i])
            oc = o - c
            b = (oc * d).sum(1)
            disc = b * b - (oc * oc).sum(1) + r * r
            t = -b - np.sqrt(np.maximum(disc, 0.0))
            t = np.where(t > 1e-3, t, -b + np.sqrt(np.maximum(disc, 0.0)))
            ok = (disc > 0) & (t > 1e-3) & (t < best_t)
            best_t[ok], best_i[ok] = t[ok], i
        alive &= best_i >= 0
        p = o + best_t[:, None] * d
        n = (p - sph["center"][np.maximum(best_i, 0)]) / sph["radius"][np.maximum(best_i, 0)][:, None]
        d = d - 2.0 * (d * n).sum(1, keepdims=True) * n
        o = p
    assert alive.mean() > 0.8, alive.mean()


# ---- 4. the estimators agree on a real scene -----------------------------------------------------------------------
def _checker(w=32, h=16, lo=0.1, hi=1.9):
    ii, jj = np.meshgrid(np.arange(w) // 4, np.arange(h) // 4)
    v = np.where((ii + jj) % 2 == 0, hi, lo).astype(np.float32)
    return np.repeat(v[None, :, :, None], 3, axis=3)


def test_checker_emitters_converge_with_light_sampling_on_and_off(ectx):
    """The per-first-hit-sphere means of light sampling on and off agree within 5 standard errors (estimated from the
    spread across frames). With the untextured emission in the cones the lit spheres near the emitters would differ."""
    w, h, spp, nf = 64, 36, 32, 24
    s, m, c, em = scenes.reference_scene(w, h)
    layers = np.where((m["emissive"] != 0).any(1), 0, -1).astype(np.int32)
    ectx.set_scene(s, m, c, em)
    ids = torch.zeros((h, w), dtype=torch.int32, device="cuda")
    ectx.set_spp(1)
    ectx.draw_aovs(0, 1, w, h, ids=ids)
    ids = ids.cpu().numpy().ravel()
    bins = [i for i in np.unique(ids) if (ids == i).sum() >= 20]
    means = {}
    for ls in (1, 0):
        ectx.set_option("light_sampling", ls)
        ectx.set_scene(s, m, c, em)
        ectx.set_emission_textures(_checker(), layers)
        per = []
        for f in range(nf):
            img, _ = _draw(ectx, w, h, spp, frame=f)
            rgb = img[..., :3].reshape(-1, 3).astype(np.float64)
            per.append([rgb[ids == b].mean(0) for b in bins])
        per = np.array(per)                               # frames x bins x 3
        means[ls] = (per.mean(0), per.std(0, ddof=1) / np.sqrt(nf))
    (on, se_on), (off, se_off) = means[1], means[0]
    z = np.abs(on - off) / np.maximum(np.hypot(se_on, se_off), 1e-9)
    assert (z < 5.0).all(), (float(z.max()), bins[int(np.argmax(z.max(1)))])


# ---- 5. no change where they are not set ---------------------------------------------------------------------------
def _same(a, b):
    for k in b:
        (ga, gr), (ra, rr) = a[k], b[k]
        assert gr == rr, (k, gr, rr)
        assert np.asarray(ga).tobytes() == np.asarray(ra).tobytes(), k


def test_clearing_restores_a_context_that_never_had_emission_textures(libs, ectx):
    w, h = 48, 27
    s, m, c, em = scenes.reference_scene(w, h)
    fresh = libs.Context(0)
    try:
        fresh.set_option("fast_kform", 0)
        fresh.set_scene(s, m, c, em)
        ref = _every_call(fresh, w, h, c, s, (-1, 3, 9))
    finally:
        fresh.close()
    ectx.set_option("fast_kform", 0)
    ectx.set_scene(s, m, c, em)
    ectx.set_emission_textures(_const_layers(C_EMIT), np.zeros(len(s), np.int32))
    ectx.set_emission_textures(None)
    _same(_every_call(ectx, w, h, c, s, (-1, 3, 9)), ref)


def test_aovs_ignore_emission_textures(ectx):
    w, h = 48, 27
    s, m, c, em = scenes.reference_scene(w, h)
    ectx.set_scene(s, m, c, em)
    rays = scenes.camera_rays(c, w, h)

    def aovs():
        out = [t.cpu().numpy() for t in (torch.zeros((h, w, 4), device="cuda"), torch.zeros((h, w, 4), device="cuda"),
                                         torch.zeros((h, w), dtype=torch.int32, device="cuda"))]
        a, n, i = (torch.from_numpy(x).cuda() for x in out)
        ectx.draw_aovs(0, 2, w, h, a, n, i)
        (ta, tn, ti), _ = ectx.trace_aovs(rays)
        return [x.cpu().numpy().tobytes() for x in (a, n, i)] + [ta.tobytes(), tn.tobytes(), ti.tobytes()]

    ref = aovs()
    ectx.set_emission_textures(np.random.default_rng(3).uniform(0, 2, (2, 8, 16, 3)).astype(np.float32),
                               np.arange(len(s)) % 2)
    assert aovs() == ref


def test_layers_without_emission_leave_albedo_textured_calls_alone(ectx):
    """Albedo-textured calls with emission textures that bind no emitter (layers only on spheres whose emission is
    zero, or no layer at all) give the bits of the same calls without emission textures: a zero emission stays dark."""
    w, h = 48, 27
    s, m, c, em = scenes.reference_scene(w, h)
    rng = np.random.default_rng(4)
    ectx.set_option("fast_kform", 0)
    ectx.set_scene(s, m, c, em)
    ectx.set_textures(rng.uniform(0, 1, (2, 8, 16, 3)).astype(np.float32), np.arange(len(s)) % 3 - 1)
    ref = _every_call(ectx, w, h, c, s, (-1, 3, 9))
    dark = np.where((m["emissive"] != 0).any(1), -1, 0).astype(np.int32)
    for layers in (dark, np.full(len(s), -1, np.int32)):
        ectx.set_emission_textures(rng.uniform(0, 5, (1, 8, 16, 3)).astype(np.float32), layers)
        _same(_every_call(ectx, w, h, c, s, (-1, 3, 9)), ref)


# ---- 6. routing, refusals, lifetime --------------------------------------------------------------------------------
@pytest.mark.parametrize("ls", [1, 0])
def test_emission_textured_calls_run_the_texture_instances(ectx, ls):
    w, h = 64, 36
    ectx.set_option("light_sampling", ls)
    s, m, c, em = scenes.reference_scene(w, h)
    ectx.set_scene(s, m, c, em)
    ectx.set_emission_textures(_const_layers(C_EMIT), np.zeros(len(s), np.int32))
    for v in (-1, 3, 9):
        ectx.set_option("fast_variant", v)
        _draw(ectx, w, h)
        assert _texture_kernels_only(ectx), (v, ectx.last_kernels())
    host = np.zeros((h, w, 4), np.float32)
    ectx.set_option("fast_variant", -1)
    ectx.draw(0, 1, w, h, host, flags=0, mode=MODE_FAST)
    assert _texture_kernels_only(ectx), ectx.last_kernels()
    rays = scenes.camera_rays(c, w, h)
    for call in (lambda: ectx.trace_rays(rays, spp=2), lambda: ectx.draw_samples(0, w, h, spp=2),
                 lambda: ectx.trace_samples(rays, spp=2),
                 lambda: ectx.trace_irradiance(np.concatenate([np.zeros((8, 3)), np.tile([0, 1, 0], (8, 1))], 1)
                                               .astype(np.float32), spp=2)):
        call()
        assert _texture_kernels_only(ectx), ectx.last_kernels()
    for v in (0, 1, 2, 4, 5, 6, 7, 8):
        ectx.set_option("fast_variant", v)
        with pytest.raises(TptError, match=f"emission textures are set \\(tpt_set_emission_textures\\), and "
                                           f"fast_variant {v} does not"):
            _draw(ectx, w, h)
    ectx.set_option("fast_variant", -1)
    for mode in (MODE_EXACT, MODE_REFGPU, MODE_REFGPU_FAST):
        with pytest.raises(TptError, match="emission textures are set, and only TPT_MODE_FAST draws use them"):
            _draw(ectx, w, h, 1, mode=mode)
    ectx.set_emission_textures(None)
    for mode in (MODE_EXACT, MODE_REFGPU_FAST):
        _img, r = _draw(ectx, w, h, 1, mode=mode)
        assert r > 0


def test_emission_textures_set_during_a_draw_are_not_seen_by_it(ectx):
    w, h, spp = 1920, 1080, 16
    s, m, c, em = scenes.reference_scene(w, h)
    ectx.set_scene(s, m, c, em)
    ectx.set_spp(spp)
    every = np.zeros(len(s), np.int32)
    a, b = _const_layers([1.0, 1.0, 1.0]), _const_layers([0.0, 0.0, 0.0])
    bufs = [torch.zeros((h, w, 4), dtype=torch.float32, device="cuda") for _ in range(2)]
    torch.cuda.synchronize()
    ectx.set_emission_textures(a, every)
    ectx.draw(0, 1, w, h, bufs[0], flags=0, mode=MODE_FAST, want_rays=False)
    ectx.set_emission_textures(b, every)
    ectx.draw(0, 1, w, h, bufs[1], flags=0, mode=MODE_FAST, want_rays=False)
    torch.cuda.synchronize()
    got = [t.cpu().numpy() for t in bufs]
    ectx.set_emission_textures(a, every)
    ref_a, _ = _draw(ectx, w, h)
    ectx.set_emission_textures(b, every)
    ref_b, _ = _draw(ectx, w, h)
    assert rel_l2(got[0], ref_a) < 1e-5, rel_l2(got[0], ref_a)
    assert rel_l2(got[1], ref_b) < 1e-5, rel_l2(got[1], ref_b)
    assert rel_l2(ref_b, ref_a) > 0.1


def test_emission_textures_survive_set_scene_and_take_cuda_tensors(ectx):
    w, h = 96, 54
    rng = np.random.default_rng(8)
    tex = rng.uniform(0.0, 2.0, (3, 16, 32, 3)).astype(np.float32)
    s, mats, c, em = scenes.reference_scene(w, h)
    layers = rng.integers(-1, 3, len(s)).astype(np.int32)
    layers[em] = np.arange(len(em)) % 3
    ectx.set_scene(s, mats, c, em)
    ectx.set_emission_textures(tex, layers)
    ref, rref = _draw(ectx, w, h, 1)
    s2 = s.copy()
    s2["center"][1, 1] += 0.5
    ectx.set_scene(s2, mats, c, em)
    other, _ = _draw(ectx, w, h, 1)
    assert bits_differ(other, ref).any()
    ectx.set_scene(s, mats, c, em)
    img, rimg = _draw(ectx, w, h, 1)
    assert rimg == rref and not bits_differ(img, ref).any()
    ectx.set_emission_textures(None)
    plain, _ = _draw(ectx, w, h, 1)
    assert bits_differ(plain, ref).any()
    rgba = torch.from_numpy(np.concatenate([tex, np.full(tex.shape[:3] + (1,), np.nan, np.float32)], 3)).cuda()
    ectx.set_emission_textures(rgba, torch.from_numpy(layers))
    img, _ = _draw(ectx, w, h, 1)
    assert not bits_differ(img, ref).any()
    ectx.set_emission_textures(torch.from_numpy(tex).cuda(), layers)
    img, _ = _draw(ectx, w, h, 1)
    assert not bits_differ(img, ref).any()


def test_emission_and_albedo_textures_are_independent(ectx):
    """Setting or clearing one set leaves the other in place."""
    w, h = 48, 27
    s, m, c, em = scenes.reference_scene(w, h)
    rng = np.random.default_rng(5)
    alb = rng.uniform(0, 1, (1, 8, 16, 3)).astype(np.float32)
    emi = rng.uniform(0, 2, (2, 4, 8, 3)).astype(np.float32)
    ectx.set_scene(s, m, c, em)
    ectx.set_textures(alb, np.zeros(len(s), np.int32))
    ectx.set_emission_textures(emi, np.arange(len(s)) % 2)
    both, _ = _draw(ectx, w, h, 1)
    ectx.set_textures(None)
    only_e, _ = _draw(ectx, w, h, 1)
    ectx.set_textures(alb, np.zeros(len(s), np.int32))
    again, _ = _draw(ectx, w, h, 1)
    ectx.set_emission_textures(None)
    only_a, _ = _draw(ectx, w, h, 1)
    assert not bits_differ(again, both).any()
    assert bits_differ(only_e, both).any() and bits_differ(only_a, both).any()


def _raw_set(ctx, ptr, w, h, n, layers, on_dev, num=None):
    arr = np.ascontiguousarray(layers, np.int32)
    rc = ctx._L.tpt_set_emission_textures(ctx._h, ctypes.c_void_p(ptr), w, h, n, arr.ctypes.data if arr.size else None,
                                          len(arr) if num is None else num, on_dev)
    return rc, ctx._L.tpt_last_error(ctx._h).decode()


def test_bad_emission_textures_are_refused_and_leave_them_as_they_were(ectx):
    w, h = 48, 27
    s, m, c, em = scenes.reference_scene(w, h)
    ectx.set_scene(s, m, c, em)
    good = np.random.default_rng(2).uniform(0, 2, (2, 8, 16, 3)).astype(np.float32)
    layers = np.arange(len(s)) % 3 - 1
    ectx.set_emission_textures(good, layers)
    ref, _ = _draw(ectx, w, h, 1)
    host = np.ones((2, 8, 16, 4), np.float32)
    for (tw, th, tn), text in (((0, 8, 2), "width, height and layers must be >= 1"),
                               ((16, 8, 0), "width, height and layers must be >= 1"),
                               ((65536, 16384, 2), "below 2\\^31")):
        rc, err = _raw_set(ectx, host.ctypes.data, tw, th, tn, [0], 0)
        assert rc != 0 and err.startswith("tpt_set_emission_textures: ") and re.search(text, err), (tw, th, tn, err)
    rc, err = _raw_set(ectx, host.ctypes.data, 16, 8, 2, [0], 0, num=-1)
    assert rc != 0 and "numSpheres must be >= 0" in err, err
    rc, err = _raw_set(ectx, host.ctypes.data, 16, 8, 2, [0, 2], 0)
    assert rc != 0 and re.search(r"sphereLayers\[1\] = 2 is outside \[-1, 2\)", err), err
    dev = torch.ones((2 * 8 * 16 + 1, 4), dtype=torch.float32, device="cuda")
    rc, err = _raw_set(ectx, dev.data_ptr() + 4, 16, 8, 2, [0], 1)
    assert rc != 0 and "16-byte aligned" in err, err
    for (l, y, x, ch), v in (((0, 3, 5, 0), np.nan), ((1, 7, 15, 2), np.inf), ((1, 5, 1, 2), -0.0)):
        bad = host.copy()
        bad[l, y, x, ch] = v
        want = f"tpt_set_emission_textures: texel of layer {l} \\(x {x}, y {y}\\) has {'RGB'[ch]} = "
        rc, err = _raw_set(ectx, bad.ctypes.data, 16, 8, 2, [0], 0)
        assert rc != 0 and re.search(want, err), (v, err)
        dbad = torch.from_numpy(bad).cuda()
        torch.cuda.synchronize()
        rc, err = _raw_set(ectx, dbad.data_ptr(), 16, 8, 2, [0], 1)
        assert rc != 0 and re.search(want, err), (v, "device", err)
    img, _ = _draw(ectx, w, h, 1)
    assert not bits_differ(img, ref).any()
