"""Sphere albedo textures (tpt_set_textures, Context.set_textures) on the GPU.

1. Lookup through the AOVs: rays aimed at chosen normals of textured spheres report albedo x the float64 lookup of their
   layer (env_lookup, the pinned lat-long mapping) at the seam, the poles, on 1 x 1 and non-square layers, and for a
   one-hot texel at its centre; spheres with layer -1 or ids past the table keep their albedo.
2. Deterministic furnace (scene A) through trace_rays: a textured receiver returns exactly albedo * T(n) * sky per
   sample for Lambert (light sampling on and off) and Metal, with 2 + K or 2 rays per sample.
3. A constant texture c on every sphere is, bit for bit and ray for ray, the untextured scene with albedo fl32(a * c),
   through every fast call, with light sampling on and off, under a sampled map, and on a scene past 64 KB of blob.
4. A texture on a glass sphere changes no bit.
5. Light-sampled vertices see the texture: a checker-board ground converges to the same image with light sampling on and
   off.
6. Routing: textured calls run the reference-form slab-queue instances; other variants and the parity modes are refused.
7. Lifetime: textures set while a draw is in flight are not seen by it; clearing restores a context that never had
   textures; textures survive set_scene; CUDA tensors; bad texels refused on host and device, keeping the old textures."""
import ctypes
import re

import numpy as np
import pytest
import torch

import furnace as F
from conftest import bits_differ, rel_l2
from test_gpu_environment import env_lookup, lat_long_dir, lookup_tolerance
from toypathtracer_b200 import (MATERIAL_DTYPE, MODE_EXACT, MODE_FAST, MODE_REFGPU, MODE_REFGPU_FAST, SPHERE_DTYPE,
                                TptError, kFlagProgressive, scenes)

pytestmark = pytest.mark.gpu

TEX_KERNELS = ("k_fast_queue<128, 6, 0>", "k_fast_queue<768, 1, 0>", "k_fast_rays<128, 6, 0>", "k_fast_rays<768, 1, 0>",
               "k_fast_samples<128, 6, 0,", "k_fast_samples<768, 1, 0,",
               "k_fast_queue_nolight<128, 6, 0>", "k_fast_queue_nolight<768, 1, 0>", "k_fast_rays_nolight<128, 6, 0>",
               "k_fast_rays_nolight<768, 1, 0>", "k_fast_samples_nolight<128, 6, 0,", "k_fast_samples_nolight<768, 1, 0,")


@pytest.fixture
def tctx(gpu_ctx):
    yield gpu_ctx
    gpu_ctx.set_textures(None)
    gpu_ctx.set_environment(None)
    for k, v in (("fast_variant", -1), ("fast_kform", 2), ("mitsuba_compare", 0), ("light_sampling", 1),
                 ("environment_sampling", 0)):
        gpu_ctx.set_option(k, v)
    gpu_ctx.set_spp(4)


def _draw(ctx, w, h, spp=None, frame=0, frames=1, flags=0, mode=MODE_FAST, prev=None):
    if spp is not None:
        ctx.set_spp(spp)
    buf = torch.zeros((h, w, 4), dtype=torch.float32, device="cuda") if prev is None else prev.clone()
    rays = ctx.draw(frame, frames, w, h, buf, flags=flags, mode=mode)
    return buf.cpu().numpy(), rays


def _const_layers(c, n=1, w=5, h=3):
    return np.broadcast_to(np.float32(c), (n, h, w, 3)).copy()


# ---- 1. the lookup through the AOVs ------------------------------------------------------------------------------
ALB = np.float32([[0.9, 0.7, 0.5], [0.6, 0.8, 0.4], [0.5, 0.5, 0.9], [1.0, 1.0, 1.0], [0.3, 0.6, 0.9]])
TYPES = [F.LAMBERT, F.METAL, F.LAMBERT, F.DIELECTRIC, F.LAMBERT]
CENTRES = np.array([[0.0, 0.0, -6.0], [4.0, 0.0, -6.0], [-4.0, 0.0, -6.0], [0.0, 4.0, -6.0], [0.0, -4.0, -6.0]])
LAYER_OF = np.array([1, 0, -1, 1], np.int32)      # sphere 4 lies past the table: untextured


def aov_scene():
    sph = np.zeros(len(CENTRES), SPHERE_DTYPE)
    mats = np.zeros(len(CENTRES), MATERIAL_DTYPE)
    for i, c in enumerate(CENTRES):
        sph[i] = (c, 1.0, 1.0)
        mats[i] = (TYPES[i], ALB[i], (0, 0, 0), 0.3, 1.5)
    return sph, mats, F.furnace_camera(8, 8), np.zeros(0, np.int32)


def aimed_rays(sphere, normals):
    """Rays that hit sphere `sphere` (radius 1) head-on at the unit normals, and those normals in float64 from the
    float32 rays (the ray through the hit point, solved in float64)."""
    c = CENTRES[sphere]
    n = np.asarray(normals, np.float64)
    rays = np.concatenate([c + 2.5 * n, -n], 1).astype(np.float32)
    o, d = rays[:, :3].astype(np.float64), rays[:, 3:].astype(np.float64)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    oc = o - c
    b = (oc * d).sum(1)
    t = -b - np.sqrt(b * b - (oc * oc).sum(1) + 1.0)
    hit = o + t[:, None] * d - c
    return rays, hit / np.linalg.norm(hit, axis=1, keepdims=True)


def _normals(w, h, rng):
    d = rng.normal(size=(400, 3))
    dirs = [d / np.linalg.norm(d, axis=1, keepdims=True)]
    vs = rng.uniform(0, h, 6)
    for u in (0.0, 1e-4, 0.5, w - 0.5, w - 1e-4, w):                   # the phi = +-pi seam, both sides
        dirs.append(lat_long_dir(np.full(6, u), vs, w, h))
    us = rng.uniform(0, w, 6)
    for v in (0.0, 1e-4, 0.5, h - 0.5, h - 1e-4, h):                   # both poles
        dirs.append(lat_long_dir(us, np.full(6, v), w, h))
    ii, jj = np.meshgrid(np.arange(w) + 0.5, np.arange(h) + 0.5)
    dirs.append(lat_long_dir(ii.ravel(), jj.ravel(), w, h))              # every texel centre
    return np.concatenate(dirs)


@pytest.mark.parametrize("size", [(64, 16), (1, 1), (7, 24)])
def test_aov_albedo_is_the_lookup(tctx, size):
    w, h = size
    rng = np.random.default_rng(w * 100 + h)
    layers = rng.uniform(0.0, 2.0, (2, h, w, 3)).astype(np.float32)
    tctx.set_scene(*aov_scene())
    tctx.set_textures(layers, LAYER_OF)
    for sphere in range(len(CENTRES)):
        rays, n = aimed_rays(sphere, _normals(w, h, rng))
        (alb, nrm, ids), traced = tctx.trace_aovs(rays)
        assert traced == len(rays) and (ids == sphere).all(), (sphere, np.unique(ids))
        # the lookup's direction is the normal the AOV reports ((pos - centre) / r in float32, as path_step has it): the
        # sweep's distance error moves it further than the lookup's own rounding
        assert np.abs(nrm[:, :3] - n).max() < 1e-4
        n = nrm[:, :3].astype(np.float64)
        layer = LAYER_OF[sphere] if sphere < len(LAYER_OF) else -1
        if layer < 0:
            assert (alb[:, :3] == ALB[sphere]).all(), sphere
            continue
        want = ALB[sphere].astype(np.float64) * env_lookup(layers[layer], n)
        tol = lookup_tolerance(layers[layer], n)[:, None] * ALB[sphere] + 2.0 ** -21 * np.abs(want) + 1e-7
        bad = (np.abs(alb[:, :3] - want) > tol).any(1)
        assert not bad.any(), (size, sphere, int(bad.sum()), n[bad][:3], alb[bad][:3], want[bad][:3])
        if w == h == 1:
            assert (alb[:, :3] == (ALB[sphere] * layers[layer, 0, 0]).astype(np.float32)).all()


def test_one_hot_texel_orientation_and_row_order(tctx):
    """Texel (2, 1) of an 8 x 4 layer is lit: the normal through its centre sees it, every other texel centre sees
    nothing. Its centre lies at phi < 0, left of the -z centre column (toward -x)."""
    w, h = 8, 4
    layer = np.zeros((1, h, w, 3), np.float32)
    layer[0, 1, 2] = (1.0, 2.0, 3.0)
    tctx.set_scene(*aov_scene())
    tctx.set_textures(layer, [0])
    ii, jj = np.meshgrid(np.arange(w) + 0.5, np.arange(h) + 0.5)
    rays, _n = aimed_rays(0, lat_long_dir(ii.ravel(), jj.ravel(), w, h))
    (alb, _nrm, _ids), _ = tctx.trace_aovs(rays)
    np.testing.assert_allclose(alb[:, :3].reshape(h, w, 3), ALB[0] * layer[0], atol=1e-4)
    assert lat_long_dir(2.5, 1.5, w, h)[0] < 0


# ---- 2. the deterministic furnace through trace_rays ---------------------------------------------------------------
@pytest.mark.parametrize("metal,ls", [(False, 1), (False, 0), (True, 1)])
def test_furnace_receiver_is_albedo_times_lookup(tctx, metal, ls):
    w, h, spp, K = 40, 24, 4, 3
    rng = np.random.default_rng(3)
    layer = rng.uniform(0.2, 1.0, (1, 8, 16, 3)).astype(np.float32)
    tctx.set_option("mitsuba_compare", 1)        # constant sky, and the Metal receiver's zero roughness
    tctx.set_option("light_sampling", ls)
    s, m, c, em = F.furnace_scene(w, h, K, metal)
    tctx.set_scene(s, m, c, em)
    tctx.set_textures(layer, [0])
    rays = scenes.camera_rays(c, w, h)
    out, traced = tctx.trace_rays(rays, spp=spp)
    assert traced == len(rays) * spp * F.furnace_rays_per_sample(m, K, bool(ls)), (traced, len(rays))
    o, d = rays[:, :3].astype(np.float64), rays[:, 3:].astype(np.float64)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    b = (o * d).sum(1)
    t = -b - np.sqrt(b * b - (o * o).sum(1) + F.RECEIVER_R ** 2)
    n = (o + t[:, None] * d) / F.RECEIVER_R
    scale = m["albedo"][0].astype(np.float64) * F.MITSUBA_SKY
    want = scale * env_lookup(layer[0], n)
    tol = lookup_tolerance(layer[0], n, eps=1e-5)[:, None] * scale + 2.0 ** -19 * np.abs(want)
    bad = (np.abs(out[:, :3] - want) > tol).any(1)
    assert not bad.any(), (metal, ls, int(bad.sum()), out[bad][:3], want[bad][:3])


# ---- 3. a constant texture is the albedo, bit for bit -------------------------------------------------------------
C_TEX = np.float32([0.7, 0.55, 0.3])


def _every_call(ctx, w, h, cam, sph, variants, spp=1):
    """Outputs and ray counts of every fast call on one scene: draws (`variants`; progressive frames, one call each),
    trace_rays, trace_irradiance, draw_samples, trace_samples, draw_aovs, trace_aovs. One sample per output and call:
    several samples of one output are summed by atomic adds in no fixed order, which is not bitwise reproducible."""
    res = {}
    ctx.set_spp(1)
    for v in variants:
        ctx.set_option("fast_variant", v)
        img, r = None, []
        for f in range(3):
            img, rf = _draw(ctx, w, h, frame=f, flags=kFlagProgressive, prev=None if img is None else torch.from_numpy(img).cuda())
            r.append(rf)
        res[f"draw{v}"] = (img, r)
    ctx.set_option("fast_variant", -1)
    rays = scenes.camera_rays(cam, w, h, seed=5)
    res["rays"] = ctx.trace_rays(rays, spp=spp)
    rng = np.random.default_rng(9)
    ids = rng.integers(0, len(sph), 512).astype(np.int32)
    nrm = rng.normal(size=(512, 3))
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    pts = np.concatenate([sph["center"][ids] + sph["radius"][ids][:, None] * nrm, nrm], 1).astype(np.float32)
    res["irr"] = ctx.trace_irradiance(pts, ids, spp=spp)
    (s4, q4), r = ctx.draw_samples(0, w, h, spp=spp)
    res["dsamples"] = (np.concatenate([s4.cpu().numpy(), q4.cpu().numpy()]), r)
    (s4, q4), r = ctx.trace_samples(rays, spp=spp)
    res["tsamples"] = (np.concatenate([s4, q4]), r)
    alb, nm, ii = (torch.zeros((h, w, 4), device="cuda"), torch.zeros((h, w, 4), device="cuda"),
                   torch.zeros((h, w), dtype=torch.int32, device="cuda"))
    r = ctx.draw_aovs(0, 2, w, h, alb, nm, ii)
    res["daovs"] = (np.concatenate([alb.cpu().numpy().ravel(), nm.cpu().numpy().ravel(), ii.cpu().numpy().ravel()]), r)
    (a, nn, i2), r = ctx.trace_aovs(rays)
    res["taovs"] = (np.concatenate([a.ravel(), nn.ravel(), i2.ravel()]), r)
    return res


def _textured_vs_scaled(ctx, scene, w, h, variants=(-1, 3, 9)):
    s, m, c, em = scene
    ctx.set_option("fast_kform", 0)                # the AOV kernel's sweep form follows it; the trace calls run form 0 anyway
    ctx.set_scene(s, m, c, em)
    ctx.set_textures(_const_layers(C_TEX), np.zeros(len(s), np.int32))
    got = _every_call(ctx, w, h, c, s, variants)
    ctx.set_textures(None)
    m2 = m.copy()
    m2["albedo"] = (m["albedo"].astype(np.float32) * C_TEX).astype(np.float32)
    ctx.set_scene(s, m2, c, em)
    ref = _every_call(ctx, w, h, c, s, variants)
    for k in ref:
        (ga, gr), (ra, rr) = got[k], ref[k]
        assert gr == rr, (k, gr, rr)
        ga, ra = np.asarray(ga), np.asarray(ra)
        assert ga.dtype == ra.dtype and ga.shape == ra.shape, k
        assert ga.tobytes() == ra.tobytes(), (k, int((ga.view(np.uint32) != ra.view(np.uint32)).sum()))


@pytest.mark.parametrize("ls", [1, 0])
def test_constant_texture_is_the_scaled_albedo_bitwise(tctx, ls):
    tctx.set_option("light_sampling", ls)
    _textured_vs_scaled(tctx, scenes.reference_scene(64, 36), 64, 36)


def test_constant_texture_under_a_sampled_map_bitwise(tctx):
    tctx.set_environment(np.random.default_rng(6).uniform(0.0, 3.0, (16, 32, 3)).astype(np.float32))
    tctx.set_option("environment_sampling", 1)
    _textured_vs_scaled(tctx, scenes.reference_scene(64, 36), 64, 36)


def test_constant_texture_on_a_big_scene_bitwise(tctx):
    """Past 64 KB of blob the slab queue runs its 768-thread instance. (Untextured, the automatic variant of a scene
    of 4096 spheres swept in the reference form is the block wavefront: only the slab-queue variants are compared.)"""
    _textured_vs_scaled(tctx, scenes.stress_scene(48, 27), 48, 27, variants=(3, 9))
    tctx.set_textures(_const_layers(C_TEX), [0])
    _draw(tctx, 48, 27)
    assert tctx.last_kernels() == ["k_fast_queue<768, 1, 0>"], tctx.last_kernels()


# ---- 4. glass --------------------------------------------------------------------------------------------------------
def test_textured_glass_changes_nothing(tctx):
    w, h = 64, 36
    s, m, c, em = scenes.reference_scene(w, h)
    glass = np.nonzero(m["type"] == F.DIELECTRIC)[0]
    assert len(glass)
    tctx.set_option("fast_kform", 0)
    tctx.set_scene(s, m, c, em)
    ref, rref = _draw(tctx, w, h, 1)
    rays = scenes.camera_rays(c, w, h)
    tref, trref = tctx.trace_rays(rays, spp=1)
    layers = np.full(len(s), -1, np.int32)
    layers[glass] = 0
    tctx.set_textures(np.random.default_rng(1).uniform(0, 1, (1, 8, 16, 3)).astype(np.float32), layers)
    img, rimg = _draw(tctx, w, h, 1)
    tout, trout = tctx.trace_rays(rays, spp=1)
    assert rimg == rref and not bits_differ(img, ref).any()
    assert trout == trref and tout.tobytes() == tref.tobytes()


# ---- 5. light-sampled vertices see the texture -------------------------------------------------------------------
def _checker(w=64, h=32, lo=0.15, hi=1.0):
    ii, jj = np.meshgrid(np.arange(w) // 4, np.arange(h) // 4)
    v = np.where((ii + jj) % 2 == 0, hi, lo).astype(np.float32)
    return np.repeat(v[None, :, :, None], 3, axis=3)


def test_checker_ground_converges_with_light_sampling_on_and_off(tctx):
    """The ground (the largest sphere) under a checker-board, compared on the pixels whose first hit is the ground: with
    light sampling on the light cones carry the textured albedo, so both estimators converge to one image. With the
    untextured albedo in the cones the direct light on the dark squares would be ~6x too bright."""
    w, h, spp, nf = 96, 54, 128, 128
    s, m, c, em = scenes.reference_scene(w, h)
    ground = int(np.argmax(s["radius"]))
    layers = np.full(len(s), -1, np.int32)
    layers[ground] = 0
    tctx.set_scene(s, m, c, em)
    ids = torch.zeros((h, w), dtype=torch.int32, device="cuda")
    tctx.set_spp(1)
    tctx.draw_aovs(0, 1, w, h, ids=ids)
    mask = ids.cpu().numpy() == ground
    assert mask.sum() > 0.05 * w * h
    imgs = {}
    for ls in (1, 0):
        tctx.set_option("light_sampling", ls)
        tctx.set_scene(s, m, c, em)
        tctx.set_textures(_checker(), layers)
        a, _ = _draw(tctx, w, h, spp, frames=nf, flags=kFlagProgressive)
        full, _ = _draw(tctx, w, h, spp, frames=2 * nf, flags=kFlagProgressive)
        a, full = a[mask].astype(np.float64), full[mask].astype(np.float64)
        imgs[ls] = (full, rel_l2(a, 2.0 * full - a) / 2.0)     # the mean's own noise (the halves' spread / 2)
    (on, n_on), (off, n_off) = imgs[1], imgs[0]
    bound = 3.0 * np.hypot(n_on, n_off)
    assert rel_l2(on, off) < bound, (rel_l2(on, off), n_on, n_off)
    tctx.set_textures(None)
    tctx.set_option("light_sampling", 1)
    tctx.set_scene(s, m, c, em)
    plain, _ = _draw(tctx, w, h, spp, frames=2 * nf, flags=kFlagProgressive)
    assert rel_l2(on, plain[mask]) > 3.0 * bound        # the texture is visible at this noise level


# ---- 6. routing ----------------------------------------------------------------------------------------------------
def _texture_kernels_only(ctx):
    kinds = [k for k in ctx.last_kernels() if k.startswith("k_fast") and not k.startswith("k_fast_aov")]
    return bool(kinds) and all(k.startswith(TEX_KERNELS) for k in kinds)


@pytest.mark.parametrize("ls", [1, 0])
def test_textured_calls_run_the_reference_form_instances(tctx, ls):
    w, h = 64, 36
    tctx.set_option("light_sampling", ls)
    s, m, c, em = scenes.reference_scene(w, h)
    tctx.set_scene(s, m, c, em)
    tctx.set_textures(_const_layers(C_TEX), np.zeros(len(s), np.int32))
    for v in (-1, 3, 9):
        tctx.set_option("fast_variant", v)
        _draw(tctx, w, h)
        assert _texture_kernels_only(tctx), (v, tctx.last_kernels())
    host = np.zeros((h, w, 4), np.float32)            # a host buffer: no zero-copy store, the slab queue stages it
    tctx.set_option("fast_variant", -1)
    tctx.draw(0, 1, w, h, host, flags=0, mode=MODE_FAST)
    assert _texture_kernels_only(tctx), tctx.last_kernels()
    rays = scenes.camera_rays(c, w, h)
    for call in (lambda: tctx.trace_rays(rays, spp=2), lambda: tctx.draw_samples(0, w, h, spp=2),
                 lambda: tctx.trace_samples(rays, spp=2),
                 lambda: tctx.trace_irradiance(np.concatenate([np.zeros((8, 3)), np.tile([0, 1, 0], (8, 1))], 1)
                                               .astype(np.float32), spp=2)):
        call()
        assert _texture_kernels_only(tctx), tctx.last_kernels()
    for v in (0, 1, 2, 4, 5, 6, 7, 8):
        tctx.set_option("fast_variant", v)
        with pytest.raises(TptError, match=f"textures are set \\(tpt_set_textures\\), and fast_variant {v} does not"):
            _draw(tctx, w, h)
    tctx.set_option("fast_variant", -1)
    for mode in (MODE_EXACT, MODE_REFGPU, MODE_REFGPU_FAST):
        with pytest.raises(TptError, match="textures are set, and only TPT_MODE_FAST draws use them"):
            _draw(tctx, w, h, 1, mode=mode)
    tctx.set_textures(None)
    for v in (0, 4, 8):
        tctx.set_option("fast_variant", v)
        _img, rays_v = _draw(tctx, w, h)
        assert rays_v > 0
    tctx.set_option("fast_variant", -1)
    for mode in (MODE_EXACT, MODE_REFGPU, MODE_REFGPU_FAST):
        _img, r = _draw(tctx, w, h, 1, mode=mode)
        assert r > 0


# ---- 7. lifetime and refusals -------------------------------------------------------------------------------------
def test_textures_set_during_a_draw_are_not_seen_by_it(tctx):
    w, h, spp = 1920, 1080, 16
    s, m, c, em = scenes.reference_scene(w, h)
    tctx.set_scene(s, m, c, em)
    tctx.set_spp(spp)
    every = np.zeros(len(s), np.int32)
    a, b = _const_layers([1.0, 1.0, 1.0]), _const_layers([0.0, 0.0, 0.0])
    bufs = [torch.zeros((h, w, 4), dtype=torch.float32, device="cuda") for _ in range(2)]
    torch.cuda.synchronize()
    tctx.set_textures(a, every)
    tctx.draw(0, 1, w, h, bufs[0], flags=0, mode=MODE_FAST, want_rays=False)
    tctx.set_textures(b, every)
    tctx.draw(0, 1, w, h, bufs[1], flags=0, mode=MODE_FAST, want_rays=False)
    torch.cuda.synchronize()
    got = [t.cpu().numpy() for t in bufs]
    tctx.set_textures(a, every)
    ref_a, _ = _draw(tctx, w, h)
    tctx.set_textures(b, every)
    ref_b, _ = _draw(tctx, w, h)
    assert rel_l2(got[0], ref_a) < 1e-5, rel_l2(got[0], ref_a)
    assert rel_l2(got[1], ref_b) < 1e-5, rel_l2(got[1], ref_b)
    assert rel_l2(ref_b, ref_a) > 0.1


def test_clearing_restores_a_context_that_never_had_textures(libs, tctx):
    w, h = 96, 54
    s, m, c, em = scenes.reference_scene(w, h)
    fresh = libs.Context(0)
    try:
        fresh.set_scene(s, m, c, em)
        ref, rref = _draw(fresh, w, h, 1)
    finally:
        fresh.close()
    tctx.set_scene(s, m, c, em)
    tctx.set_textures(_const_layers(C_TEX), np.zeros(len(s), np.int32))
    tctx.set_textures(None)
    img, rimg = _draw(tctx, w, h, 1)
    assert rimg == rref and not bits_differ(img, ref).any()
    assert not any(k.startswith("k_fast_queue<128, 6, 0>") for k in tctx.last_kernels())


def test_textures_survive_set_scene_and_take_cuda_tensors(tctx):
    w, h = 96, 54
    rng = np.random.default_rng(8)
    tex = rng.uniform(0.0, 1.0, (3, 16, 32, 3)).astype(np.float32)
    s, mats, c, em = scenes.reference_scene(w, h)
    layers = rng.integers(-1, 3, len(s)).astype(np.int32)
    tctx.set_scene(s, mats, c, em)
    tctx.set_textures(tex, layers)
    ref, rref = _draw(tctx, w, h, 1)
    s2 = s.copy()
    s2["center"][1, 1] += 0.5
    tctx.set_scene(s2, mats, c, em)
    other, _ = _draw(tctx, w, h, 1)
    assert bits_differ(other, ref).any()
    tctx.set_scene(s, mats, c, em)
    img, rimg = _draw(tctx, w, h, 1)
    assert rimg == rref and not bits_differ(img, ref).any()
    tctx.set_textures(None)
    plain, _ = _draw(tctx, w, h, 1)
    assert bits_differ(plain, ref).any()
    rgba = torch.from_numpy(np.concatenate([tex, np.full(tex.shape[:3] + (1,), np.nan, np.float32)], 3)).cuda()
    tctx.set_textures(rgba, torch.from_numpy(layers))     # (L, H, W, 4) CUDA tensor, alpha ignored
    img, _ = _draw(tctx, w, h, 1)
    assert not bits_differ(img, ref).any()
    tctx.set_textures(torch.from_numpy(tex).cuda(), layers)
    img, _ = _draw(tctx, w, h, 1)
    assert not bits_differ(img, ref).any()


def _raw_set(ctx, ptr, w, h, n, layers, on_dev, num=None):
    arr = np.ascontiguousarray(layers, np.int32)
    rc = ctx._L.tpt_set_textures(ctx._h, ctypes.c_void_p(ptr), w, h, n, arr.ctypes.data if arr.size else None,
                                 len(arr) if num is None else num, on_dev)
    return rc, ctx._L.tpt_last_error(ctx._h).decode()


def test_bad_textures_are_refused_and_leave_the_textures_as_they_were(tctx):
    w, h = 48, 27
    s, m, c, em = scenes.reference_scene(w, h)
    tctx.set_scene(s, m, c, em)
    good = np.random.default_rng(2).uniform(0, 1, (2, 8, 16, 3)).astype(np.float32)
    layers = np.arange(len(s)) % 3 - 1
    tctx.set_textures(good, layers)
    ref, _ = _draw(tctx, w, h, 1)
    host = np.ones((2, 8, 16, 4), np.float32)
    for (tw, th, tn), text in (((0, 8, 2), "width, height and layers must be >= 1"),
                               ((16, 0, 2), "width, height and layers must be >= 1"),
                               ((16, 8, 0), "width, height and layers must be >= 1"),
                               ((65536, 16384, 2), "below 2\\^31")):
        rc, err = _raw_set(tctx, host.ctypes.data, tw, th, tn, [0], 0)
        assert rc != 0 and re.search(text, err), (tw, th, tn, err)
    rc, err = _raw_set(tctx, host.ctypes.data, 16, 8, 2, [0], 0, num=-1)
    assert rc != 0 and "numSpheres must be >= 0" in err, err
    for bad_layers, text in (([0, 2], r"sphereLayers\[1\] = 2 is outside \[-1, 2\)"),
                             ([-2], r"sphereLayers\[0\] = -2 is outside")):
        rc, err = _raw_set(tctx, host.ctypes.data, 16, 8, 2, bad_layers, 0)
        assert rc != 0 and re.search(text, err), err
    dev = torch.ones((2 * 8 * 16 + 1, 4), dtype=torch.float32, device="cuda")
    rc, err = _raw_set(tctx, dev.data_ptr() + 4, 16, 8, 2, [0], 1)
    assert rc != 0 and "16-byte aligned" in err, err
    if torch.cuda.device_count() > 1:
        other = torch.ones((2, 8, 16, 4), dtype=torch.float32, device="cuda:1")
        rc, err = _raw_set(tctx, other.data_ptr(), 16, 8, 2, [0], 1)
        assert rc != 0 and "lives on device 1" in err, err
    for (l, y, x, ch), v in (((0, 3, 5, 0), np.nan), ((1, 7, 15, 2), np.inf), ((1, 0, 0, 1), -np.inf),
                             ((0, 2, 9, 1), -0.5), ((1, 5, 1, 2), -0.0)):
        bad = host.copy()
        bad[l, y, x, ch] = v
        want = f"texel of layer {l} \\(x {x}, y {y}\\) has {'RGB'[ch]} = "
        rc, err = _raw_set(tctx, bad.ctypes.data, 16, 8, 2, [0], 0)
        assert rc != 0 and re.search(want, err), (v, err)
        dbad = torch.from_numpy(bad).cuda()
        torch.cuda.synchronize()
        rc, err = _raw_set(tctx, dbad.data_ptr(), 16, 8, 2, [0], 1)
        assert rc != 0 and re.search(want, err), (v, "device", err)
    # after all the refusals the textures are still `good`
    img, _ = _draw(tctx, w, h, 1)
    assert not bits_differ(img, ref).any()
    alpha = host.copy()
    alpha[..., 3] = np.nan                                # alpha is not checked
    rc, err = _raw_set(tctx, torch.from_numpy(alpha).cuda().data_ptr(), 16, 8, 2, [0], 1)
    assert rc == 0, err
