"""Environment lighting (tpt_set_environment, Context.set_environment) on the GPU.

1. Lookup: caller rays that miss every sphere return the map's bilinear lat-long value, against the float64 oracle of the
   pinned mapping below (env_lookup), across the phi = +-pi seam, at both poles, on non-square and 1 x 1 maps, and on a
   one-hot texel hit at its centre and its neighbours' (orientation and row order).
2. Constant map c: furnace scene A gives exactly albedo * c per sample with the furnace's ray counts in every fast variant
   and through trace_rays; c = mitsuba's sky with mitsuba_compare on is bitwise mitsuba_compare alone.
3. sky_environment(2048, 1024) against the default sky at the same streams, in every fast variant and through
   trace_rays, trace_irradiance, draw_samples and trace_samples: equal ray counts, differences within the map's
   bilinear error (every miss site reads the map).
4. Closed forms: scene B2's cosine lobe under affine maps along x and along z; irradiance under a map lit above the
   horizon only.
5. Mirror chains: the float64 chain oracle of tests/mirror_chain.py with the pinned lookup as its terminal sky.
6. Ordering and lifetime: a map set while a draw is in flight is not seen by it; clearing restores the bits of a context
   that never had a map; the map survives tpt_set_scene; CUDA tensor input.
7. Refusals (parity modes, sizes, alignment, other device, bad texels on host and device) and unchanged AOVs."""
import ctypes

import numpy as np
import pytest
import torch

import furnace as F
import mirror_chain as mc
from conftest import bits_differ, rel_l2
from toypathtracer_b200 import MATERIAL_DTYPE, MODE_EXACT, MODE_FAST, MODE_REFGPU, MODE_REFGPU_FAST, SPHERE_DTYPE, scenes

pytestmark = pytest.mark.gpu


# ---- the pinned mapping in float64 --------------------------------------------------------------------------------
def lat_long_dir(u, v, w, h):
    """Unit direction(s) at continuous texel coordinates (u, v) of a w x h map."""
    phi = np.asarray(u, np.float64) / w * 2.0 * np.pi - np.pi
    theta = np.asarray(v, np.float64) / h * np.pi
    return np.stack([np.sin(theta) * np.sin(phi), np.cos(theta), -np.sin(theta) * np.cos(phi)], -1)


def env_lookup(m, d):
    """The map m [h, w, >= 3] in the directions d [n, 3], as include/tpt_b200.h pins it: phi = atan2(d.x, -d.z),
    theta = acos(d.y), u = (phi + pi) / 2pi * w, v = theta / pi * h, texel centres at + 1/2, bilinear, columns wrap,
    rows clamp. Float64 throughout."""
    m = np.asarray(m, np.float64)[..., :3]
    h, w = m.shape[:2]
    d = np.asarray(d, np.float64).reshape(-1, 3)
    phi = np.arctan2(d[:, 0], -d[:, 2])
    theta = np.arccos(np.clip(d[:, 1], -1.0, 1.0))
    u = (phi + np.pi) / (2.0 * np.pi) * w - 0.5
    v = theta / np.pi * h - 0.5
    fu, fv = np.floor(u), np.floor(v)
    tu, tv = (u - fu)[:, None], (v - fv)[:, None]
    x0 = fu.astype(np.int64) % w
    x1 = (x0 + 1) % w
    y0 = fv.astype(np.int64)
    y1 = np.clip(y0 + 1, 0, h - 1)
    y0 = np.clip(y0, 0, h - 1)
    a, b, c, e = m[y0, x0], m[y0, x1], m[y1, x0], m[y1, x1]
    top, bot = a + tu * (b - a), c + tu * (e - c)
    return top + tv * (bot - top)


def lookup_tolerance(m, d, eps=4e-6):
    """Per direction: how much the oracle moves when d moves by eps (the kernel's normalisation, atan2f and acosf), plus the
    float32 rounding of the texel coordinates and of the blends."""
    base = env_lookup(m, d)
    tol = np.zeros(len(base))
    for k in range(3):
        for s in (-1.0, 1.0):
            dp = d.copy()
            dp[:, k] += s * eps
            dp /= np.linalg.norm(dp, axis=1, keepdims=True)
            tol = np.maximum(tol, np.abs(env_lookup(m, dp) - base).max(1))
    span = float(np.ptp(np.asarray(m, np.float64)[..., :3])) if np.size(m) > 3 else 0.0
    return tol + 2.0 ** -22 * max(m.shape[:2]) * span + 2.0 ** -21 * np.abs(base).max(1) + 1e-7


# ---- scenes and fixtures ------------------------------------------------------------------------------------------
FAR_CENTRE = np.array([37.0, -41.0, 53.0])


def far_scene():
    """One black sphere of radius 1e-3 far from the origin (tpt_set_scene needs one): rays from the origin miss it."""
    sph = np.zeros(1, SPHERE_DTYPE)
    sph[0] = (FAR_CENTRE, 1e-3, 1e3)
    mats = np.zeros(1, MATERIAL_DTYPE)
    return sph, mats, F.furnace_camera(8, 8), np.zeros(0, np.int32)


def far_rays(d):
    """Rays from the origin in the unit directions d, none toward the far sphere."""
    d = np.asarray(d, np.float64)
    c = FAR_CENTRE / np.linalg.norm(FAR_CENTRE)
    keep = d @ c < np.cos(0.01)
    rays = np.concatenate([np.zeros((len(d), 3)), d], 1).astype(np.float32)
    return rays[keep]


@pytest.fixture
def ectx(gpu_ctx):
    yield gpu_ctx
    gpu_ctx.set_environment(None)
    for k, v in (("fast_variant", -1), ("fast_kform", 2), ("mitsuba_compare", 0), ("light_sampling", 1)):
        gpu_ctx.set_option(k, v)
    gpu_ctx.set_spp(4)


def _rays_dirs(rays):
    d = rays[:, 3:].astype(np.float64)
    return d / np.linalg.norm(d, axis=1, keepdims=True)


def _draw(ctx, w, h, spp=None, frame=0, mode=MODE_FAST, frames=1):
    if spp is not None:
        ctx.set_spp(spp)
    buf = torch.zeros((h, w, 4), dtype=torch.float32, device="cuda")
    rays = ctx.draw(frame, frames, w, h, buf, flags=0, mode=mode)
    return buf.cpu().numpy(), rays


# ---- 1. lookup -----------------------------------------------------------------------------------------------------
MAPS = {"64x16": (64, 16), "1x1": (1, 1), "7x24": (7, 24)}


@pytest.mark.parametrize("name", list(MAPS))
def test_lookup_matches_the_oracle(ectx, name):
    w, h = MAPS[name]
    rng = np.random.default_rng(w * 100 + h)
    m = rng.uniform(0.0, 1.0, (h, w, 3)).astype(np.float32)
    ectx.set_scene(*far_scene())
    ectx.set_environment(m)
    d = rng.normal(size=(2000, 3))
    dirs = [d / np.linalg.norm(d, axis=1, keepdims=True)]
    vs = rng.uniform(0, h, 6)
    for u in (0.0, 1e-4, 0.2, 0.5, w - 0.5, w - 0.2, w - 1e-4, w):        # the seam, both sides
        dirs.append(lat_long_dir(np.full(6, u), vs, w, h))
    us = rng.uniform(0, w, 6)
    for v in (0.0, 1e-4, 0.3, 0.5, h - 0.5, h - 0.3, h - 1e-4, h):        # both poles
        dirs.append(lat_long_dir(us, np.full(6, v), w, h))
    ii, jj = np.meshgrid(np.arange(w) + 0.5, np.arange(h) + 0.5)
    dirs.append(lat_long_dir(ii.ravel(), jj.ravel(), w, h))                # every texel centre
    rays = far_rays(np.concatenate(dirs))
    out, traced = ectx.trace_rays(rays, spp=1)
    assert traced == len(rays)
    dd = _rays_dirs(rays)
    want = env_lookup(m, dd)
    err = np.abs(out[:, :3] - want).max(1)
    tol = lookup_tolerance(m, dd)
    bad = err > tol
    assert not bad.any(), (name, int(bad.sum()), dd[bad][:4], out[bad][:4], want[bad][:4], tol[bad][:4])
    if w == h == 1:
        assert (out[:, :3] == m[0, 0]).all()


def test_one_hot_texel_orientation_and_row_order(ectx):
    """Texel (2, 1) of an 8 x 4 map is lit: a ray at its centre sees it, rays at every other texel centre see nothing.
    A mirrored phi moves it to column 5, flipped rows to row 2."""
    w, h = 8, 4
    m = np.zeros((h, w, 3), np.float32)
    m[1, 2] = (1.0, 2.0, 3.0)
    ectx.set_scene(*far_scene())
    ectx.set_environment(m)
    ii, jj = np.meshgrid(np.arange(w) + 0.5, np.arange(h) + 0.5)
    rays = far_rays(lat_long_dir(ii.ravel(), jj.ravel(), w, h))
    assert len(rays) == w * h
    out, _ = ectx.trace_rays(rays, spp=1)
    np.testing.assert_allclose(out[:, :3].reshape(h, w, 3), m, atol=1e-4)
    # the lit texel's centre column lies at phi = 2.5 / 8 * 2pi - pi: left of the -z centre column, toward -x
    assert lat_long_dir(2.5, 1.5, w, h)[0] < 0


# ---- 2. constant maps ------------------------------------------------------------------------------------------------
C_MAP = np.float32([0.7, 0.5, 0.25])


def _const_map(c, w=6, h=3):
    return np.broadcast_to(np.float32(c), (h, w, 3)).copy()


@pytest.mark.parametrize("variant", range(10))
def test_constant_map_gives_the_furnace_value(ectx, variant):
    """Scene A under a constant map c: every sample is albedo * c, so every pixel equals it within a quarter of one
    sample's weight, with exactly 2 + K rays per sample (Lambert, light sampling) or 2; the Metal receiver relies on
    mitsuba_compare's zero roughness, which still applies under a map."""
    w, h, spp = 48, 30, 3
    ectx.set_option("fast_variant", variant)
    ectx.set_environment(_const_map(C_MAP))
    for metal, ls, K in ((False, 1, 3), (False, 0, 3), (True, 1, 2)):
        s, m, c, em = F.furnace_scene(w, h, K, metal)
        ectx.set_option("mitsuba_compare", 1 if metal else 0)
        ectx.set_option("light_sampling", ls)
        ectx.set_scene(s, m, c, em)
        img, rays = _draw(ectx, w, h, spp)
        v = (m["albedo"][0].astype(np.float32) * C_MAP).astype(np.float32)
        exp, tol = F.furnace_expect(np.zeros(3), v, 0, 1, 0, spp)
        err = np.abs(img[..., :3] - exp)
        assert (err <= tol).all(), (variant, metal, ls, float(err.max()), tol)
        assert rays == w * h * spp * F.furnace_rays_per_sample(m, K, bool(ls)), (variant, metal, ls, rays)


def test_constant_map_through_trace_rays(ectx):
    w, h, spp, K = 40, 24, 4, 3
    s, m, c, em = F.furnace_scene(w, h, K)
    ectx.set_scene(s, m, c, em)
    ectx.set_environment(_const_map(C_MAP, 1, 1))
    rays = scenes.camera_rays(c, w, h)
    out, traced = ectx.trace_rays(rays, spp=spp)
    v = (m["albedo"][0].astype(np.float32) * C_MAP).astype(np.float32)
    _exp, tol = F.furnace_expect(np.zeros(3), v, 0, 1, 0, spp)
    assert (np.abs(out[:, :3] - v) <= tol).all()
    assert traced == len(rays) * spp * F.furnace_rays_per_sample(m, K, True)


@pytest.mark.parametrize("variant", range(10))
def test_mitsuba_sky_as_a_map_is_bitwise_mitsuba(ectx, variant):
    """One sample per pixel (each pixel is then a single sum, so the image is deterministic): the reference scene with
    mitsuba_compare under a constant map of mitsuba's sky is bitwise the image of mitsuba_compare alone."""
    w, h = 96, 54
    s, m, c, em = scenes.reference_scene(w, h, mitsuba_compare=True)
    ectx.set_option("fast_variant", variant)
    ectx.set_option("mitsuba_compare", 1)
    ectx.set_scene(s, m, c, em)
    ref, rref = _draw(ectx, w, h, 1)
    ectx.set_environment(_const_map(F.MITSUBA_SKY))
    img, rimg = _draw(ectx, w, h, 1)
    assert rimg == rref
    assert not bits_differ(img, ref).any(), (variant, int(bits_differ(img, ref).sum()))


# ---- 3. the reference sky as a map ---------------------------------------------------------------------------------
SKY_W, SKY_H = 2048, 1024


def sky_map_bound(scale=1.0):
    """Per sample and unit throughput: the map interpolates the sky, linear in cos(theta), linearly in theta (error
    <= (pi / H)^2 / 8 in cos(theta), x 0.075, the sky's largest slope in d_y), plus the float32 lookup (angles to ~1e-6,
    texels and blends to 2^-24 of 0.3)."""
    return scale * (0.075 * (np.pi / SKY_H) ** 2 / 8 + 0.075 * 2e-6 + 4 * 2.0 ** -24 * 0.3)


def _close(a, b, bound, what):
    a = np.asarray(a, np.float64)[..., :3]
    b = np.asarray(b, np.float64)[..., :3]
    tol = 2 * bound + 2.0 ** -19 * np.abs(b)
    err = np.abs(a - b)
    assert (err <= tol).all(), (what, float(err.max()), float((err / tol).max()))


@pytest.fixture(scope="module")
def sky_map():
    return scenes.sky_environment(SKY_W, SKY_H)


def _reference_scene(ectx, w, h):
    s, m, c, em = scenes.reference_scene(w, h)
    ectx.set_scene(s, m, c, em)
    return c


@pytest.mark.parametrize("variant", range(10))
def test_sky_map_matches_the_default_sky_in_draws(ectx, sky_map, variant):
    w, h, spp = 96, 54, 2
    ectx.set_option("fast_variant", variant)
    _reference_scene(ectx, w, h)
    ref, rref = _draw(ectx, w, h, spp)
    ectx.set_environment(sky_map)
    img, rimg = _draw(ectx, w, h, spp)
    assert rimg == rref
    _close(img, ref, sky_map_bound(), f"variant {variant}")
    assert rel_l2(img, ref) < 1e-5


def test_sky_map_matches_the_default_sky_in_caller_calls(ectx, sky_map):
    w, h, spp = 64, 36, 2
    cam = _reference_scene(ectx, w, h)
    rays = scenes.camera_rays(cam, w, h)
    rng = np.random.default_rng(5)
    nrm = rng.normal(size=(777, 3))
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    points = np.concatenate([np.broadcast_to(cam["origin"][0], (777, 3)), nrm], 1).astype(np.float32)

    def run():
        out = {}
        out["rays"] = ectx.trace_rays(rays, spp=spp)
        out["irr"] = ectx.trace_irradiance(points, spp=spp)
        (s4, q4), r = ectx.draw_samples(0, w, h, spp=spp, sum4=np.zeros((w * h, 4), np.float32),
                                        sq4=np.zeros((w * h, 4), np.float32))
        out["draw_samples"] = (s4, r)
        (s4, q4), r = ectx.trace_samples(rays, spp=spp, sum4=np.zeros((len(rays), 4), np.float32),
                                         sq4=np.zeros((len(rays), 4), np.float32))
        out["trace_samples"] = (s4, r)
        (s4, q4), r = ectx.trace_samples(points, points=True, spp=spp, sum4=np.zeros((len(points), 4), np.float32),
                                         sq4=np.zeros((len(points), 4), np.float32))
        out["trace_samples_points"] = (s4, r)
        return out

    ref = run()
    ectx.set_environment(sky_map)
    got = run()
    scale = {"rays": 1, "irr": np.pi, "draw_samples": spp, "trace_samples": spp, "trace_samples_points": np.pi * spp}
    for k in ref:
        assert got[k][1] == ref[k][1], (k, got[k][1], ref[k][1])
        _close(got[k][0], ref[k][0], sky_map_bound(scale[k]), k)


# ---- 4. closed forms -------------------------------------------------------------------------------------------------
def _texel_dirs(w, h):
    ii, jj = np.meshgrid(np.arange(w) + 0.5, np.arange(h) + 0.5)
    return lat_long_dir(ii, jj, w, h)


@pytest.mark.parametrize("axis", [0, 2], ids=["x", "z"])
def test_affine_map_cosine_lobe(ectx, axis):
    """Scene B2's closed form for an affine map L(d) = a + b d_axis: the cosine lobe's mean direction is (2/3) n, so the
    irradiance at a receiver point is E = pi (a + b (2/3) n_axis) (white Lambert vertex of trace_samples' points). Along
    z the lobes of the points facing +z straddle the phi = +-pi seam; along x a mirrored phi flips the sign of b."""
    a, b = np.array([0.5, 0.4, 0.3]), np.array([0.3, 0.2, 0.1])
    mw, mh = 1024, 512
    m = (a + b * _texel_dirs(mw, mh)[..., axis:axis + 1]).astype(np.float32)
    s, mats, c, em = F.b2_scene(8, 8)
    ectx.set_scene(s, mats, c, em)
    ectx.set_environment(m)
    rng = np.random.default_rng(11 + axis)
    n = rng.normal(size=(2048, 3))
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    pts = np.concatenate([F.RECEIVER_R * n, n], 1).astype(np.float32)
    ids = np.zeros(len(pts), np.int32)
    batches = []
    for f in range(8):
        (s4, _q4), _r = ectx.trace_samples(pts, ids=ids, points=True, spp=32, frame=f)
        batches.append(s4[:, :3] / s4[:, 3:4])
    e = np.pi * (a + b * (2.0 / 3.0) * n[:, axis:axis + 1])
    F.check_bins(np.stack(batches)[:, None], e[None], F.bins_by(e[None], 8, key=n[None, :, axis]))


def test_irradiance_under_a_horizon_map(ectx):
    """A map lit with L above the horizon and black below: E(n) = pi L (1 + n_y) / 2. The bilinear blur reaches half a
    texel (pi / 2H) either side of the horizon; it moves E by less than pi L * (pi / 2H)."""
    L = np.array([1.0, 0.5, 0.25])
    mw, mh = 16, 2048
    m = np.zeros((mh, mw, 3), np.float32)
    m[:mh // 2] = L
    ectx.set_scene(*far_scene()[:3], None)
    ectx.set_environment(m)
    rng = np.random.default_rng(3)
    n = rng.normal(size=(1024, 3))
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    pts = np.concatenate([np.zeros((len(n), 3)), n], 1).astype(np.float32)
    batches = [ectx.trace_irradiance(pts, spp=128, frame=f)[0][:, :3] for f in range(8)]
    bt = np.stack(batches)
    e = np.pi * L * (1.0 + n[:, 1:2]) / 2.0
    bins = np.digitize(n[:, 1], [-0.5, 0.0, 0.5])
    blur = np.pi * L * np.pi / (2 * mh)
    for bn in range(4):
        sel = bins == bn
        bm = bt[:, sel].mean(1)
        mean, se = bm.mean(0), bm.std(0, ddof=1) / np.sqrt(len(bm))
        assert (np.abs(mean - e[sel].mean(0)) <= 5 * se + blur + 1e-6).all(), (bn, mean, e[sel].mean(0), se)


# ---- 5. mirror chains ------------------------------------------------------------------------------------------------
CHAIN_A, CHAIN_B, CHAIN_W = np.array([0.6, 0.5, 0.4]), np.array([0.15, 0.2, -0.1]), np.array([1.0, 0.8, 0.6])


def test_mirror_chains_end_in_the_map(ectx, monkeypatch):
    """The mirror-chain oracle (zero-roughness metal chains, deterministic) with the pinned lookup of an affine map as
    its terminal sky: every well-conditioned caller ray's value within the oracle's tolerance, exact ray counts."""
    mw, mh = 256, 128
    m = (CHAIN_A + (_texel_dirs(mw, mh) @ CHAIN_B)[..., None] * CHAIN_W).astype(np.float32)
    monkeypatch.setattr(mc, "sky", lambda d, mitsuba: env_lookup(m, d))
    # the map's slope per unit of direction: the affine part's, with a margin for the bilinear interpolation
    monkeypatch.setattr(mc, "SKY_SLOPE", 1.5 * float(np.linalg.norm(CHAIN_B)))
    s, mats, em = mc.corridor(46, "compact")
    rays = mc.candidate_rays(s, 1500, seed=63)
    res = mc.chains(rays, s, mats)
    well = res["well"]
    rays, res = rays[well], mc.subset(res, well)
    assert len(rays) >= 20 and (res["seg_cpu"] >= 3).any()
    ectx.set_scene(s, mats, mc.point_camera(mc.CAMERA_O, (0, 0, -1))[0], em)
    ectx.set_environment(m)
    for ls in (1, 0):
        ectx.set_option("light_sampling", ls)
        ectx.set_scene(s, mats, mc.point_camera(mc.CAMERA_O, (0, 0, -1))[0], em)
        out, traced = ectx.trace_rays(rays, spp=2, frame=ls)
        err = np.abs(out[:, :3] - res["v_cpu"]).max(1)
        tol = res["tol_cpu"] + 4 * 2.0 ** -23 * np.abs(res["v_cpu"]).max(1) + 1e-6
        bad = err > tol
        assert not bad.any(), (ls, int(bad.sum()), res["seg_cpu"][bad][:5], (err / tol)[bad][:5])
        assert traced == 2 * int(res["seg_cpu"].sum())


# ---- 6. ordering and lifetime --------------------------------------------------------------------------------------
def test_a_map_set_during_a_draw_is_not_seen_by_it(ectx):
    """Map A, a long draw into a device buffer without synchronising, map B, another draw: the first image is the
    A-only image and the second the B-only image (maps 100x apart)."""
    w, h, spp = 1920, 1080, 16
    _reference_scene(ectx, w, h)
    ectx.set_spp(spp)
    a, b = _const_map([1.0, 1.0, 1.0]), _const_map([0.01, 0.01, 0.01])
    bufs = [torch.zeros((h, w, 4), dtype=torch.float32, device="cuda") for _ in range(2)]
    torch.cuda.synchronize()
    ectx.set_environment(a)
    ectx.draw(0, 1, w, h, bufs[0], flags=0, mode=MODE_FAST, want_rays=False)
    ectx.set_environment(b)
    ectx.draw(0, 1, w, h, bufs[1], flags=0, mode=MODE_FAST, want_rays=False)
    torch.cuda.synchronize()
    got = [t.cpu().numpy() for t in bufs]
    ectx.set_environment(a)
    ref_a, _ = _draw(ectx, w, h)
    ectx.set_environment(b)
    ref_b, _ = _draw(ectx, w, h)
    assert rel_l2(got[0], ref_a) < 1e-5, rel_l2(got[0], ref_a)
    assert rel_l2(got[1], ref_b) < 1e-5, rel_l2(got[1], ref_b)
    assert rel_l2(ref_b, ref_a) > 0.1


def test_clearing_restores_a_context_that_never_had_a_map(libs, ectx):
    w, h = 96, 54
    s, m, c, em = scenes.reference_scene(w, h)
    fresh = libs.Context(0)
    try:
        fresh.set_scene(s, m, c, em)
        ref, rref = _draw(fresh, w, h, 1)
    finally:
        fresh.close()
    ectx.set_scene(s, m, c, em)
    ectx.set_environment(_const_map(C_MAP))
    ectx.set_environment(None)
    img, rimg = _draw(ectx, w, h, 1)
    assert rimg == rref and not bits_differ(img, ref).any()


def test_the_map_survives_set_scene_and_takes_cuda_tensors(ectx):
    w, h = 96, 54
    rng = np.random.default_rng(8)
    m = rng.uniform(0.0, 2.0, (32, 64, 3)).astype(np.float32)
    s, mats, c, em = scenes.reference_scene(w, h)
    ectx.set_scene(s, mats, c, em)
    ectx.set_environment(m)
    ref, rref = _draw(ectx, w, h, 1)
    s2 = s.copy()
    s2["center"][1, 1] += 0.5                          # another scene, then the first one again
    ectx.set_scene(s2, mats, c, em)
    other, _ = _draw(ectx, w, h, 1)
    assert bits_differ(other, ref).any()
    ectx.set_scene(s, mats, c, em)
    img, rimg = _draw(ectx, w, h, 1)
    assert rimg == rref and not bits_differ(img, ref).any()
    ectx.set_environment(None)
    plain, _ = _draw(ectx, w, h, 1)
    assert bits_differ(plain, ref).any()
    rgba = torch.from_numpy(np.concatenate([m, np.full(m.shape[:2] + (1,), np.nan, np.float32)], 2)).cuda()
    ectx.set_environment(rgba)                         # (H, W, 4) CUDA tensor, alpha ignored
    img, _ = _draw(ectx, w, h, 1)
    assert not bits_differ(img, ref).any()
    ectx.set_environment(torch.from_numpy(m).cuda())   # (H, W, 3) CUDA tensor
    img, _ = _draw(ectx, w, h, 1)
    assert not bits_differ(img, ref).any()


# ---- 7. refusals and AOVs ------------------------------------------------------------------------------------------
def _raw_set(ctx, ptr, w, h, on_dev):
    rc = ctx._L.tpt_set_environment(ctx._h, ctypes.c_void_p(ptr), w, h, on_dev)
    return rc, ctx._L.tpt_last_error(ctx._h).decode()


def test_parity_modes_are_refused_while_a_map_is_set(ectx):
    w, h = 32, 18
    _reference_scene(ectx, w, h)
    ectx.set_environment(_const_map(C_MAP))
    for mode in (MODE_EXACT, MODE_REFGPU, MODE_REFGPU_FAST):
        with pytest.raises(libs_error(), match="only TPT_MODE_FAST draws use one"):
            _draw(ectx, w, h, 1, mode=mode)
    ectx.set_environment(None)
    for mode in (MODE_EXACT, MODE_REFGPU, MODE_REFGPU_FAST):
        _img, rays = _draw(ectx, w, h, 1, mode=mode)
        assert rays > 0


def libs_error():
    import toypathtracer_b200 as tpt
    return tpt.TptError


def test_bad_maps_are_refused_and_leave_the_map_as_it_was(ectx):
    w, h = 48, 27
    _reference_scene(ectx, w, h)
    good = np.random.default_rng(2).uniform(0, 1, (8, 16, 3)).astype(np.float32)
    ectx.set_environment(good)
    ref, _ = _draw(ectx, w, h, 1)
    host = np.ones((8, 16, 4), np.float32)
    for (mw, mh), text in (((0, 8), "width and height must be >= 1"), ((16, 0), "width and height must be >= 1"),
                           ((-3, 8), "width and height must be >= 1"), ((65536, 32768), "below 2\\^31")):
        rc, err = _raw_set(ectx, host.ctypes.data, mw, mh, 0)
        assert rc != 0 and __import__("re").search(text, err), (mw, mh, err)
    dev = torch.ones((8 * 16 + 1, 4), dtype=torch.float32, device="cuda")
    rc, err = _raw_set(ectx, dev.data_ptr() + 4, 16, 8, 1)
    assert rc != 0 and "16-byte aligned" in err, err
    if torch.cuda.device_count() > 1:
        other = torch.ones((8, 16, 4), dtype=torch.float32, device="cuda:1")
        rc, err = _raw_set(ectx, other.data_ptr(), 16, 8, 1)
        assert rc != 0 and "lives on device 1" in err, err
    for (y, x, ch), v in (((3, 5, 0), np.nan), ((7, 15, 2), np.inf), ((0, 0, 1), -np.inf), ((2, 9, 1), -0.5),
                          ((5, 1, 2), -0.0)):
        bad = host.copy()
        bad[y, x, ch] = v
        want = f"texel {y * 16 + x} \\(x {x}, y {y}\\) has {'RGB'[ch]} = "
        rc, err = _raw_set(ectx, bad.ctypes.data, 16, 8, 0)
        assert rc != 0 and __import__("re").search(want, err), (v, err)
        dbad = torch.from_numpy(bad).cuda()
        torch.cuda.synchronize()
        rc, err = _raw_set(ectx, dbad.data_ptr(), 16, 8, 1)
        assert rc != 0 and __import__("re").search(want, err), (v, "device", err)
    alpha = host.copy()
    alpha[..., 3] = np.nan                                # alpha is not checked
    rc, err = _raw_set(ectx, torch.from_numpy(alpha).cuda().data_ptr(), 16, 8, 1)
    assert rc == 0, err
    ectx.set_environment(good)
    # after all the refusals the map is still `good`
    img, _ = _draw(ectx, w, h, 1)
    assert not bits_differ(img, ref).any()


def test_aovs_ignore_the_map(ectx):
    w, h = 64, 36
    cam = _reference_scene(ectx, w, h)
    rays = scenes.camera_rays(cam, w, h)

    def aovs():
        alb, nrm, ids = (torch.zeros((h, w, 4), device="cuda"), torch.zeros((h, w, 4), device="cuda"),
                         torch.zeros((h, w), dtype=torch.int32, device="cuda"))
        r1 = ectx.draw_aovs(0, 1, w, h, alb, nrm, ids)
        (ra, rn, ri), r2 = ectx.trace_aovs(rays)
        return [t.cpu().numpy() for t in (alb, nrm, ids)] + [ra, rn, ri], (r1, r2)

    ref, rr = aovs()
    ectx.set_environment(np.random.default_rng(4).uniform(0, 5, (16, 32, 3)).astype(np.float32))
    got, rg = aovs()
    assert rg == rr
    for a, b in zip(got, ref):
        assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))
