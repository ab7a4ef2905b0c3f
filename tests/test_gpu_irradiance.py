"""tpt_trace_irradiance (Context.trace_irradiance): fast-mode irradiance at caller surface points, checked where the answer is
exact or known — furnace scene A point by point in every k_fast_rays instance (value pi * sky, exact ray count), the closed
forms B1 and B2 of tests/furnace.py on their quadrature nodes, the self-skip of a point's own light — against the draw's own
estimator on camera rays (trace_rays = Le + albedo * E / pi at Lambert first hits), and the C-ABI behaviour around it
(streams, buffers, refusals, untraceable points, ordering and accounting)."""
import ctypes

import numpy as np
import pytest
import torch

import furnace as F
import test_sweep_oracle as so
from conftest import bits_differ
from test_gpu_mirror_chains import LONG_SLABS_PER_WARP, SLAB_PIX, queue_instance
from test_gpu_rays import _scaled, padded_furnace
from toypathtracer_b200.scenes import camera_rays

pytestmark = pytest.mark.gpu

RAYS_INSTANCES = {f"k_fast_rays{nl}<{t}, {m}, {k}>" for nl in ("", "_nolight")
                  for t, m, k in [(128, 6, 0), (128, 6, 1), (128, 6, 2), (128, 6, 3), (128, 6, 4), (128, 8, 2), (128, 8, 4),
                                  (768, 1, 0), (768, 1, 1), (768, 1, 2), (768, 1, 3)]}


@pytest.fixture
def ictx(gpu_ctx):
    yield gpu_ctx
    for k, v in (("fast_kform", 2), ("mitsuba_compare", 0), ("light_sampling", 1)):
        gpu_ctx.set_option(k, v)
    gpu_ctx.set_spp(4)


def _num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def sphere_points(centre, radius, n, seed, scale_half=True):
    """n points {p, n} uniform on a sphere, normal (p - centre) / radius; half of the normals rescaled by factors in
    [1e-3, 1e3] (the call normalises them)."""
    rng = np.random.default_rng(seed)
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    pts = np.concatenate([np.asarray(centre, np.float64) + radius * d, d], 1).astype(np.float32)
    if scale_half:
        half = np.arange(n) % 2 == 1
        pts[half] = _scaled(pts[half], seed)
    return pts


# ---- 1. furnace A, point by point, in every k_fast_rays instance -----------------------------------------------------
def speck(s, m):
    """Scene A plus one non-emissive sphere of radius 1e-6 at distance 12: it fails the expanded form's accuracy gate (so
    fast_kform 2 and 3 run the conservative form 3), and no bounce ray meets it (solid angle ~ 2e-14)."""
    s2 = np.zeros(1, s.dtype); m2 = np.zeros(1, m.dtype)
    s2["center"] = (0.0, 0.0, -12.0); s2["radius"] = 1e-6; s2["invRadius"] = np.float32(1e6)
    m2["albedo"] = 0.5
    return np.concatenate([s, s2]), np.concatenate([m, m2])


def furnace_a(K, padded=False, with_speck=False):
    s, m, c, em = padded_furnace(K, False) if padded else F.furnace_scene(64, 64, K, False)
    if with_speck:
        s, m = speck(s, m)
    return s, m, c, em


def check_points(ctx, s, m, K, ls, pts, spp, frame, seen, kopt, long=False, label=""):
    """Every traceable point gives pi * sky (a few ulps), alpha 0, and (1 + K) rays per sample with light sampling, 1
    without; the launch ran the instance the pick rules choose."""
    dev = torch.from_numpy(pts).cuda()
    ids = torch.zeros(len(pts), dtype=torch.int32, device="cuda")        # the receiver's id: not a light
    out, traced = ctx.trace_irradiance(dev, ids=ids if len(pts) % 2 else None, spp=spp, frame=frame)
    got = ctx.last_kernels()
    seen.update(got)
    want = queue_instance("rays", len(s), K, kopt, so.gate_passes(s) and kopt != 0, ls, long=long)
    assert got == [want], (label, got, want)
    out = out.cpu().numpy()
    v = np.pi * F.MITSUBA_SKY.astype(np.float64)
    tol = v * (spp + 2) * 2.0 ** -23
    err = np.abs(out[:, :3] - v)
    assert (err <= tol).all(), (label, int((err > tol).any(1).sum()), out[(err > tol).any(1)][:4], v)
    assert (out[:, 3] == 0).all(), label
    assert traced == len(pts) * spp * ((1 + K) if ls else 1), (label, traced)


def test_furnace_points_every_instance(ictx):
    """Scene A with points all over the receiver (normal p / R): every sample is exactly the sky, E = pi * sky. Small
    scenes with 0-300 buried lights, 65 spheres (pair array in shared memory), 1 500 padding spheres (past 64 KB: the
    768-thread instance), each with and without a far speck that fails the accuracy gate, under fast_kform 0-3 and light
    sampling on and off, and launches of >= 48 slabs per warp (the 8-CTA instances): the union of the instances run is
    all 22 k_fast_rays instances."""
    ictx.set_option("mitsuba_compare", 1)
    seen = set()
    cases = [(3, False, False), (64, False, False), (3, True, False), (3, False, True), (3, True, True)]
    for K, padded, with_speck in cases:
        s, m, c, em = furnace_a(K, padded, with_speck)
        for kopt in (0, 1, 2, 3):
            ictx.set_option("fast_kform", kopt)
            for ls in (1, 0):
                ictx.set_option("light_sampling", ls)
                ictx.set_scene(s, m, c, em)
                pts = sphere_points((0, 0, 0), F.RECEIVER_R, 5001, 10 * K + kopt)
                check_points(ictx, s, m, K, ls, pts, 3, kopt, seen, kopt,
                             label=f"K{K} padded{padded} speck{with_speck} kform{kopt} ls{ls}")
    # the 8-CTA instances: forms 4 (5 spheres) and 2 (65 spheres), >= 48 slabs of 64 points per warp on every SM
    n = 65536
    spp = -(-LONG_SLABS_PER_WARP * _num_sms() * 32 // (n // SLAB_PIX))
    pts = sphere_points((0, 0, 0), F.RECEIVER_R, n, 5)
    ictx.set_option("fast_kform", 2)
    for K in (3, 64):
        s, m, c, em = furnace_a(K)
        for ls in (1, 0):
            ictx.set_option("light_sampling", ls)
            ictx.set_scene(s, m, c, em)
            check_points(ictx, s, m, K, ls, pts, spp, 9, seen, 2, long=True, label=f"long K{K} ls{ls}")
    # no lights, and 300 lights
    for K in (0, 300):
        s, m, c, em = furnace_a(K)
        ictx.set_option("light_sampling", 1)
        ictx.set_scene(s, m, c, em)
        check_points(ictx, s, m, K, 1, sphere_points((0, 0, 0), F.RECEIVER_R, 3000, K), 2, 1, seen, 2, label=f"K{K}")
    assert seen == RAYS_INSTANCES, (sorted(RAYS_INSTANCES - seen), sorted(seen - RAYS_INSTANCES))


# ---- 2. closed forms B1, B2 --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("scene", ["b1_ls", "b1_nols", "b2"])
def test_closed_forms_on_quadrature_points(ictx, scene):
    """The receiver points of furnace.footprint_hits with normal p / R, weighted by their Gauss-Legendre weights: per
    pixel E / pi = sky + sum_i (Le_i - sky) Phi_i (B1, light sampling on and off) or gradient_sky(2/3 n_y) (B2), i.e. the
    B expectations without the albedo. 32 frames of 16 nodes x 64 spp, per-bin means within max(5 se, 1e-4 E)."""
    s, m, c, em, w, h, e, bins, mitsuba, ls = F.b_case(scene)
    ictx.set_option("mitsuba_compare", 1 if mitsuba else 0)
    ictx.set_option("light_sampling", 1 if ls else 0)
    ictx.set_scene(s, m, c, em)
    p, wq, _ = F.footprint_hits(c, w, h)
    pts = torch.from_numpy(np.concatenate([p, p / F.RECEIVER_R], -1).reshape(-1, 6).astype(np.float32)).cuda()
    ids = torch.zeros(len(pts), dtype=torch.int32, device="cuda")
    wt = torch.from_numpy(wq).cuda()
    batches = []
    for b in range(32):
        out, _ = ictx.trace_irradiance(pts, ids=ids, spp=64, frame=b)
        px = (out[:, :3].double().view(h, w, len(wq), 3) * wt[None, None, :, None]).sum(2) / np.pi
        batches.append(px.cpu().numpy())
    F.check_bins(np.array(batches), e / m["albedo"][0].astype(np.float64), bins)


# ---- 3. a point's own light -------------------------------------------------------------------------------------------
def test_ids_skip_the_points_own_light(ictx):
    """One emissive Lambert sphere under the constant sky, points on it: with its id every sample is the sky (its only
    light is its own, never sampled) and traces one ray, the bounce; without ids each sample also samples the sphere
    itself, one more ray. Ids of other spheres, or -1, change nothing."""
    sph = np.zeros(1, F.SPHERE_DTYPE); mats = np.zeros(1, F.MATERIAL_DTYPE)
    sph[0] = ((0.3, -0.2, 0.1), 0.4, np.float32(1) / np.float32(0.4))
    mats[0] = (F.LAMBERT, (0.7, 0.5, 0.3), (4.0, 5.0, 6.0), 0.0, 0.0)
    ictx.set_option("mitsuba_compare", 1)
    ictx.set_scene(sph, mats, F.furnace_camera(64, 64), np.array([0], np.int32))
    n, spp = 4000, 3
    pts = torch.from_numpy(sphere_points((0.3, -0.2, 0.1), 0.4, n, 3)).cuda()
    v = np.pi * F.MITSUBA_SKY.astype(np.float64)
    own = torch.zeros(n, dtype=torch.int32, device="cuda")
    out, traced = ictx.trace_irradiance(pts, ids=own, spp=spp, frame=2)
    out = out.cpu().numpy()
    assert (np.abs(out[:, :3] - v) <= v * (spp + 2) * 2.0 ** -23).all() and (out[:, 3] == 0).all()
    assert traced == n * spp
    for other in (None, -1, 1, 7):
        ids = None if other is None else torch.full((n,), other, dtype=torch.int32, device="cuda")
        _, t2 = ictx.trace_irradiance(pts, ids=ids, spp=spp, frame=2)
        assert t2 == 2 * n * spp, (other, t2)
    # mixed: the odd points name their sphere
    mixed = torch.where(torch.arange(n, device="cuda") % 2 == 1, 0, -1).to(torch.int32)
    _, t3 = ictx.trace_irradiance(pts, ids=mixed, spp=spp, frame=2)
    assert t3 == n * spp + (n // 2) * spp


# ---- 4. the draw's estimator: trace_rays = Le + albedo * E / pi at Lambert first hits -----------------------------------
def lambert_hits(ctx, sph, mats, rays):
    """The camera rays whose first hit (trace_aovs) is a Lambert sphere met from outside, and the surface points
    {o + t d, normal} and sphere ids there."""
    (alb, nrm, ids), _ = ctx.trace_aovs(torch.from_numpy(rays).cuda())
    alb, nrm, ids = alb.cpu().numpy(), nrm.cpu().numpy(), ids.cpu().numpy()
    d = rays[:, 3:].astype(np.float64)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    hit = (ids >= 0) & (ids < len(sph))
    lam = hit & (mats["type"][np.clip(ids, 0, len(sph) - 1)] == F.LAMBERT)
    front = (nrm[:, :3].astype(np.float64) * d).sum(1) < 0
    sel = np.nonzero(lam & front)[0]
    p = rays[sel, :3].astype(np.float64) + nrm[sel, 3:4].astype(np.float64) * d[sel]
    pts = np.concatenate([p, nrm[sel, :3]], 1).astype(np.float32)
    return sel, pts, ids[sel]


@pytest.mark.parametrize("scene", ["reference", "stress"])
@pytest.mark.parametrize("ls", [1, 0])
def test_matches_the_draws_estimator(ictx, libs, scene, ls):
    """Camera rays whose first hit is a Lambert sphere (light spheres included, passing their id): per bin of (first-hit
    sphere, luminance quartile), the mean of trace_rays equals the mean of Le + albedo * trace_irradiance(o + t d, normal,
    id) / pi, 32 frames as independent batches of >= 10^4 rays x 64 spp each, within max(5 se, 1e-4 E) with se from the
    spread of the per-frame differences. This pins the depth budget, the order of the stream's draws and the self-skip
    rule of the irradiance start against the estimator itself."""
    w, h = (256, 144) if scene == "reference" else (320, 180)
    if scene == "reference":
        sph, mats, cam, em = libs.reference_scene(w, h)
    else:
        sph, mats, cam = libs.stress_scene(w, h, count=4096)[:3]
        em = None
    ictx.set_option("light_sampling", ls)
    ictx.set_scene(sph, mats, cam, em)
    rays = camera_rays(cam, w, h, per_pixel=1, seed=31)
    sel, pts, ids = lambert_hits(ictx, sph, mats, rays)
    assert len(sel) >= 10_000, len(sel)
    if scene == "reference":
        assert (mats["emissive"][ids].max(1) > 0).any()          # light spheres are among the points
    r_dev = torch.from_numpy(rays[sel]).cuda()
    p_dev = torch.from_numpy(pts).cuda()
    i_dev = torch.from_numpy(ids.astype(np.int32)).cuda()
    le = mats["emissive"][ids].astype(np.float64)
    alb = mats["albedo"][ids].astype(np.float64)
    L, P = [], []
    for f in range(32):
        lo, _ = ictx.trace_rays(r_dev, spp=64, frame=f)
        eo, _ = ictx.trace_irradiance(p_dev, ids=i_dev, spp=64, frame=f)
        L.append(lo[:, :3].double().cpu().numpy())
        P.append(le + alb * eo[:, :3].double().cpu().numpy() / np.pi)
    L, P = np.array(L), np.array(P)
    assert np.isfinite(L).all() and np.isfinite(P).all()
    pm = P.mean(0)
    lum = pm @ np.array([0.25, 0.5, 0.25])
    key = np.zeros(len(ids), np.int64)
    for sid in np.unique(ids):
        msk = ids == sid
        if msk.sum() >= 400:
            key[msk] = (sid + 1) * 4 + F.bins_by(pm[msk], 4, lum[msk])
    _, bins = np.unique(key, return_inverse=True)
    # per-frame differences re-centred on the prediction: their batch mean is L's, their spread that of L - P
    F.check_bins(L - P + pm[None], pm, bins)


# ---- 5. streams, buffers, refusals, ordering, accounting --------------------------------------------------------------
def reference_points(ctx, libs, w=160, h=90):
    sph, mats, cam, em = libs.reference_scene(w, h)
    ctx.set_scene(sph, mats, cam, em)
    _, pts, ids = lambert_hits(ctx, sph, mats, camera_rays(cam, w, h, per_pixel=1, seed=1))
    return pts, ids.astype(np.int32)


def test_frames_and_determinism(ictx, libs):
    """A repeat call gives the same bits (spp 1: one reduction per output) or the same values (spp 4); frames are
    independent: against the mean of 32 frames at spp 4, a call at spp 128 of another frame deviates by the variance
    of two independent 128-sample means (F test on the pooled spread)."""
    pts, ids = reference_points(ictx, libs)
    pts_d, ids_d = torch.from_numpy(pts).cuda(), torch.from_numpy(ids).cuda()
    a, ra = ictx.trace_irradiance(pts_d, ids_d, spp=1, frame=7)
    b, rb = ictx.trace_irradiance(pts_d, ids_d, spp=1, frame=7)
    assert ra == rb and not bits_differ(a.cpu().numpy()[None], b.cpu().numpy()[None]).any()
    a4, _ = ictx.trace_irradiance(pts_d, ids_d, spp=4, frame=7)
    b4, _ = ictx.trace_irradiance(pts_d, ids_d, spp=4, frame=7)
    c4, _ = ictx.trace_irradiance(pts_d, ids_d, spp=4, frame=8)
    assert torch.allclose(a4, b4, rtol=1e-5, atol=0) and (a4 != c4).double().mean() > 0.5
    lum = torch.tensor([0.25, 0.5, 0.25], dtype=torch.float64, device="cuda")
    X = torch.stack([ictx.trace_irradiance(pts_d, ids_d, spp=4, frame=100 + f)[0][:, :3].double() @ lum for f in range(32)])
    mu = X.mean(0)
    V = ((X - mu) ** 2).sum() / (X.shape[1] * 31)                    # var of a 4-sample mean, pooled over the points
    Y = ictx.trace_irradiance(pts_d, ids_d, spp=128, frame=999)[0][:, :3].double() @ lum
    Fstat = float(((Y - mu) ** 2).mean() / (V / 16))                   # var(Y - mu) = V / 32 + V / 32
    assert 0.8 < Fstat < 1.25, Fstat


def test_buffer_kinds_agree(ictx, libs):
    """Host numpy (pageable and page-locked), torch CUDA on a side stream from a row slice at an odd row offset (8-byte
    aligned), and DevicePtr buffers give the same bits (spp 1) and ray counts, ids in the points' kind."""
    pts, ids = reference_points(ictx, libs)
    n = len(pts)
    ref, traced = ictx.trace_irradiance(pts, ids, spp=1, frame=3)
    assert isinstance(ref, np.ndarray) and ref.shape == (n, 4) and np.isfinite(ref).all() and (ref[:, 3] == 0).all()
    assert traced > n
    pin_p = torch.empty((n, 6), dtype=torch.float32, pin_memory=True); pin_p.numpy()[...] = pts
    pin_i = torch.empty(n, dtype=torch.int32, pin_memory=True); pin_i.numpy()[...] = ids
    pin_o = torch.empty((n, 4), dtype=torch.float32, pin_memory=True)
    out, t2 = ictx.trace_irradiance(pin_p, pin_i, spp=1, frame=3, out=pin_o)
    assert out is pin_o and t2 == traced and not bits_differ(pin_o.numpy()[None], ref[None]).any()
    side = torch.cuda.Stream()
    base = torch.zeros((n + 1, 6), dtype=torch.float32, device="cuda")
    base[1:] = torch.from_numpy(pts).cuda()
    sl = base[1:]
    assert sl.data_ptr() % 16 == 8
    dev_i = torch.from_numpy(ids).cuda()
    torch.cuda.synchronize()
    dev_out = ictx.trace_irradiance(sl, dev_i, spp=1, frame=3, stream=side.cuda_stream, want_rays=False)
    assert dev_out.is_cuda and dev_out.shape == (n, 4)
    side.synchronize()
    assert not bits_differ(dev_out.cpu().numpy()[None], ref[None]).any()
    pp, ip, op = ictx.mem_alloc(n * 24), ictx.mem_alloc(n * 4), ictx.mem_alloc(n * 16)
    try:
        ictx.mem_from_host(pp, pts); ictx.mem_from_host(ip, ids)
        _, t3 = ictx.trace_irradiance(pp, ip, spp=1, frame=3, out=op, n=n)
        got = ictx.mem_to_host(op, np.empty((n, 4), np.float32))
    finally:
        ictx.mem_free(pp); ictx.mem_free(ip); ictx.mem_free(op)
    assert t3 == traced and not bits_differ(got[None], ref[None]).any()


def test_untraceable_points_give_zero_and_no_rays(ictx):
    """A point with a non-finite component, or a normal that does not normalise, gives (0, 0, 0, 0) and adds no rays; the
    others are the furnace value."""
    K = 3
    s, m, c, em = furnace_a(K)
    ictx.set_option("mitsuba_compare", 1)
    ictx.set_scene(s, m, c, em)
    pts = sphere_points((0, 0, 0), F.RECEIVER_R, 1000, 4)
    bad = [(3, 0.0), (3, np.nan), (4, np.inf), (5, -np.inf), (0, np.nan), (1, np.inf), (3, "tiny")]
    for i in range(0, 1000, 3):            # every third point broken, in runs that straddle the 64-entry slabs
        col, val = bad[(i // 3) % len(bad)]
        if val == "tiny":
            pts[i, 3:] = (1e-30, -1e-30, 1e-30)      # squared length underflows
        elif col == 3 and val == 0.0:
            pts[i, 3:] = 0.0
        else:
            pts[i, col] = val
    valid = np.isfinite(pts).all(1) & (np.abs(pts[:, 3:]).max(1) > 1e-20)
    out, traced = ictx.trace_irradiance(pts, spp=3)
    v = np.pi * F.MITSUBA_SKY.astype(np.float64)
    assert (np.abs(out[valid, :3] - v) <= v * 5 * 2.0 ** -23).all() and (out[valid, 3] == 0).all()
    assert (out[~valid] == 0).all() and not np.signbit(out[~valid]).any()
    assert traced == int(valid.sum()) * 3 * (1 + K)


def test_refusals(ictx, libs):
    s, m, c, em = furnace_a(3)
    ictx.set_scene(s, m, c, em)
    L, hdl = ictx._L, ictx._h
    dev = torch.zeros((70, 6), dtype=torch.float32, device="cuda")
    dids = torch.zeros(71, dtype=torch.int32, device="cuda")
    dout = torch.zeros((70, 4), dtype=torch.float32, device="cuda")
    p, i, o = (ctypes.c_void_p(t.data_ptr()) for t in (dev, dids, dout))
    cnt = ctypes.c_longlong(-1)

    def call(pts, ids, pon, n, spp, out, oon):
        return L.tpt_trace_irradiance(hdl, pts, ids, pon, n, spp, 0, out, oon, ctypes.byref(cnt), None)

    def refused(text, *args):
        assert call(*args) != 0
        assert text in L.tpt_last_error(hdl).decode(), (text, L.tpt_last_error(hdl).decode())

    refused("tpt_trace_irradiance: null points6 or out4", None, i, 1, 4, 1, o, 1)
    refused("null points6 or out4", p, i, 1, 4, 1, None, 1)
    refused("tpt_trace_irradiance: n < 0", p, i, 1, -1, 1, o, 1)
    refused("spp < 1", p, i, 1, 4, 0, o, 1)
    refused("n * spp > 2^32", p, i, 1, (1 << 31) + 1, 2, o, 1)
    refused("n * spp > 2^32", p, i, 1, 1 << 32, 1, o, 1)
    refused("out4 is not 16-byte aligned", p, i, 1, 4, 1, ctypes.c_void_p(dout.data_ptr() + 4), 1)
    refused("points6 is not 4-byte aligned", ctypes.c_void_p(dev.data_ptr() + 2), i, 1, 4, 1, o, 1)
    refused("ids is not 4-byte aligned", p, ctypes.c_void_p(dids.data_ptr() + 2), 1, 4, 1, o, 1)
    host = np.zeros((4, 6), np.float32)
    hids = np.zeros(4, np.int32)
    refused("points6 is not CUDA memory", ctypes.c_void_p(host.ctypes.data), i, 1, 4, 1, o, 1)
    refused("ids is not CUDA memory", p, ctypes.c_void_p(hids.ctypes.data), 1, 4, 1, o, 1)
    with pytest.raises(libs.TptError, match="spp < 1"):
        ictx.trace_irradiance(np.zeros((4, 6), np.float32), spp=0)
    # a device-aligned ids pointer at a 4-byte offset is fine
    assert call(p, ctypes.c_void_p(dids.data_ptr() + 4), 1, 70, 1, o, 1) == 0
    # n == 0: nothing launched, no rays
    cnt.value = -1
    assert call(ctypes.c_void_p(host.ctypes.data), None, 0, 0, 4, ctypes.c_void_p(host.ctypes.data), 0) == 0
    assert cnt.value == 0 and ictx.last_launch_count() == 0 and ictx.last_kernels() == []
    out, traced = ictx.trace_irradiance(np.zeros((0, 6), np.float32), ids=np.zeros(0, np.int32))
    assert out.shape == (0, 4) and traced == 0


def test_accounting_and_neighbours(ictx, libs):
    """One trace launch and the counter fold; the rays count toward read_ray_count with a draw's; a fast draw and a
    trace_rays call before and after an irradiance call, and a side-stream irradiance call between two progressive draws,
    give the bits they give alone."""
    K = 3
    s, m, c, em = furnace_a(K)
    ictx.set_option("mitsuba_compare", 1)
    ictx.set_scene(s, m, c, em)
    pts = sphere_points((0, 0, 0), F.RECEIVER_R, 3000, 2)
    ictx.read_ray_count()
    _, traced = ictx.trace_irradiance(pts, spp=2)
    assert traced == 3000 * 2 * (1 + K)
    assert ictx.last_launch_count() == 2 and ictx.last_kernel_ms() > 0
    assert len(ictx.last_kernels()) == 1 and ictx.last_kernels()[0].startswith("k_fast_rays<")
    img = np.zeros((32, 32, 4), np.float32)
    drawn = ictx.draw(0, 1, 32, 32, img, mode=libs.MODE_FAST)
    assert ictx.read_ray_count() == traced + drawn

    sph, mats, cam, em = libs.reference_scene(160, 90)
    ictx.set_option("mitsuba_compare", 0)
    ictx.set_scene(sph, mats, cam, em)
    ictx.set_spp(1)                      # one reduction per pixel and per ray: bitwise repeatable
    rays = torch.from_numpy(camera_rays(cam, 160, 90, per_pixel=2, seed=9)).cuda()
    _, ppts, pids = lambert_hits(ictx, sph, mats, rays.cpu().numpy())
    ppts, pids = torch.from_numpy(ppts).cuda(), torch.from_numpy(pids.astype(np.int32)).cuda()

    def draw_and_trace():
        im = torch.zeros((90, 160, 4), dtype=torch.float32, device="cuda")
        ictx.draw(5, 1, 160, 90, im, mode=libs.MODE_FAST)
        r, _ = ictx.trace_rays(rays, spp=1, frame=5)
        return im.cpu().numpy(), r.cpu().numpy()

    im0, r0 = draw_and_trace()
    e0, _ = ictx.trace_irradiance(ppts, pids, spp=4, frame=1)
    im1, r1 = draw_and_trace()
    assert not bits_differ(im0, im1).any() and not bits_differ(r0[None], r1[None]).any()
    # ordered after a draw on another stream: draw -> irradiance (side stream) -> draw, as the two draws alone
    alone = torch.zeros((90, 160, 4), dtype=torch.float32, device="cuda")
    ictx.draw(0, 1, 160, 90, alone, flags=2, mode=libs.MODE_EXACT)
    ictx.draw(1, 1, 160, 90, alone, flags=2, mode=libs.MODE_EXACT)
    side = torch.cuda.Stream()
    mixed = torch.zeros((90, 160, 4), dtype=torch.float32, device="cuda")
    ictx.draw(0, 1, 160, 90, mixed, flags=2, mode=libs.MODE_EXACT, want_rays=False)
    e1 = ictx.trace_irradiance(ppts, pids, spp=4, frame=1, stream=side.cuda_stream, want_rays=False)
    ictx.draw(1, 1, 160, 90, mixed, flags=2, mode=libs.MODE_EXACT, stream=side.cuda_stream, want_rays=False)
    torch.cuda.synchronize()
    assert not bits_differ(alone.cpu().numpy(), mixed.cpu().numpy()).any()
    assert torch.allclose(e0, e1, rtol=1e-5, atol=0)
