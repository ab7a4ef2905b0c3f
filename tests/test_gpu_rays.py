"""tpt_trace_rays (Context.trace_rays): fast-mode radiance estimates for caller rays, checked where the answer is exact or
known — the furnace scene A per ray (value and ray count), the nearest hit of an emission-only scene against the float64
oracle of test_sweep_oracle.py, per-pixel averages of camera_rays against the exact image renderer, the closed forms B1
and B2 of tests/furnace.py on their quadrature-node rays — and the C-ABI behaviour around it (buffers, streams,
alignment, refusals, ordering with draws, accounting)."""
import ctypes

import numpy as np
import pytest
import torch

import furnace as F
from conftest import bits_differ, rel_l2
from test_gpu_configs import CLASS_NAMES, ExactPair, first_hit_classes, rl2
from test_gpu_fast import surface_rays
from test_gpu_sweep_oracle import _geom_bytes
import test_sweep_oracle as so
from toypathtracer_b200.scenes import camera_rays

pytestmark = pytest.mark.gpu


@pytest.fixture
def rctx(gpu_ctx):
    yield gpu_ctx
    for k, v in (("fast_kform", 2), ("mitsuba_compare", 0), ("light_sampling", 1)):
        gpu_ctx.set_option(k, v)


def _scaled(rays, seed):
    """The same rays with each direction multiplied by a random factor in [1e-3, 1e3]."""
    rng = np.random.default_rng(seed)
    out = rays.copy()
    out[:, 3:] = (rays[:, 3:].astype(np.float64) * 10.0 ** rng.uniform(-3, 3, (len(rays), 1))).astype(np.float32)
    return out


# ---- 1. furnace A per ray ------------------------------------------------------------------------------------------
def furnace_rays(n, seed):
    """n rays from the furnace camera's origin into its cone (every one meets the receiver with incidence cos >= 0.8), half
    of them with non-unit directions."""
    cam = F.furnace_camera(64, 64)
    rays = camera_rays(cam, 64, 64, per_pixel=-(-n // 4096), seed=seed)[:n]
    half = np.arange(n) % 2 == 1
    rays[half] = _scaled(rays[half], seed)
    return rays


def padded_furnace(n_lights, metal):
    """Scene A with 1 500 tiny non-emissive spheres inside the receiver: a blob past 64 KB (the 768-thread instance), and
    nothing a camera, bounce or shadow ray can reach."""
    s, m, c, em = F.furnace_scene(64, 64, n_lights, metal)
    k = 1500
    rng = np.random.default_rng(11)
    d = rng.normal(size=(k, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
    pad_s = np.zeros(k, s.dtype); pad_m = np.zeros(k, m.dtype)
    pad_s["center"] = d * 0.12 * rng.random((k, 1)); pad_s["radius"] = 0.001
    pad_s["invRadius"] = np.float32(1) / pad_s["radius"]
    pad_m["albedo"] = 0.5
    return np.concatenate([s, pad_s]), np.concatenate([m, pad_m]), c, em


def check_furnace(ctx, s, m, c, em, n_lights, ls, n, spp, frame=0, rays=None, label=""):
    ctx.set_option("mitsuba_compare", 1)
    ctx.set_option("light_sampling", 1 if ls else 0)
    ctx.set_scene(s, m, c, em)
    rays = furnace_rays(n, n + spp) if rays is None else rays
    dev = torch.from_numpy(rays).cuda()
    out, traced = ctx.trace_rays(dev, spp=spp, frame=frame)
    out = out.cpu().numpy()
    valid = np.isfinite(rays).all(1) & (np.abs(rays[:, 3:]).max(1) > 0)
    v = F.furnace_value(m).astype(np.float64)
    tol = v * (spp + 2) * 2.0 ** -23
    err = np.abs(out[valid, :3] - v)
    assert (err <= tol).all(), (label, int((err > tol).any(1).sum()), out[valid][(err > tol).any(1)][:4], v)
    assert (out[valid, 3] == 0).all(), label
    assert (out[~valid] == 0).all() and not np.signbit(out[~valid]).any(), label
    want = int(valid.sum()) * spp * F.furnace_rays_per_sample(m, n_lights, ls)
    assert traced == want, (label, traced, want)


def test_furnace_per_ray(rctx):
    for K in (0, 3, 300):
        for metal in (False, True):
            for ls in (True, False):
                s, m, c, em = F.furnace_scene(64, 64, K, metal)
                check_furnace(rctx, s, m, c, em, K, ls, 5000, 3, label=f"K{K} metal{metal} ls{ls}")
    s, m, c, em = F.furnace_scene(64, 64, 3, False)
    for kform in (0, 1, 2):
        rctx.set_option("fast_kform", kform)
        check_furnace(rctx, s, m, c, em, 3, True, 5000, 2, label=f"kform{kform}")
    rctx.set_option("fast_kform", 2)
    for K, metal, ls in ((3, False, True), (0, True, False), (300, False, True)):
        s, m, c, em = padded_furnace(K, metal)
        assert _geom_bytes(len(s), K) + 2 * len(s) * 16 > 64 * 1024
        check_furnace(rctx, s, m, c, em, K, ls, 5000, 2, label=f"padded K{K} metal{metal} ls{ls}")


def test_furnace_counts_and_tails(rctx):
    s, m, c, em = F.furnace_scene(64, 64, 3, False)
    for spp in (1, 3, 7):
        for n in (1, 63, 65, 100_003):
            check_furnace(rctx, s, m, c, em, 3, True, n, spp, frame=spp, label=f"spp{spp} n{n}")


def test_untraceable_rays_give_zero_and_no_rays(rctx):
    s, m, c, em = F.furnace_scene(64, 64, 3, False)
    rays = furnace_rays(1000, 5)
    bad = [(3, 0.0), (3, np.nan), (4, np.inf), (5, -np.inf), (0, np.nan), (1, np.inf)]
    for i in range(0, 1000, 3):            # every third ray broken, in runs that straddle the 64-ray slabs
        col, val = bad[(i // 3) % len(bad)]
        if col == 3 and val == 0.0:
            rays[i, 3:] = 0.0              # zero-length direction
        else:
            rays[i, col] = val
    check_furnace(rctx, s, m, c, em, 3, True, len(rays), 3, rays=rays, label="broken rays")
    tiny = furnace_rays(2, 6)
    tiny[1, 3:] = (1e-30, -1e-30, 1e-30)    # squared length underflows: does not normalise
    out, traced = rctx.trace_rays(tiny, spp=2)
    assert traced == 2 * F.furnace_rays_per_sample(m, 3, True) and (out[1] == 0).all() and (out[0, :3] > 0).all()


# ---- 2. nearest hit against the float64 oracle -----------------------------------------------------------------------
DIR_ERR = 2.0 ** -19     # |normalize(d) - d/|d|| on the GPU (rsqrt.approx, the scaling and dot product), generously


def emission_scene(count, layout):
    """make_scene geometry with every sphere Lambert, albedo 0 and emission (id + 1, 8, 0.5): with light sampling off a
    ray's radiance is the emission of its nearest sphere, or the sky (green <= 0.3) on a miss."""
    sph, mats, cam, dup = so.make_scene(count, layout)
    mats = np.zeros(count, mats.dtype)
    mats["emissive"][:, 0] = np.arange(1, count + 1)
    mats["emissive"][:, 1] = 8.0
    mats["emissive"][:, 2] = 0.5
    return sph, mats, cam, dup


def decode(out):
    """id per ray: the nearest sphere, -1 for the sky, -2 for anything else."""
    hit = out[:, 1] == 8.0
    ids = np.where(hit, out[:, 0].astype(np.int64) - 1, -1)
    sky = (~hit) & (out[:, 1] > 0.2) & (out[:, 1] <= 0.3 + 1e-6)
    return np.where(hit | sky, ids, -2)


def sky64(d):
    d = d.astype(np.float64)
    d = d / np.linalg.norm(d, axis=1, keepdims=True)
    return F.gradient_sky(d[:, 1])


def oracle(monkeypatch, rays, sph):
    """The float64 nearest-hit oracle with the kernel's renormalisation of the direction added to its error bounds: the
    kernel sweeps with normalize(d), which differs from d / |d| by <= DIR_ERR, moving nb by <= DIR_ERR |s - o|."""
    orig = so.pair_bounds

    def widened(o, d, s, r2, expanded=True):
        nb, c, enb, ec = orig(o, d, s, r2, expanded)
        return nb, c, enb + DIR_ERR * np.sqrt(((s - o) ** 2).sum(-1)), ec

    monkeypatch.setattr(so, "pair_bounds", widened)
    try:
        return so.nearest_hit(rays, sph)
    finally:
        monkeypatch.setattr(so, "pair_bounds", orig)


def max_queue_count(n_lights):
    """Largest scene the slab queue stages: 768-thread CTA, [geometry | 24 warps x 2 KB of ray buffers] within the 227 KB
    of dynamic shared memory a block may have (less 2 KB for the kernel's static arrays)."""
    c = 4
    while ((_geom_bytes(c + 4, n_lights) + 127) // 128 * 128 + 24 * 2048 + 2048 <= 232448):
        c += 4
    return c


HIT_CASES = [(46, "compact", (0, 1, 2)), (46, "spread", (2,)), (1300, "compact", (2,)), (1300, "spread", (2,)),
             ("max", "compact", (2,)), ("max", "spread", (2,))]


@pytest.mark.parametrize("count,layout,kforms", HIT_CASES, ids=[f"{c}-{l}" for c, l, _ in HIT_CASES])
def test_nearest_hit_against_oracle(rctx, monkeypatch, count, layout, kforms):
    """46 spheres: 128-thread instances (KFORM 0/1/2 compact, 3 spread); 1 300: past 64 KB of blob, 768 threads (KFORM 2 /
    3); the largest stageable count: 768 threads on the expanded / reference form."""
    count = max_queue_count(0) if count == "max" else count
    sph, mats, cam, dup = emission_scene(count, layout)
    assert so.gate_passes(sph) == (layout == "compact")
    rctx.set_option("light_sampling", 0)
    rctx.set_option("mitsuba_compare", 0)
    rctx.set_scene(sph, mats, cam, np.zeros(0, np.int32))      # emissive everywhere, but no light table
    seed = 300 + count
    n = int(np.clip(300_000 / count, 64, 3000))
    surf = surface_rays(sph, 4 * n, seed)
    aimed, target = so.aimed_rays(sph, seed + 5)
    sets = {"surface": surf[np.isfinite(surf).all(1)], "tangent": so.near_tangent_rays(sph, n, seed + 1)[0],
            "degenerate": so.degenerate_rays(sph, seed + 3), "aimed": aimed}
    for kform in kforms:
        rctx.set_option("fast_kform", kform)
        for name, rays in sets.items():
            ids, outs = {}, {}
            for scaled in (False, True):
                r = _scaled(rays, seed) if scaled else rays
                out, _ = rctx.trace_rays(torch.from_numpy(r).cuda(), spp=1)
                outs[scaled] = out.cpu().numpy()
                ids[scaled] = decode(outs[scaled])
                if name == "aimed":
                    assert (ids[scaled] == target).all(), (count, layout, kform, scaled, "aimed")
            if name == "aimed" and count > 2048:
                continue                 # the geometric construction alone decides these
            ora = oracle(monkeypatch, rays, sph)
            well = ora["well"]
            if name == "surface":
                assert well.mean() > 0.6, (count, layout, well.mean())     # the oracle decides most of them
            for scaled in (False, True):
                bad = well & (ids[scaled] != ora["id"])
                assert not bad.any(), (count, layout, kform, name, scaled, int(bad.sum()), ids[scaled][bad][:8], ora["id"][bad][:8])
            # a miss returns the sky of the direction
            miss = well & (ora["id"] == -1)
            if miss.any():
                sky = sky64(rays[miss, 3:])
                for scaled in (False, True):
                    assert (np.abs(outs[scaled][miss, :3] - sky) <= 1e-6 * sky).all(), (count, layout, name, scaled)


# ---- 3. equivalence with the image renderer ------------------------------------------------------------------------
EW, EH = 320, 180


@pytest.mark.parametrize("ls", [1, 0])
def test_camera_rays_average_to_the_exact_image(rctx, libs, ls):
    """Per-pixel means of camera_rays (128 rays per pixel x 8 calls at spp 1 = 1 024 independent camera rays: samples that
    share a camera ray would not be independent in the pixel and lens) against exact mode at 1 024 spp, with the bars
    test_gpu_configs applies to the fast mode: relL2 <= 1.10 x the exact-vs-exact floor, and every first-hit-material
    region's mean within max(6 sigma, 2e-4 relative) of the 2 048-spp exact mean."""
    sph, mats, cam, em = libs.reference_scene(EW, EH)
    rctx.set_option("light_sampling", ls)
    rctx.set_scene(sph, mats, cam, em)
    ex = ExactPair(rctx, EW, EH, 256)
    P, S, calls = 128, 1, 8
    acc = torch.zeros((EH * EW, 4), dtype=torch.float64, device="cuda")
    for k in range(calls):
        rays = torch.from_numpy(libs.camera_rays(cam, EW, EH, per_pixel=P, seed=100 + k)).cuda()
        out, _ = rctx.trace_rays(rays, spp=S, frame=k)
        acc += out.view(EH * EW, P, 4).double().mean(1)
    img = (acc / calls).cpu().numpy().reshape(EH, EW, 4)[..., :3]
    assert np.isfinite(img).all()
    floor = rl2(ex.B, ex.A)
    r = rl2(img, ex.A)
    assert r <= 1.10 * floor, (ls, r, floor)
    cls = first_hit_classes(sph, mats, cam, EW, EH)
    for k, name in enumerate(CLASS_NAMES):
        msk = cls == k
        npx = int(msk.sum())
        if npx < 200:
            continue
        mean_f, mean_c = img[msk].mean(axis=0), ex.C[msk].mean(axis=0)
        se = np.sqrt(ex.var_px[msk].sum(axis=0) * 1.5) / npx
        assert (np.abs(mean_f - mean_c) <= np.maximum(6 * se, 2e-4 * mean_c)).all(), (ls, name, mean_f, mean_c, se)


# ---- 4. closed forms B1, B2 ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("scene", ["b1_ls", "b1_nols", "b2"])
def test_closed_forms_on_quadrature_rays(rctx, scene):
    """The quadrature-node rays of furnace.footprint_hits, weighted by their Gauss-Legendre weights, estimate exactly the
    per-pixel integral the B expectations compute: 32 batches of 16 nodes x 64 spp, per-bin means within max(5 se, 1e-4 E)."""
    s, m, c, em, w, h, e, bins, mitsuba, ls = F.b_case(scene)
    rctx.set_option("mitsuba_compare", 1 if mitsuba else 0)
    rctx.set_option("light_sampling", 1 if ls else 0)
    rctx.set_scene(s, m, c, em)
    _, wq, d = F.footprint_hits(c, w, h)
    o = np.broadcast_to(c["origin"][0].astype(np.float64), d.shape)
    rays = torch.from_numpy(np.concatenate([o, d], -1).reshape(-1, 6).astype(np.float32)).cuda()
    wt = torch.from_numpy(wq).cuda()
    batches = []
    for b in range(32):
        out, _ = rctx.trace_rays(rays, spp=64, frame=b)
        px = (out[:, :3].double().view(h, w, len(wq), 3) * wt[None, None, :, None]).sum(2)
        batches.append(px.cpu().numpy())
    F.check_bins(np.array(batches), e, bins)


# ---- 5. API behaviour ----------------------------------------------------------------------------------------------
def furnace_ctx(ctx, K=3):
    s, m, c, em = F.furnace_scene(64, 64, K, False)
    ctx.set_option("mitsuba_compare", 1)
    ctx.set_scene(s, m, c, em)
    return F.furnace_value(m), F.furnace_rays_per_sample(m, K, True)


def golden_ctx(ctx, libs):
    sph, mats, cam, em = libs.reference_scene(160, 90)
    ctx.set_scene(sph, mats, cam, em)
    return libs.camera_rays(cam, 160, 90, per_pixel=2, seed=1)


def test_buffer_kinds_agree(rctx, libs):
    """Host numpy (pageable and page-locked), torch CUDA on a side stream, a device row slice at an odd row offset (8-byte
    aligned) and DevicePtr buffers all give the same estimates (spp 1: one reduction per output, the same bits)."""
    rays = golden_ctx(rctx, libs)
    n = len(rays)
    ref, traced = rctx.trace_rays(rays, spp=1, frame=3)
    assert isinstance(ref, np.ndarray) and ref.shape == (n, 4) and np.isfinite(ref).all() and (ref[:, 3] == 0).all()
    assert traced > n
    pin_r = torch.empty((n, 6), dtype=torch.float32, pin_memory=True); pin_r.numpy()[...] = rays
    pin_o = torch.empty((n, 4), dtype=torch.float32, pin_memory=True)
    out, t2 = rctx.trace_rays(pin_r, spp=1, frame=3, out=pin_o)
    assert out is pin_o and t2 == traced and not bits_differ(pin_o.numpy()[None], ref[None]).any()
    side = torch.cuda.Stream()
    base = torch.zeros((n + 1, 6), dtype=torch.float32, device="cuda")
    base[1:] = torch.from_numpy(rays).cuda()
    sl = base[1:]
    assert sl.data_ptr() % 16 == 8
    torch.cuda.synchronize()
    dev_out = rctx.trace_rays(sl, spp=1, frame=3, stream=side.cuda_stream, want_rays=False)
    assert dev_out.is_cuda and dev_out.shape == (n, 4)
    side.synchronize()
    assert not bits_differ(dev_out.cpu().numpy()[None], ref[None]).any()
    rp = rctx.mem_alloc(n * 24); op = rctx.mem_alloc(n * 16)
    try:
        rctx.mem_from_host(rp, rays)
        _, t3 = rctx.trace_rays(rp, spp=1, frame=3, out=op, n=n)
        got = rctx.mem_to_host(op, np.empty((n, 4), np.float32))
    finally:
        rctx.mem_free(rp); rctx.mem_free(op)
    assert t3 == traced and not bits_differ(got[None], ref[None]).any()


def test_frames_and_determinism(rctx, libs):
    rays = golden_ctx(rctx, libs)
    a, ra = rctx.trace_rays(rays, spp=4, frame=7)
    b, rb = rctx.trace_rays(rays, spp=4, frame=7)
    c, _ = rctx.trace_rays(rays, spp=4, frame=8)
    assert np.allclose(a, b, rtol=1e-5, atol=0) and ra == rb
    assert (a != c).mean() > 0.5
    # frames average progressively: the mean of 8 frames is closer to a 64-frame reference than one frame is
    ref = np.mean([rctx.trace_rays(rays, spp=4, frame=100 + f)[0] for f in range(64)], axis=0)
    m8 = np.mean([rctx.trace_rays(rays, spp=4, frame=f)[0] for f in range(8)], axis=0)
    assert rel_l2(m8[None], ref[None]) < 0.5 * rel_l2(a[None], ref[None])


def test_refusals(rctx, libs):
    furnace_ctx(rctx)
    L, h = rctx._L, rctx._h
    dev = torch.zeros((70, 6), dtype=torch.float32, device="cuda")
    dout = torch.zeros((70, 4), dtype=torch.float32, device="cuda")
    r, o = ctypes.c_void_p(dev.data_ptr()), ctypes.c_void_p(dout.data_ptr())
    cnt = ctypes.c_longlong(-1)

    def call(rays, ron, n, spp, out, oon):
        return L.tpt_trace_rays(h, rays, ron, n, spp, 0, out, oon, ctypes.byref(cnt), None)

    def refused(text, *args):
        assert call(*args) != 0
        assert text in L.tpt_last_error(h).decode(), (text, L.tpt_last_error(h).decode())

    refused("null rays6 or out4", None, 1, 4, 1, o, 1)
    refused("null rays6 or out4", r, 1, 4, 1, None, 1)
    refused("n < 0", r, 1, -1, 1, o, 1)
    refused("spp < 1", r, 1, 4, 0, o, 1)
    refused("n * spp > 2^32", r, 1, (1 << 31) + 1, 2, o, 1)
    refused("n * spp > 2^32", r, 1, 1 << 32, 1, o, 1)
    refused("out4 is not 16-byte aligned", r, 1, 4, 1, ctypes.c_void_p(dout.data_ptr() + 4), 1)
    refused("rays6 is not 4-byte aligned", ctypes.c_void_p(dev.data_ptr() + 2), 1, 4, 1, o, 1)
    host = np.zeros((4, 6), np.float32)
    refused("rays6 is not CUDA memory", ctypes.c_void_p(host.ctypes.data), 1, 4, 1, o, 1)
    if torch.cuda.device_count() > 1:
        other = torch.zeros((4, 4), dtype=torch.float32, device="cuda:1")
        refused("lives on device 1", r, 1, 4, 1, ctypes.c_void_p(other.data_ptr()), 1)
    with pytest.raises(libs.TptError, match="spp < 1"):
        rctx.trace_rays(np.zeros((4, 6), np.float32), spp=0)
    # n == 0: nothing launched, no rays
    cnt.value = -1
    assert call(ctypes.c_void_p(host.ctypes.data), 0, 0, 4, ctypes.c_void_p(host.ctypes.data), 0) == 0
    assert cnt.value == 0 and rctx.last_launch_count() == 0
    out, traced = rctx.trace_rays(np.zeros((0, 6), np.float32))
    assert out.shape == (0, 4) and traced == 0


def test_accounting_and_scene_changes(rctx, libs):
    v, rps = furnace_ctx(rctx)
    rays = furnace_rays(3000, 2)
    rctx.read_ray_count()
    out, traced = rctx.trace_rays(rays, spp=2)
    assert traced == 3000 * 2 * rps
    assert rctx.last_launch_count() == 2                     # the trace kernel and the counter fold
    assert rctx.last_kernel_ms() > 0
    img = np.zeros((32, 32, 4), np.float32)
    drawn = rctx.draw(0, 1, 32, 32, img, mode=libs.MODE_FAST)
    assert rctx.read_ray_count() == traced + drawn
    # set_scene between calls takes effect: another albedo, another furnace value
    s, m, c, em = F.furnace_scene(64, 64, 3, False)
    m["albedo"][0] = (0.3, 0.9, 0.5)
    rctx.set_scene(s, m, c, em)
    out2, _ = rctx.trace_rays(rays, spp=2)
    v2 = F.furnace_value(m)
    assert np.allclose(out[:, :3], v, rtol=1e-6) and np.allclose(out2[:, :3], v2, rtol=1e-6)


@pytest.mark.parametrize("mode", ["exact", "fast"])
def test_draws_around_a_trace_are_unchanged(rctx, libs, mode):
    """draw -> trace_rays -> draw on one context leaves the image as the two draws alone do: bit for bit in exact mode,
    within the float sum order of the L2 reductions in fast mode. Device image, the context's stream and a side stream."""
    sph, mats, cam, em = libs.reference_scene(160, 90)
    rctx.set_scene(sph, mats, cam, em)
    md = libs.MODE_EXACT if mode == "exact" else libs.MODE_FAST
    rays = torch.from_numpy(libs.camera_rays(cam, 160, 90, per_pixel=4, seed=9)).cuda()
    alone = torch.zeros((90, 160, 4), dtype=torch.float32, device="cuda")
    rctx.draw(0, 1, 160, 90, alone, flags=2, mode=md)
    rctx.draw(1, 1, 160, 90, alone, flags=2, mode=md)
    side = torch.cuda.Stream()
    mixed = torch.zeros((90, 160, 4), dtype=torch.float32, device="cuda")
    rctx.draw(0, 1, 160, 90, mixed, flags=2, mode=md, want_rays=False)
    rctx.trace_rays(rays, spp=8, stream=side.cuda_stream, want_rays=False)
    rctx.draw(1, 1, 160, 90, mixed, flags=2, mode=md, stream=side.cuda_stream, want_rays=False)
    torch.cuda.synchronize()
    a, b = alone.cpu().numpy(), mixed.cpu().numpy()
    if mode == "exact":
        assert not bits_differ(a, b).any()
    else:
        assert rel_l2(b, a) < 1e-5
