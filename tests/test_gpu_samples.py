"""tpt_draw_samples (Context.draw_samples) and Context.render_adaptive, checked where the answer is exact or known: the
fast draw's own image (same samples), the furnace scene A per entry (sums, squares and ray counts exact), scene B2's
closed form for the binned means, the variance across independent frames for the second moments, lists against
all-pixel calls (continuation), the 4096-spp exact image for the adaptive render — and the C-ABI around it (buffer kinds,
accumulation, refusals, accounting)."""
import numpy as np
import pytest
import torch
from scipy import stats

import furnace as F
from conftest import rel_l2
from test_gpu_configs import ExactPair, first_hit_classes
from test_gpu_rays import padded_furnace

pytestmark = pytest.mark.gpu


@pytest.fixture
def sctx(gpu_ctx):
    yield gpu_ctx
    for k, v in (("fast_kform", 2), ("mitsuba_compare", 0), ("light_sampling", 1), ("fast_variant", -1)):
        gpu_ctx.set_option(k, v)
    gpu_ctx.set_spp(4)


def zeros4(n):
    return torch.zeros((n, 4), dtype=torch.float32, device="cuda")


# ---- the draw's own samples ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("scene", ["46-1280x720", "stress4096-640x360"])
def test_same_samples_as_the_draw(sctx, libs, scene):
    w, h = (1280, 720) if scene.startswith("46") else (640, 360)
    sph, mats, cam, em = libs.reference_scene(w, h) if scene.startswith("46") else libs.stress_scene(w, h, count=4096)
    sctx.set_scene(sph, mats, cam, em)
    sctx.set_option("fast_variant", 3)
    for frame in (0, 7):
        img = torch.full((h, w, 4), 5.0, dtype=torch.float32, device="cuda")
        drawn = sctx.draw(frame, 1, w, h, img, flags=0, mode=libs.MODE_FAST)       # flags 0: `prev` has weight 0
        (s, q), traced = sctx.draw_samples(frame, w, h)
        s, q, img = s.cpu().numpy().astype(np.float64), q.cpu().numpy(), img.view(-1, 4).cpu().numpy().astype(np.float64)
        assert (s[:, 3] == sctx.spp).all() and (q[:, 3] == 0).all()
        mean = s[:, :3] / sctx.spp
        err = np.abs(mean - img[:, :3])
        bad = (err > 1e-5 * img[:, :3] + 1e-30).any(1)
        # different kernel instances may contract the shading code differently (DESIGN §3.1a): a path that then takes
        # another turn changes its pixel and, almost always, the ray count
        assert abs(traced - drawn) <= 2e-6 * drawn, (scene, frame, traced, drawn)
        assert int(bad.sum()) <= abs(traced - drawn), (scene, frame, int(bad.sum()), traced - drawn)
        # the second moment is consistent with the sum: sum^2 / n <= sq <= sum^2 (non-negative samples)
        sq = q[:, :3].astype(np.float64)
        assert (sq >= s[:, :3] ** 2 / sctx.spp * (1 - 1e-5)).all() and (sq <= s[:, :3] ** 2 * (1 + 1e-5) + 1e-30).all()


# ---- furnace A: every sample is exactly albedo * sky -----------------------------------------------------------------
def check_furnace_entries(ctx, m, n_lights, ls, w, h, pixels, spp, frame=0):
    dev = None if pixels is None else torch.from_numpy(pixels).cuda()
    (s, q), traced = ctx.draw_samples(frame, w, h, dev, spp)
    s, q = s.cpu().numpy().astype(np.float64), q.cpu().numpy().astype(np.float64)
    n = w * h if pixels is None else len(pixels)
    v = F.furnace_value(m).astype(np.float64)
    assert (s[:, 3] == spp).all() and (q[:, 3] == 0).all()
    tol = v * spp * (spp + 2) * 2.0 ** -23
    assert (np.abs(s[:, :3] - spp * v) <= tol).all(), (n_lights, ls, s[:4], spp * v)
    assert (np.abs(q[:, :3] - spp * v * v) <= 4 * v * tol).all(), (n_lights, ls, q[:4], spp * v * v)
    var = (q[:, :3] - s[:, :3] ** 2 / spp) / max(spp - 1, 1)
    assert (np.abs(var) <= 1e-6 * spp * v * v).all()
    assert traced == n * spp * F.furnace_rays_per_sample(m, n_lights, ls), (traced, n, spp)
    return s, q


def furnace_lists(w, h, seed):
    rng = np.random.default_rng(seed)
    return {"one": np.array([w * h // 2 + 3], np.int32),
            "tail": rng.permutation(w * h)[:200].astype(np.int32),                  # unsorted, 200 = 3 x 64 + 8
            "dups": np.repeat(rng.integers(0, w * h, 70).astype(np.int32), 3),     # 210 entries, each pixel 3 x
            "big": rng.integers(0, w * h, 5001).astype(np.int32)}


def test_furnace_exact_per_entry(sctx):
    w, h = 64, 64
    sctx.set_option("mitsuba_compare", 1)
    for K in (0, 3, 300):
        for metal in (False, True):
            for ls in (True, False):
                s, m, c, em = F.furnace_scene(w, h, K, metal)
                sctx.set_option("light_sampling", 1 if ls else 0)
                sctx.set_scene(s, m, c, em)
                for name, px in furnace_lists(w, h, K).items():
                    check_furnace_entries(sctx, m, K, ls, w, h, px, 3, frame=K)
                check_furnace_entries(sctx, m, K, ls, w, h, None, 2)
    sctx.set_option("light_sampling", 1)
    for kform in (0, 1):
        sctx.set_option("fast_kform", kform)
        s, m, c, em = F.furnace_scene(w, h, 3, False)
        sctx.set_scene(s, m, c, em)
        check_furnace_entries(sctx, m, 3, True, w, h, furnace_lists(w, h, 1)["tail"], 5)
    sctx.set_option("fast_kform", 2)
    for K, metal, ls in ((3, False, True), (0, True, False), (300, False, True)):
        s, m, c, em = padded_furnace(K, metal)          # past 64 KB of blob: the 768-thread instance
        sctx.set_option("light_sampling", 1 if ls else 0)
        sctx.set_scene(s, m, c, em)
        check_furnace_entries(sctx, m, K, ls, w, h, furnace_lists(w, h, 2)["dups"], 2)
        check_furnace_entries(sctx, m, K, ls, w, h, None, 1)


def test_furnace_long_list_picks_the_8_cta_instance(sctx):
    """Enough slabs per warp for pick_queue's 64-register instance (KFORM 2, >= 48 slabs per warp)."""
    w, h = 64, 64
    sctx.set_option("mitsuba_compare", 1)
    s, m, c, em = F.furnace_scene(w, h, 3, False)
    sctx.set_scene(s, m, c, em)
    px = np.random.default_rng(3).integers(0, w * h, 400_000).astype(np.int32)
    check_furnace_entries(sctx, m, 3, True, w, h, px, 40)


def test_host_and_device_buffers_accumulate_alike(sctx):
    w, h = 64, 64
    sctx.set_option("mitsuba_compare", 1)
    s, m, c, em = F.furnace_scene(w, h, 3, False)
    sctx.set_scene(s, m, c, em)
    v = F.furnace_value(m).astype(np.float64)
    px = furnace_lists(w, h, 4)["tail"]
    hs = np.zeros((len(px), 4), np.float32); hs[:, 0] = 1.0
    hq = np.zeros((len(px), 4), np.float32)
    ds, dq = torch.from_numpy(hs.copy()).cuda(), zeros4(len(px))
    ts = torch.from_numpy(hs.copy())                      # torch CPU tensors, without moments
    for f in range(3):
        (_, _), r = sctx.draw_samples(f, w, h, px, 2, hs, hq)
        sctx.draw_samples(f, w, h, torch.from_numpy(px).cuda(), 2, ds, dq)
        sctx.draw_samples(f, w, h, torch.from_numpy(px), 2, ts)
        assert r == len(px) * 2 * 5
    for got in (hs, ds.cpu().numpy(), ts.numpy()):
        assert (got[:, 3] == 6).all()
        assert np.allclose(got[:, :3], 6 * v + np.array([1.0, 0, 0]), rtol=1e-6, atol=0)
    assert np.array_equal(hq, dq.cpu().numpy()) or np.allclose(hq, dq.cpu().numpy(), rtol=1e-6, atol=0)
    # DevicePtr buffers with n
    dp = torch.from_numpy(px).cuda()
    s2 = zeros4(len(px))
    sctx.draw_samples(0, w, h, libs_devptr(dp), 2, libs_devptr(s2), n=len(px))
    assert np.allclose(s2.cpu().numpy()[:, :3], 2 * v, rtol=1e-6, atol=0)


def libs_devptr(t):
    import toypathtracer_b200 as tpt
    return tpt.DevicePtr(t.data_ptr())


# ---- moments on B2 ---------------------------------------------------------------------------------------------------
def test_b2_binned_means_and_moments(sctx):
    s, m, c, em, w, h, E, bins, mitsuba, ls = F.b_case("b2")
    sctx.set_option("mitsuba_compare", 1 if mitsuba else 0)
    sctx.set_option("light_sampling", 1 if ls else 0)
    sctx.set_scene(s, m, c, em)
    batches = []
    for f in range(16):
        (sm, _), _ = sctx.draw_samples(f, w, h, None, 16)
        sm = sm.cpu().numpy().astype(np.float64)
        batches.append((sm[:, :3] / sm[:, 3:]).reshape(h, w, 3))
    F.check_bins(np.stack(batches), E, bins)
    # per-pixel variance from the moments of one 64-sample call vs the spread of 32 independent single samples
    px = np.random.default_rng(9).permutation(w * h)[:300].astype(np.int32)
    dpx = torch.from_numpy(px).cuda()
    (sa, qa), _ = sctx.draw_samples(100, w, h, dpx, 64)
    sa, qa = sa.cpu().numpy().astype(np.float64), qa.cpu().numpy().astype(np.float64)
    var_a = (qa[:, :3] - sa[:, :3] ** 2 / 64) / 63
    singles = np.stack([sctx.draw_samples(200 + k, w, h, dpx, 1)[0][0].cpu().numpy()[:, :3] for k in range(32)]).astype(np.float64)
    var_b = singles.var(axis=0, ddof=1)
    # the gradient sky's blue is 1 in every direction, so every blue sample is the receiver's albedo: zero variance
    mean_b = sa[:, 2] / 64
    assert (np.abs(var_a[:, 2]) <= 1e-5 * mean_b ** 2).all() and (var_b[:, 2] <= 1e-5 * mean_b ** 2).all()
    var_a, var_b = var_a[:, :2], var_b[:, :2]
    assert (var_a > 0).all() and (var_b > 0).all()
    ratio = var_a / var_b                                   # ~ F(63, 31) per pixel and channel
    lo, hi = stats.f.ppf([1e-6, 1 - 1e-6], 63, 31)
    assert ((ratio > lo) & (ratio < hi)).all(), (ratio.min(), ratio.max(), lo, hi)
    # pooled over the 600 pixel-channels: the ratio of the summed variances, well inside a chi-square-based band
    assert abs(np.log(var_a.sum() / var_b.sum())) < 0.15, var_a.sum() / var_b.sum()


# ---- continuation ----------------------------------------------------------------------------------------------------
def test_list_continues_the_all_pixel_call(sctx, libs):
    w, h = 1280, 720
    sph, mats, cam, em = libs.reference_scene(w, h)
    sctx.set_scene(sph, mats, cam, em)
    rng = np.random.default_rng(5)
    px = np.concatenate([rng.permutation(w * h)[:6000], rng.integers(0, w * h, 1000)]).astype(np.int32)
    for frame in (3, 11):
        (sa, qa), _ = sctx.draw_samples(frame, w, h, None, 4)
        (sl, ql), _ = sctx.draw_samples(frame, w, h, torch.from_numpy(px).cuda(), 4)
        sa, qa = sa.cpu().numpy()[px].astype(np.float64), qa.cpu().numpy()[px].astype(np.float64)
        sl, ql = sl.cpu().numpy().astype(np.float64), ql.cpu().numpy().astype(np.float64)
        assert (sl[:, 3] == 4).all()
        assert (np.abs(sl - sa) <= 1e-6 * sa + 1e-30).all(), np.abs(sl - sa).max()
        assert (np.abs(ql - qa) <= 1e-6 * qa + 1e-30).all(), np.abs(ql - qa).max()
    # the ray count is the subset's share: exact in scene A
    s, m, c, em = F.furnace_scene(64, 64, 3, False)
    sctx.set_option("mitsuba_compare", 1)
    sctx.set_scene(s, m, c, em)
    _, all_rays = sctx.draw_samples(0, 64, 64, None, 4)
    sub = px[px < 4096][:777]
    _, sub_rays = sctx.draw_samples(0, 64, 64, torch.from_numpy(sub).cuda(), 4)
    assert all_rays * len(sub) == sub_rays * 64 * 64


# ---- adaptive against uniform ----------------------------------------------------------------------------------------
def pixel_err(img, ref):
    lum = np.array([0.2126, 0.7152, 0.0722])
    return np.abs((img - ref) @ lum) / (ref @ lum + 0.05)


def test_adaptive_beats_uniform_at_equal_rays(sctx, libs):
    w, h = 640, 360
    sph, mats, cam, em = libs.reference_scene(w, h)
    sctx.set_scene(sph, mats, cam, em)
    ex = ExactPair(sctx, w, h, 1024)                           # two 4096-spp exact images
    ref = ex.A.reshape(-1, 3)
    img, spp_map, rays = sctx.render_adaptive(w, h, base_spp=4, max_spp=64, rel_err=0.05, frame=0)
    img = img.view(-1, 4).cpu().numpy().astype(np.float64)
    spp_map = spp_map.view(-1).cpu().numpy()
    assert (img[:, 3] == 0).all() and spp_map.min() >= 4 and spp_map.max() <= 64 and (spp_map % 4 == 0).all()
    # uniform: the fewest samples per pixel that trace at least as many rays
    (s4, _), r4 = sctx.draw_samples(100, w, h, None, 4)
    u = 4
    while r4 * u / 4 < rays:
        u += 1
    (su, _), ru = sctx.draw_samples(200, w, h, None, u)
    assert ru >= rays * 0.99, (ru, rays, u)
    uni = su.cpu().numpy().astype(np.float64)
    uni = uni[:, :3] / uni[:, 3:]
    a_l2, u_l2 = rel_l2(img[:, :3], ref), rel_l2(uni, ref)
    a90, u90 = np.percentile(pixel_err(img[:, :3], ref), 90), np.percentile(pixel_err(uni, ref), 90)
    report = dict(rays=rays, uniform_spp=u, uniform_rays=ru, mean_spp=float(spp_map.mean()),
                  relL2=(a_l2, u_l2), p90=(a90, u90), floor=rel_l2(ex.B, ex.A))
    print(report)
    assert a_l2 < u_l2 and a90 < u90, report
    # bias: region means against the 8192-spp exact mean, bar max(5 se, 1e-4 E) plus the stopping-rule allowance
    # rel_err * (E + 0.05) (a stopped pixel sits within about one of its own standard errors, which the rule caps)
    cls = first_hit_classes(sph, mats, cam, w, h).reshape(-1)
    var1 = ex.var_px.reshape(-1, 3) * 4096                     # per-sample variance estimate
    for k in range(5):
        msk = cls == k
        nk = int(msk.sum())
        if nk < 200:
            continue
        mean_a, mean_c = img[msk, :3].mean(0), ex.C.reshape(-1, 3)[msk].mean(0)
        se = np.sqrt((var1[msk] / spp_map[msk, None]).sum(0)) / nk
        bar = np.maximum(5 * se, 1e-4 * mean_c) + 0.05 * (mean_c + 0.05)
        assert (np.abs(mean_a - mean_c) <= bar).all(), (k, mean_a, mean_c, se)


# ---- ordering with torch's streams -----------------------------------------------------------------------------------
SPIN = 200_000_000          # torch.cuda._sleep cycles: ~0.1 s of a spinning kernel ahead of the call on a torch stream


def test_calls_are_ordered_with_torch_streams(sctx):
    """The buffers draw_samples allocates are zeroed, and the lists render_adaptive builds are converted, by torch on its
    own streams. With a long kernel queued ahead on that stream, a call that did not wait for the fill would have its
    sums zeroed after the fact, and a list read before its conversion would hold stale indices."""
    w, h = 64, 64
    sctx.set_option("mitsuba_compare", 1)
    s, m, c, em = F.furnace_scene(w, h, 3, False)
    sctx.set_scene(s, m, c, em)
    v = F.furnace_value(m).astype(np.float64)

    def check(sums, n, spp):
        sums = sums.cpu().numpy().astype(np.float64)
        assert sums.shape == (n, 4) and (sums[:, 3] == spp).all(), sums[:3]
        assert np.allclose(sums[:, :3], spp * v, rtol=1e-6, atol=0), sums[:3]

    side = torch.cuda.Stream()
    for current in (torch.cuda.default_stream(), side):
        with torch.cuda.stream(current):
            torch.cuda.synchronize()
            torch.cuda._sleep(SPIN)                          # outputs allocated here: their fill waits behind the spin
            (s4, _), r = sctx.draw_samples(0, w, h, None, 2)
            check(s4, w * h, 2)
            torch.cuda._sleep(SPIN)                          # caller's buffer zeroed behind the spin, no ray count
            own = torch.empty((w * h, 4), device="cuda").zero_()
            sctx.draw_samples(1, w, h, None, 2, own, want_rays=False)
            check(own, w * h, 2)                             # read by torch after the call, on the same stream
            torch.cuda._sleep(SPIN)                          # a list written by torch kernels behind the spin
            idx = (torch.arange(300, device="cuda") * 13 % (w * h)).to(torch.int32)
            (sl, _), _ = sctx.draw_samples(2, w, h, idx, 3)
            check(sl, 300, 3)
            torch.cuda._sleep(SPIN)
            img, spp, rays = sctx.render_adaptive(w, h, base_spp=2, max_spp=8, rel_err=0.05, frame=3)
            assert (spp == 2).all() and rays == w * h * 2 * 5        # every sample equal: no pixel is refined
            assert np.allclose(img.view(-1, 4).cpu().numpy()[:, :3], v, rtol=1e-6, atol=0)
    # an explicit stream while torch's current stream is busy: the outputs are zeroed on the call's stream
    torch.cuda.synchronize()
    torch.cuda._sleep(SPIN)
    (s4, _), _ = sctx.draw_samples(4, w, h, None, 2, stream=side.cuda_stream)
    side.synchronize()
    check(s4, w * h, 2)
    torch.cuda.synchronize()


# ---- refusals and accounting -----------------------------------------------------------------------------------------
def test_refusals_and_accounting(sctx, libs):
    w, h = 64, 64
    sctx.set_option("mitsuba_compare", 1)
    s, m, c, em = F.furnace_scene(w, h, 3, False)
    sctx.set_scene(s, m, c, em)
    sctx.read_ray_count()
    for bad in (-1, w * h, 2 ** 31 - 1):
        px = torch.arange(300, dtype=torch.int32, device="cuda")
        px[137] = bad
        px[250] = -5
        s4, q4 = zeros4(300), zeros4(300)
        with pytest.raises(libs.TptError, match=rf"pixels\[137\] = {bad} is outside the 64 x 64 image"):
            sctx.draw_samples(0, w, h, px, 2, s4, q4)
        assert not s4.any() and not q4.any()
        assert sctx.read_ray_count() == 0
    hpx = np.array([0, 5, w * h], np.int32)                  # host list
    with pytest.raises(libs.TptError, match=r"pixels\[2\]"):
        sctx.draw_samples(0, w, h, hpx, 2)
    # misaligned device buffers
    px = torch.arange(100, dtype=torch.int32, device="cuda")
    buf = torch.zeros(4 * 100 + 4, dtype=torch.float32, device="cuda")
    with pytest.raises(libs.TptError, match="sum4 is not 16-byte aligned"):
        sctx.draw_samples(0, w, h, px, 1, libs.DevicePtr(buf.data_ptr() + 4), n=100)
    with pytest.raises(libs.TptError, match="sq4 is not 16-byte aligned"):
        sctx.draw_samples(0, w, h, px, 1, zeros4(100), libs.DevicePtr(buf.data_ptr() + 8))
    with pytest.raises(libs.TptError, match="pixels is not 4-byte aligned"):
        sctx.draw_samples(0, w, h, libs.DevicePtr(px.data_ptr() + 2), 1, zeros4(100), n=100)
    host = np.zeros((100, 4), np.float32)
    with pytest.raises(libs.TptError, match="sum4 is not CUDA memory"):
        sctx.draw_samples(0, w, h, px, 1, libs.DevicePtr(host.ctypes.data), n=100)
    if torch.cuda.device_count() > 1:
        with pytest.raises(libs.TptError, match="lives on device 1"):
            sctx.draw_samples(0, w, h, px, 1, torch.zeros((100, 4), device="cuda:1"))
    # 32-bit sample streams
    with pytest.raises(libs.TptError, match="2\\^32"):
        sctx.draw_samples(0, 65536, 32768, px, 3, zeros4(100))
    with pytest.raises(libs.TptError, match="spp < 1"):
        sctx.draw_samples(0, w, h, px, 0, zeros4(100))
    # n == 0 launches nothing; a list call counts 3 launches (index check, trace, ray accumulation), an all-pixel call 2
    (e, _), r = sctx.draw_samples(0, w, h, torch.zeros(0, dtype=torch.int32, device="cuda"), 2)
    assert r == 0 and e.shape == (0, 4) and sctx.last_launch_count() == 0
    # without a list n must be width * height, n == 0 included; sum4 must not be NULL even then
    L, s0 = sctx._L, zeros4(1)
    assert L.tpt_draw_samples(sctx._h, 0, w, h, None, 0, 2, s0.data_ptr(), None, 1, None, None) != 0
    assert "n must be width * height" in L.tpt_last_error(sctx._h).decode()
    assert L.tpt_draw_samples(sctx._h, 0, w, h, px.data_ptr(), 0, 2, None, None, 1, None, None) != 0
    assert "null sum4" in L.tpt_last_error(sctx._h).decode()
    sctx.draw_samples(0, w, h, px, 2)
    assert sctx.last_launch_count() == 3 and sctx.last_kernel_ms() > 0
    sctx.draw_samples(0, w, h, None, 2)
    assert sctx.last_launch_count() == 2
    # ordering and the running ray count, mixed with draws
    sctx.read_ray_count()
    img = torch.zeros((h, w, 4), device="cuda")
    d = sctx.draw(0, 1, w, h, img, mode=libs.MODE_FAST)
    (_, _), r = sctx.draw_samples(0, w, h, px, 2)
    assert sctx.read_ray_count() == d + r == w * h * 4 * 5 + 100 * 2 * 5
