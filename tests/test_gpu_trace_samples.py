"""tpt_trace_samples (Context.trace_samples) and Context.trace_adaptive, checked where the answer is exact or known: furnace
scene A entry by entry in every k_fast_rays instance (sums, squares and ray counts exact), the mean calls' own samples
(trace_rays, trace_irradiance), lists against all-input calls (continuation, ids per input), the variance across
independent frames and the closed forms B1 / B2 for the moments, adaptive sampling of a panorama and a lightmap against
uniform sampling at equal rays — and the C-ABI around it (accumulation, untraceable inputs, refusals, buffer kinds,
ordering with torch's streams)."""
import ctypes

import numpy as np
import pytest
import torch
from scipy import stats

import furnace as F
from conftest import rel_l2
from test_gpu_irradiance import RAYS_INSTANCES, furnace_a, lambert_hits, sphere_points
from test_gpu_mirror_chains import LONG_SLABS_PER_WARP, SLAB_PIX, queue_instance
from test_gpu_rays import furnace_rays
from test_gpu_samples import SPIN, pixel_err
import test_sweep_oracle as so
from toypathtracer_b200.scenes import camera_rays

pytestmark = pytest.mark.gpu

SEEN = set()          # k_fast_rays instances the furnace tests ran (the union must be all 22)


@pytest.fixture
def tctx(gpu_ctx):
    yield gpu_ctx
    for k, v in (("fast_kform", 2), ("mitsuba_compare", 0), ("light_sampling", 1)):
        gpu_ctx.set_option(k, v)
    gpu_ctx.set_spp(4)


def zeros4(n):
    return torch.zeros((n, 4), dtype=torch.float32, device="cuda")


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


# ---- 1. furnace A entry by entry, every instance -----------------------------------------------------------------------
def entry_lists(n, seed):
    rng = np.random.default_rng(seed)
    return {"all": None,
            "one": np.array([n // 2 + 3], np.int32),
            "tail": rng.permutation(n)[:200].astype(np.int32),                  # unsorted, 200 = 3 x 64 + 8
            "dups": np.repeat(rng.integers(0, n, 70).astype(np.int32), 3)}     # 210 entries, each input 3 x


def check_entries(ctx, s, m, K, ls, inputs, points, entries, spp, frame, kopt, long=False, label=""):
    """Every sample of every entry is the furnace value v (rays: albedo x sky, points: pi x sky): sum = count v, sq =
    count v^2, count = spp, and (2 + K) rays per ray sample or (1 + K) per point sample (light sampling off: 2 or 1); the
    launch ran the instance the pick rules choose."""
    ids = torch.zeros(len(inputs), dtype=torch.int32, device="cuda") if points else None
    lst = None if entries is None else cuda(entries)
    n = len(inputs) if entries is None else len(entries)
    (sm, sq), traced = ctx.trace_samples(cuda(inputs), ids, points, lst, spp, frame)
    got = ctx.last_kernels()
    SEEN.update(got)
    want = queue_instance("rays", len(s), K, kopt, so.gate_passes(s) and kopt != 0, ls, long=long)
    assert got == [want], (label, got, want)
    sm, sq = sm.cpu().numpy().astype(np.float64), sq.cpu().numpy().astype(np.float64)
    v = np.pi * F.MITSUBA_SKY.astype(np.float64) if points else F.furnace_value(m).astype(np.float64)
    assert sm.shape == (n, 4) and (sm[:, 3] == spp).all() and (sq[:, 3] == 0).all(), label
    tol = v * spp * (spp + 2) * 2.0 ** -23
    assert (np.abs(sm[:, :3] - spp * v) <= tol).all(), (label, sm[:4], spp * v)
    assert (np.abs(sq[:, :3] - spp * v * v) <= 4 * v * tol).all(), (label, sq[:4], spp * v * v)
    var = (sq[:, :3] - sm[:, :3] ** 2 / spp) / max(spp - 1, 1)
    assert (np.abs(var) <= 1e-6 * spp * v * v).all(), label
    per = ((1 + K) if ls else 1) if points else F.furnace_rays_per_sample(m, K, ls)
    assert traced == n * spp * per, (label, traced, n * spp * per)


def test_furnace_entries_every_instance(tctx):
    """Rays at the receiver and points on it, with the all-input call and one-entry, unsorted, duplicate and
    non-multiple-of-64 lists; 0-300 lights, a Metal receiver, light sampling on and off, fast_kform 0-3, the 768-thread
    instance (1 500 padding spheres) and launches of >= 48 slabs per warp (the 8-CTA instances)."""
    tctx.set_option("mitsuba_compare", 1)
    cases = [(3, False, False), (64, False, False), (3, True, False), (3, False, True), (3, True, True)]
    for K, padded, with_speck in cases:
        s, m, c, em = furnace_a(K, padded, with_speck)
        for kopt in (0, 1, 2, 3):
            tctx.set_option("fast_kform", kopt)
            for ls in (1, 0):
                tctx.set_option("light_sampling", ls)
                tctx.set_scene(s, m, c, em)
                points = (kopt + ls) % 2 == 1
                inputs = sphere_points((0, 0, 0), F.RECEIVER_R, 1001, K + kopt) if points else furnace_rays(1001, K + kopt)
                for name, lst in entry_lists(len(inputs), 10 * K + kopt).items():
                    check_entries(tctx, s, m, K, ls, inputs, points, lst, 3, kopt, kopt,
                                  label=f"K{K} padded{padded} speck{with_speck} kform{kopt} ls{ls} {name}")
    for K, metal in ((0, True), (300, False)):
        s, m, c, em = F.furnace_scene(64, 64, K, metal)
        tctx.set_option("fast_kform", 2)
        tctx.set_option("light_sampling", 1)
        tctx.set_scene(s, m, c, em)
        for points in (False, True):
            inputs = sphere_points((0, 0, 0), F.RECEIVER_R, 777, K) if points else furnace_rays(777, K)
            check_entries(tctx, s, m, K, 1, inputs, points, entry_lists(777, K)["tail"], 2, 1, 2, label=f"K{K} metal{metal}")
    # the 8-CTA instances: forms 4 (5 spheres) and 2 (65 spheres), >= 48 slabs of 64 entries per warp on every SM
    n = 65536
    spp = -(-LONG_SLABS_PER_WARP * torch.cuda.get_device_properties(0).multi_processor_count * 32 // (n // SLAB_PIX))
    lst = np.random.default_rng(8).permutation(n).astype(np.int32)
    for K in (3, 64):
        s, m, c, em = furnace_a(K)
        for ls in (1, 0):
            tctx.set_option("light_sampling", ls)
            tctx.set_scene(s, m, c, em)
            inputs = sphere_points((0, 0, 0), F.RECEIVER_R, n, K) if ls else furnace_rays(n, K)
            check_entries(tctx, s, m, K, ls, inputs, bool(ls), lst, spp, 9, 2, long=True, label=f"long K{K} ls{ls}")
    assert SEEN == RAYS_INSTANCES, (sorted(RAYS_INSTANCES - SEEN), sorted(SEEN - RAYS_INSTANCES))


# ---- 2. the mean calls' own samples ------------------------------------------------------------------------------------
def scene_inputs(ctx, libs, scene, w, h):
    if scene == "reference":
        sph, mats, cam, em = libs.reference_scene(w, h)
    else:
        sph, mats, cam = libs.stress_scene(w, h, count=4096)[:3]
        em = None
    ctx.set_scene(sph, mats, cam, em)
    rays = camera_rays(cam, w, h, per_pixel=1, seed=17)
    _, pts, ids = lambert_hits(ctx, sph, mats, rays)
    return sph, mats, cam, rays, pts, ids.astype(np.int32)


@pytest.mark.parametrize("scene", ["reference", "stress"])
@pytest.mark.parametrize("ls", [1, 0])
def test_same_samples_as_the_mean_calls(tctx, libs, scene, ls):
    """An all-input call's sum.rgb / spp is trace_rays' / trace_irradiance's value at the same spp and frame (to the
    rounding of the reduction order) with the same ray count: rays, and points with and without ids."""
    tctx.set_option("light_sampling", ls)
    _, _, _, rays, pts, ids = scene_inputs(tctx, libs, scene, 320, 180)
    for kind, inp, pid in (("rays", rays, None), ("points", pts, None), ("points+ids", pts, ids)):
        points = kind != "rays"
        inp_d = cuda(inp)
        ids_d = None if pid is None else cuda(pid)
        for spp, frame in ((1, 0), (4, 7)):
            if points:
                mean, r0 = tctx.trace_irradiance(inp_d, ids_d, spp=spp, frame=frame)
            else:
                mean, r0 = tctx.trace_rays(inp_d, spp=spp, frame=frame)
            (sm, sq), r1 = tctx.trace_samples(inp_d, ids_d, points, None, spp, frame)
            assert r1 == r0, (kind, spp, r0, r1)
            mean, sm, sq = (t.cpu().numpy().astype(np.float64) for t in (mean, sm, sq))
            assert (sm[:, 3] == spp).all() and (sq[:, 3] == 0).all()
            err = np.abs(sm[:, :3] / spp - mean[:, :3])
            assert (err <= 4e-7 * spp * np.abs(mean[:, :3]) + 1e-30).all(), (kind, spp, err.max())
            assert (sq[:, :3] >= sm[:, :3] ** 2 / spp * (1 - 1e-5)).all()
            assert (sq[:, :3] <= sm[:, :3] ** 2 * (1 + 1e-5) + 1e-30).all()


# ---- 3. a list continues the all-input call ----------------------------------------------------------------------------
def test_list_continues_the_all_input_call(tctx, libs):
    """A shuffled list over points with ids, light spheres' points among them with their own ids: each listed input's sums
    are its all-input sums, a duplicate gets them once per occurrence. The list over every input once traces exactly the
    all-input call's rays, and twice exactly twice: an id read at the list position would make a point on an emissive
    sphere sample itself, one more shadow ray per sample. (Every list here is at most as long as the inputs.)"""
    _, mats, _, rays, pts, ids = scene_inputs(tctx, libs, "reference", 320, 180)
    assert (mats["emissive"][ids].max(1) > 0).any()
    n = len(pts)
    rng = np.random.default_rng(4)
    pts_d, ids_d = cuda(pts), cuda(ids)
    perm = rng.permutation(n).astype(np.int32)
    lst = np.concatenate([perm[: n // 3], rng.integers(0, n, 999)]).astype(np.int32)
    for frame in (2, 13):
        (sa, qa), ra = tctx.trace_samples(pts_d, ids_d, True, None, 4, frame)
        (sl, ql), _ = tctx.trace_samples(pts_d, ids_d, True, cuda(lst), 4, frame)
        sa, qa = sa.cpu().numpy()[lst].astype(np.float64), qa.cpu().numpy()[lst].astype(np.float64)
        sl, ql = sl.cpu().numpy().astype(np.float64), ql.cpu().numpy().astype(np.float64)
        assert (sl[:, 3] == 4).all()
        assert (np.abs(sl - sa) <= 1e-6 * sa + 1e-30).all(), np.abs(sl - sa).max()
        assert (np.abs(ql - qa) <= 1e-6 * qa + 1e-30).all(), np.abs(ql - qa).max()
        _, rp = tctx.trace_samples(pts_d, ids_d, True, cuda(perm), 4, frame)
        _, rh = tctx.trace_samples(pts_d, ids_d, True, cuda(perm[: n // 2]), 4, frame)
        _, rhh = tctx.trace_samples(pts_d, ids_d, True, cuda(np.concatenate([perm[: n // 2], perm[n // 2 - 1::-1]])), 4, frame)
        assert rp == ra and rhh == 2 * rh, (ra, rp, rh, rhh)
    # rays: the same continuation
    rays_d = cuda(rays)
    (sa, _), _ = tctx.trace_samples(rays_d, None, False, None, 2, 5)
    (sl, _), _ = tctx.trace_samples(rays_d, None, False, cuda(lst), 2, 5)
    sa, sl = sa.cpu().numpy()[lst].astype(np.float64), sl.cpu().numpy().astype(np.float64)
    assert (np.abs(sl - sa) <= 1e-6 * sa + 1e-30).all()


# ---- 4. moments ----------------------------------------------------------------------------------------------------------
def test_moments_match_the_spread_of_frames(tctx):
    """Scene B2 (bounded samples): per-entry variance from the moments of one 64-sample call against the spread of 32
    independent single samples (frames), for the camera rays and for the receiver points: each ratio inside the F(63, 31)
    band, the pooled ratio near 1. (The gradient sky's blue is 1 everywhere: that channel has no variance.)"""
    s, m, c, em, w, h, E, bins, mitsuba, ls = F.b_case("b2")
    tctx.set_option("mitsuba_compare", 1 if mitsuba else 0)
    tctx.set_option("light_sampling", 1 if ls else 0)
    tctx.set_scene(s, m, c, em)
    p, _, _ = F.footprint_hits(c, w, h)
    pts = np.concatenate([p, p / F.RECEIVER_R], -1).reshape(-1, 6).astype(np.float32)
    rays = camera_rays(c, w, h, per_pixel=1, seed=3)
    for points, inp in ((False, rays), (True, pts)):
        sel = np.random.default_rng(9).permutation(len(inp))[:300].astype(np.int32)
        inp_d, lst = cuda(inp), cuda(sel)
        ids = torch.zeros(len(inp), dtype=torch.int32, device="cuda") if points else None
        (sa, qa), _ = tctx.trace_samples(inp_d, ids, points, lst, 64, 100)
        sa, qa = sa.cpu().numpy().astype(np.float64), qa.cpu().numpy().astype(np.float64)
        var_a = ((qa[:, :3] - sa[:, :3] ** 2 / 64) / 63)[:, :2]
        singles = np.stack([tctx.trace_samples(inp_d, ids, points, lst, 1, 200 + k)[0][0].cpu().numpy()[:, :2]
                            for k in range(32)]).astype(np.float64)
        var_b = singles.var(axis=0, ddof=1)
        assert (var_a > 0).all() and (var_b > 0).all(), points
        ratio = var_a / var_b                                   # ~ F(63, 31) per entry and channel
        lo, hi = stats.f.ppf([1e-6, 1 - 1e-6], 63, 31)
        assert ((ratio > lo) & (ratio < hi)).all(), (points, ratio.min(), ratio.max(), lo, hi)
        assert abs(np.log(var_a.sum() / var_b.sum())) < 0.15, (points, var_a.sum() / var_b.sum())


@pytest.mark.parametrize("scene", ["b1_ls", "b1_nols", "b2"])
def test_closed_forms_binned(tctx, scene):
    """The receiver points of furnace.footprint_hits (points, ids 0) and the pixel rays through them: per bin the means
    sum / count over 16 frames of 16 samples meet furnace.check_bins against E / pi (points) and the B expectation (rays)."""
    s, m, c, em, w, h, e, bins, mitsuba, ls = F.b_case(scene)
    tctx.set_option("mitsuba_compare", 1 if mitsuba else 0)
    tctx.set_option("light_sampling", 1 if ls else 0)
    tctx.set_scene(s, m, c, em)
    p, wq, _ = F.footprint_hits(c, w, h)
    pts = cuda(np.concatenate([p, p / F.RECEIVER_R], -1).reshape(-1, 6).astype(np.float32))
    ids = torch.zeros(len(pts), dtype=torch.int32, device="cuda")
    wt = torch.from_numpy(wq).cuda()
    batches = []
    for b in range(16):
        (sm, sq), _ = tctx.trace_samples(pts, ids, True, None, 16, b)
        assert (sm[:, 3] == 16).all() and (sq[:, :3] >= 0).all()
        mean = sm[:, :3].double() / sm[:, 3:].double()
        px = (mean.view(h, w, len(wq), 3) * wt[None, None, :, None]).sum(2) / np.pi
        batches.append(px.cpu().numpy())
    F.check_bins(np.array(batches), e / m["albedo"][0].astype(np.float64), bins)


# ---- 5. accumulation, untraceable inputs, refusals ------------------------------------------------------------------------
def test_calls_accumulate_and_untraceable_inputs_add_nothing(tctx):
    K = 3
    s, m, c, em = furnace_a(K)
    tctx.set_option("mitsuba_compare", 1)
    tctx.set_scene(s, m, c, em)
    pts = sphere_points((0, 0, 0), F.RECEIVER_R, 1000, 4)
    for i in range(0, 1000, 3):            # every third point broken, in runs that straddle the 64-entry slabs
        k = (i // 3) % 4
        if k == 3:
            pts[i, 3:] = 0.0
        else:
            pts[i, 2 * k + 1] = (np.nan, np.inf, -np.inf)[k]
    valid = np.isfinite(pts).all(1) & (np.abs(pts[:, 3:]).max(1) > 0)
    v = np.pi * F.MITSUBA_SKY.astype(np.float64)
    rng = np.random.default_rng(1)
    sum0 = rng.normal(size=(1000, 4)).astype(np.float32)
    sum0[:, 3] = rng.integers(0, 100, 1000)                  # counts: whole numbers, so count + 5 is exact
    sq0 = rng.normal(size=(1000, 4)).astype(np.float32)
    lst = np.arange(1000, dtype=np.int32)[::-1].copy()
    for entries in (None, lst):
        sm, sq = sum0.copy(), sq0.copy()
        _, r1 = tctx.trace_samples(pts, None, True, entries, 3, 0, sm, sq)
        _, r2 = tctx.trace_samples(pts, None, True, entries, 2, 1, sm, sq)     # adds: no zeroing between calls
        assert r1 == int(valid.sum()) * 3 * (1 + K) and r2 == int(valid.sum()) * 2 * (1 + K)
        inp = np.arange(1000) if entries is None else entries
        ok = valid[inp]
        assert (sm[~ok].view(np.uint32) == sum0[~ok].view(np.uint32)).all()
        assert (sq[~ok].view(np.uint32) == sq0[~ok].view(np.uint32)).all()
        assert np.allclose(sm[ok, :3], sum0[ok, :3] + 5 * v, rtol=1e-5, atol=1e-5)
        assert (sm[ok, 3] == sum0[ok, 3] + 5).all()
        assert np.allclose(sq[ok, :3], sq0[ok, :3] + 5 * v * v, rtol=1e-5, atol=1e-5) and (sq[ok, 3] == sq0[ok, 3]).all()


def test_bad_index_fails_and_traces_nothing(tctx, libs):
    s, m, c, em = furnace_a(3)
    tctx.set_option("mitsuba_compare", 1)
    tctx.set_scene(s, m, c, em)
    rays = cuda(furnace_rays(500, 2))
    sm = zeros4(300); sm[:, 0] = 2.0
    sq = zeros4(300)
    for bad in (500, -1, 1 << 30):
        lst = torch.arange(300, dtype=torch.int32, device="cuda")
        lst[257] = bad
        lst[280] = 499
        tctx.read_ray_count()
        with pytest.raises(libs.TptError, match=rf"entries\[257\] = {bad} is outside the 500 inputs"):
            tctx.trace_samples(rays, None, False, lst, 2, 0, sm, sq)
        assert tctx.read_ray_count() == 0
        assert (sm[:, 0] == 2.0).all() and (sm[:, 1:] == 0).all() and (sq == 0).all()
    # n == 0 launches nothing and reads no buffer
    (e4, _), r = tctx.trace_samples(rays, None, False, torch.zeros(0, dtype=torch.int32, device="cuda"))
    assert r == 0 and e4.shape == (0, 4) and tctx.last_launch_count() == 0 and tctx.last_kernels() == []


def test_refusals(tctx, libs):
    s, m, c, em = furnace_a(3)
    tctx.set_scene(s, m, c, em)
    L, hdl = tctx._L, tctx._h
    dev = torch.zeros((70, 6), dtype=torch.float32, device="cuda")
    ids = torch.zeros(70, dtype=torch.int32, device="cuda")
    ent = torch.zeros(70, dtype=torch.int32, device="cuda")
    s4, q4 = zeros4(70), zeros4(70)
    p, i, e, so_, q = (ctypes.c_void_p(t.data_ptr()) for t in (dev, ids, ent, s4, q4))
    cnt = ctypes.c_longlong(-1)

    def refused(text, in6, idp, points, num_in, en, n, spp, sm, sq):
        assert L.tpt_trace_samples(hdl, in6, idp, points, num_in, en, n, spp, 0, sm, sq, 1, ctypes.byref(cnt), None) != 0
        assert text in L.tpt_last_error(hdl).decode(), (text, L.tpt_last_error(hdl).decode())

    refused("tpt_trace_samples: null in6 or sum4", None, None, 0, 70, e, 70, 1, so_, q)
    refused("null in6 or sum4", p, None, 0, 70, e, 70, 1, None, q)
    refused("n < 0", p, None, 0, 70, e, -1, 1, so_, q)
    refused("n < 0", p, None, 0, -1, e, 70, 1, so_, q)
    refused("spp < 1", p, None, 0, 70, e, 70, 0, so_, q)
    refused("numIn * spp > 2^32", p, None, 0, (1 << 31) + 1, e, 70, 2, so_, q)
    refused("ids are only taken with points", p, i, 0, 70, e, 70, 1, so_, q)
    refused("points must be 0 or 1", p, None, 2, 70, e, 70, 1, so_, q)
    refused("without entries n must be numIn", p, None, 0, 70, None, 69, 1, so_, q)
    refused("2^31 slabs", p, None, 0, 1, e, 70, 1 << 30, so_, q)
    refused("sum4 is not 16-byte aligned", p, None, 0, 70, e, 60, 1, ctypes.c_void_p(s4.data_ptr() + 4), q)
    refused("sq4 is not 16-byte aligned", p, None, 0, 70, e, 60, 1, so_, ctypes.c_void_p(q4.data_ptr() + 8))
    refused("entries is not 4-byte aligned", p, None, 0, 70, ctypes.c_void_p(ent.data_ptr() + 2), 60, 1, so_, q)
    refused("in6 is not 4-byte aligned", ctypes.c_void_p(dev.data_ptr() + 2), None, 0, 60, e, 60, 1, so_, q)
    host = np.zeros(70, np.int32)
    refused("entries is not CUDA memory", p, None, 0, 70, ctypes.c_void_p(host.ctypes.data), 70, 1, so_, q)
    # n == 0: nothing launched, no rays, no buffer read
    cnt.value = -1
    assert L.tpt_trace_samples(hdl, ctypes.c_void_p(host.ctypes.data), None, 0, 0, ctypes.c_void_p(host.ctypes.data), 0, 4,
                               0, ctypes.c_void_p(host.ctypes.data), None, 0, ctypes.byref(cnt), None) == 0
    assert cnt.value == 0 and tctx.last_launch_count() == 0


# ---- 6. buffer kinds and torch streams ---------------------------------------------------------------------------------
def test_buffer_kinds_accumulate_the_same_bits(tctx, libs):
    """Host numpy, page-locked torch, torch CPU, torch CUDA on a side stream and DevicePtr buffers, each starting from the
    same non-zero sums: the same bits (spp 1: one reduction per entry) and ray counts."""
    _, _, _, rays, pts, ids = scene_inputs(tctx, libs, "reference", 160, 90)
    lst = np.random.default_rng(3).integers(0, len(pts), 3000).astype(np.int32)
    n = len(lst)
    start = np.random.default_rng(2).random((n, 4)).astype(np.float32)
    ref_s, ref_q = start.copy(), start.copy()
    _, traced = tctx.trace_samples(pts, ids, True, lst, 1, 3, ref_s, ref_q)

    def same(sm, sq, r):
        assert r == traced
        assert (np.asarray(sm).view(np.uint32) == ref_s.view(np.uint32)).all()
        assert (np.asarray(sq).view(np.uint32) == ref_q.view(np.uint32)).all()

    pin = [torch.empty(a.shape, dtype=t, pin_memory=True) for a, t in
           ((pts, torch.float32), (ids, torch.int32), (lst, torch.int32), (start, torch.float32), (start, torch.float32))]
    for t, a in zip(pin, (pts, ids, lst, start, start)):
        t.numpy()[...] = a
    _, r = tctx.trace_samples(pin[0], pin[1], True, pin[2], 1, 3, pin[3], pin[4])
    same(pin[3].numpy(), pin[4].numpy(), r)
    cpu = [torch.from_numpy(a.copy()) for a in (pts, ids, lst, start, start)]
    _, r = tctx.trace_samples(cpu[0], cpu[1], True, cpu[2], 1, 3, cpu[3], cpu[4])
    same(cpu[3].numpy(), cpu[4].numpy(), r)
    side = torch.cuda.Stream()
    dv = [cuda(a.copy()) for a in (pts, ids, lst, start, start)]
    torch.cuda.synchronize()
    tctx.trace_samples(dv[0], dv[1], True, dv[2], 1, 3, dv[3], dv[4], stream=side.cuda_stream, want_rays=False)
    side.synchronize()
    same(dv[3].cpu().numpy(), dv[4].cpu().numpy(), traced)
    dv = [cuda(a.copy()) for a in (pts, ids, lst, start, start)]
    ptr = [libs.DevicePtr(t.data_ptr()) for t in dv]
    _, r = tctx.trace_samples(ptr[0], ptr[1], True, ptr[2], 1, 3, ptr[3], ptr[4], n=n, num_in=len(pts))
    same(dv[3].cpu().numpy(), dv[4].cpu().numpy(), r)


def test_calls_are_ordered_with_torch_streams(tctx):
    """Outputs allocated by trace_samples, a caller's zeroed buffer and a list written by torch kernels, each behind a
    spinning kernel on torch's current stream (default and side), and trace_adaptive's rounds: every sum is the furnace
    value, so no call overtook the torch work it depends on."""
    s, m, c, em = furnace_a(3)
    tctx.set_option("mitsuba_compare", 1)
    tctx.set_scene(s, m, c, em)
    v = np.pi * F.MITSUBA_SKY.astype(np.float64)
    pts = cuda(sphere_points((0, 0, 0), F.RECEIVER_R, 4096, 6))
    n = len(pts)

    def check(sums, k, spp):
        sums = sums.cpu().numpy().astype(np.float64)
        assert sums.shape == (k, 4) and (sums[:, 3] == spp).all(), sums[:3]
        assert np.allclose(sums[:, :3], spp * v, rtol=1e-6, atol=0), sums[:3]

    side = torch.cuda.Stream()
    for current in (torch.cuda.default_stream(), side):
        with torch.cuda.stream(current):
            torch.cuda.synchronize()
            torch.cuda._sleep(SPIN)
            (s4, _), _ = tctx.trace_samples(pts, None, True, None, 2)
            check(s4, n, 2)
            torch.cuda._sleep(SPIN)
            own = torch.empty((n, 4), device="cuda").zero_()
            tctx.trace_samples(pts, None, True, None, 2, 1, own, want_rays=False)
            check(own, n, 2)
            torch.cuda._sleep(SPIN)
            idx = (torch.arange(300, device="cuda") * 13 % n).to(torch.int32)
            (sl, _), _ = tctx.trace_samples(pts, None, True, idx, 3, 2)
            check(sl, 300, 3)
            torch.cuda._sleep(SPIN)
            mean, spp, rays = tctx.trace_adaptive(pts, points=True, base_spp=2, max_spp=8, rel_err=0.05, frame=3,
                                                   shape=(64, 64))
            assert (spp == 2).all() and rays == n * 2 * 4
            assert np.allclose(mean.cpu().numpy()[:, :3], v, rtol=1e-6, atol=0) and (mean[:, 3] == 0).all()
    torch.cuda.synchronize()
    torch.cuda._sleep(SPIN)
    (s4, _), _ = tctx.trace_samples(pts, None, True, None, 2, stream=side.cuda_stream)
    side.synchronize()
    check(s4, n, 2)
    torch.cuda.synchronize()


# ---- 7. adaptive against uniform at equal rays ---------------------------------------------------------------------------
def panorama(cam, w, h):
    """Equirect rays from the camera's origin, row-major (h, w), one per texel centre."""
    u = (np.arange(w) + 0.5) / w * 2 * np.pi
    t = (np.arange(h) + 0.5) / h * np.pi
    th, ph = np.meshgrid(t, u, indexing="ij")
    d = np.stack([np.sin(th) * np.cos(ph), np.cos(th), np.sin(th) * np.sin(ph)], -1).reshape(-1, 3)
    o = np.broadcast_to(np.asarray(cam["origin"], np.float64).reshape(1, 3), d.shape)
    return np.concatenate([o, d], 1).astype(np.float32)


def lightmap(sph, w, h, half=6.0):
    """Points on sphere 0 (the ground) over an x-z square around the origin, row-major (h, w)."""
    c = np.asarray(sph["center"][0], np.float64)
    r = float(sph["radius"][0])
    x = (np.arange(w) + 0.5) / w * 2 * half - half
    z = (np.arange(h) + 0.5) / h * 2 * half - half - 1.0
    zz, xx = np.meshgrid(z, x, indexing="ij")
    y = c[1] + np.sqrt(r * r - (xx - c[0]) ** 2 - (zz - c[2]) ** 2)
    p = np.stack([xx, y, zz], -1).reshape(-1, 3)
    return np.concatenate([p, (p - c) / r], 1).astype(np.float32)


# Measured on the H100 (DESIGN §3.8): adaptive wins on relL2 at every rel_err listed here. On the 90th-percentile entry
# error it wins on the lightmap at each of them, but not on the panorama: there the two tie at 0.02 and uniform wins
# at 0.05 and 0.1 (0.031 against 0.027, 0.034 against 0.031), so the tail is only asserted where ADAPTIVE_TAIL_WINS says.
ADAPTIVE_REL_ERR = (0.02, 0.05, 0.1)
ADAPTIVE_TAIL_WINS = {("lightmap", 0.02), ("lightmap", 0.05), ("lightmap", 0.1)}
STOP_ALLOWANCE = 1.0          # region-mean bias bar: max(5 se, 1e-4 E) + STOP_ALLOWANCE * rel_err * (E + 0.05)


@pytest.mark.parametrize("workload", ["panorama", "lightmap"])
def test_adaptive_beats_uniform_at_equal_rays(tctx, libs, workload):
    w, h = 256, 128
    sph, mats, cam, em = libs.reference_scene(640, 360)
    tctx.set_scene(sph, mats, cam, em)
    points = workload == "lightmap"
    inp = cuda(lightmap(sph, w, h) if points else panorama(cam, w, h))
    ids = torch.zeros(w * h, dtype=torch.int32, device="cuda") if points else None
    n = w * h
    # reference: 16 frames x 256 spp of the same API
    ref = torch.zeros((n, 4), dtype=torch.float64, device="cuda")
    for f in range(16):
        (s, _), _ = tctx.trace_samples(inp, ids, points, None, 256, 5000 + f)
        ref += s.double()
    ref = (ref[:, :3] / ref[:, 3:]).cpu().numpy()
    (_, _), r4 = tctx.trace_samples(inp, ids, points, None, 4, 100)
    rows = []
    for rel in ADAPTIVE_REL_ERR:
        mean, spp, rays = tctx.trace_adaptive(inp, ids, points, base_spp=4, max_spp=64, rel_err=rel, frame=0, shape=(h, w))
        mean, spp = mean.cpu().numpy().astype(np.float64), spp.cpu().numpy()
        assert (mean[:, 3] == 0).all() and spp.min() >= 4 and spp.max() <= 64 and (spp % 4 == 0).all()
        u = 4
        while r4 * u / 4 < rays:
            u += 1
        (su, qu), ru = tctx.trace_samples(inp, ids, points, None, u, 200)
        assert ru >= rays * 0.99, (ru, rays, u)
        su, qu = su.cpu().numpy().astype(np.float64), qu.cpu().numpy().astype(np.float64)
        var1 = np.maximum(qu[:, :3] - su[:, :3] ** 2 / u, 0) / (u - 1)          # per-sample variance per entry
        uni = su[:, :3] / su[:, 3:]
        a_l2, u_l2 = rel_l2(mean[:, :3], ref), rel_l2(uni, ref)
        a90, u90 = np.percentile(pixel_err(mean[:, :3], ref), 90), np.percentile(pixel_err(uni, ref), 90)
        rows.append(dict(workload=workload, rel_err=rel, rays=rays, mean_spp=float(spp.mean()), uniform_spp=u,
                         relL2=(a_l2, u_l2), p90=(a90, u90)))
        print(rows[-1])
        assert a_l2 < u_l2, rows[-1]
        if (workload, rel) in ADAPTIVE_TAIL_WINS:
            assert a90 < u90, rows[-1]
        # stopping bias: the mean over all entries and over the brightest and darkest quartiles
        lum = ref @ np.array([0.2126, 0.7152, 0.0722])
        for msk in (np.ones(n, bool), lum >= np.percentile(lum, 75), lum <= np.percentile(lum, 25)):
            e = ref[msk].mean(0)
            se = np.sqrt((var1[msk] / spp[msk, None]).sum(0)) / msk.sum()
            bar = np.maximum(5 * se, 1e-4 * e) + STOP_ALLOWANCE * rel * (e + 0.05)
            assert (np.abs(mean[msk, :3].mean(0) - e) <= bar).all(), (workload, rel, mean[msk, :3].mean(0), e, bar)
