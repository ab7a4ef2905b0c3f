"""tpt_draw_aovs / tpt_trace_aovs (Context.draw_aovs, Context.trace_aovs): first-hit albedo, coverage, normal, depth and
sphere id, checked where the answer is exact or known — caller rays against the float64 nearest-hit oracle of
test_sweep_oracle.py, draw pixels against the primary hits the fast draw itself decodes in an emission-only scene, pixel
footprints of the furnace scene A and the lens coverage of scene B5 in closed form (tests/furnace.py) — and the C-ABI
behaviour around them (blend, row regions, buffers, refusals, accounting, ordering)."""
import ctypes
import itertools

import numpy as np
import pytest
import torch

import furnace as F
import test_sweep_oracle as so
from conftest import bits_differ, rel_l2
from test_gpu_fast import surface_rays
from test_gpu_rays import DIR_ERR, HIT_CASES, _scaled, decode, emission_scene, max_queue_count, oracle

pytestmark = pytest.mark.gpu
PROG = 2          # kFlagProgressive


@pytest.fixture
def actx(gpu_ctx):
    yield gpu_ctx
    for k, v in (("fast_kform", 2), ("mitsuba_compare", 0), ("light_sampling", 1), ("fast_variant", -1)):
        gpu_ctx.set_option(k, v)
    gpu_ctx.set_spp(4)


def trace(ctx, rays):
    (a, nrm, ids), traced = ctx.trace_aovs(torch.from_numpy(np.ascontiguousarray(rays)).cuda())
    return a.cpu().numpy(), nrm.cpu().numpy(), ids.cpu().numpy(), traced


def dev_buffers(h, w):
    return (torch.zeros((h, w, 4), dtype=torch.float32, device="cuda"), torch.zeros((h, w, 4), dtype=torch.float32, device="cuda"),
            torch.zeros((h, w), dtype=torch.int32, device="cuda"))


def np_(*ts):
    return [t.cpu().numpy() for t in ts]


# ---- 1. caller rays against the float64 oracle -----------------------------------------------------------------------
def check_against_oracle(ctx, monkeypatch, sph, mats, rays, label, target=None):
    valid = np.isfinite(rays).all(1) & (np.abs(rays[:, 3:]).max(1) > 0)
    ora = oracle(monkeypatch, rays, sph)
    well = ora["well"] & valid
    c = sph["center"].astype(np.float64)
    inv = sph["invRadius"].astype(np.float64)
    o = rays[:, :3].astype(np.float64)
    d = rays[:, 3:].astype(np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):
        dh = d / np.linalg.norm(d, axis=1, keepdims=True)
    for scaled in (False, True):
        a, nrm, ids, _ = trace(ctx, _scaled(rays, 17) if scaled else rays)
        tag = (label, scaled)
        if target is not None:
            assert (ids == target).all(), tag
        bad = well & (ids != ora["id"])
        assert not bad.any(), (tag, int(bad.sum()), ids[bad][:8], ora["id"][bad][:8])
        hit = well & (ids >= 0)
        k = ids[hit]
        t = nrm[hit, 3].astype(np.float64)
        assert ((t >= ora["tlo"][hit]) & (t <= ora["thi"][hit])).all(), tag
        # normal = (o + d t - c) / r: the depth bound moves it by |d_k| (thi - tlo) / r, the kernel's renormalised
        # direction by DIR_ERR t / r, and float rounding of pos and pos - c by a few ulp of |o| + |d t| + |c|
        tt = ora["t"][hit]
        n64 = (o[hit] + dh[hit] * tt[:, None] - c[k]) * inv[k][:, None]
        span = (ora["thi"][hit] - ora["tlo"][hit])[:, None]
        bound = inv[k][:, None] * (np.abs(dh[hit]) * span + DIR_ERR * tt[:, None] +
                                   2.0 ** -21 * (np.abs(o[hit]) + np.abs(dh[hit]) * tt[:, None] + np.abs(c[k]))) + 2.0 ** -21
        assert (np.abs(nrm[hit, :3] - n64) <= bound).all(), (tag, np.abs(nrm[hit, :3] - n64).max())
        assert (a[hit, :3] == mats["albedo"][k]).all(), tag
        assert (a[hit, 3] == 1.0).all(), tag
        miss = ids == -1
        assert (a[miss] == 0).all() and (nrm[miss] == 0).all(), tag
        assert (ids[~valid] == -1).all(), tag


ORACLE_CASES = HIT_CASES + [("stress", "stress", (2, 0))]


@pytest.mark.parametrize("count,layout,kforms", ORACLE_CASES, ids=[f"{c}-{l}" for c, l, _ in ORACLE_CASES])
def test_rays_against_oracle(actx, monkeypatch, libs, count, layout, kforms):
    if layout == "stress":
        sph, mats, _, _ = libs.stress_scene(64, 64)
    else:
        count = max_queue_count(0) if count == "max" else count
        sph, mats, _, _ = so.make_scene(count, layout)
    actx.set_scene(sph, mats, libs.make_camera((0, 1, 5), (0, 0, 0), (0, 1, 0), 40, 1.0, 0.0, 1.0), np.zeros(0, np.int32))
    seed = 500 + len(sph)
    n = int(np.clip(300_000 / len(sph), 64, 3000))
    surf = surface_rays(sph, 4 * n, seed)
    aimed, target = so.aimed_rays(sph, seed + 5)
    sets = {"surface": surf[np.isfinite(surf).all(1)], "tangent": so.near_tangent_rays(sph, n, seed + 1)[0],
            "degenerate": so.degenerate_rays(sph, seed + 3)}
    for kform in kforms:
        actx.set_option("fast_kform", kform)
        for name, rays in sets.items():
            check_against_oracle(actx, monkeypatch, sph, mats, rays, (len(sph), layout, kform, name))
        a, nrm, ids, _ = trace(actx, aimed)
        assert (ids == target).all(), (len(sph), layout, kform, "aimed")
        assert (a[:, 3] == 1).all() and (a[:, :3] == mats["albedo"][target]).all()


def test_padding_sphere_hits_report_the_zero_material(actx, libs):
    """Form 0 on 45 spheres (padded to 48) may return a padding sphere for rays aimed at the padding point: such a hit
    reports what the draw shades with, the all-zero material and invRadius 0."""
    sph, mats, cam, _ = so.make_scene(45, "compact", seed=6)
    actx.set_scene(sph, mats, cam, None)
    actx.set_option("fast_kform", 0)
    a, nrm, ids, _ = trace(actx, so.pad_aimed_rays(256, 13))
    assert ((ids >= -1) & (ids < 48)).all()
    pad = ids >= 45
    assert (a[pad, :3] == 0).all() and (a[pad, 3] == 1).all() and (nrm[pad, :3] == 0).all() and (nrm[pad, 3] > 0).all()


# ---- 2. the same primary hits as the draw -----------------------------------------------------------------------------
EW, EH = 160, 90


def emission_ctx(ctx, spp):
    sph, mats, cam, _ = emission_scene(46, "compact")
    ctx.set_option("light_sampling", 0)
    ctx.set_option("mitsuba_compare", 1)               # constant sky: green 0.21 on a miss, 8 on every hit
    ctx.set_scene(sph, mats, cam, np.zeros(0, np.int32))
    ctx.set_spp(spp)


@pytest.mark.parametrize("variant", [3, 8, -1])
def test_ids_are_the_draws_primary_hits(actx, libs, variant):
    """spp 1, one frame per call: the id the draw's pixel decodes to (emission = id + 1) is `ids`, over several frames, a
    strided row shard and a packed band."""
    emission_ctx(actx, 1)
    actx.set_option("fast_variant", variant)
    for frame in (0, 1, 7, 300):
        img = torch.zeros((EH, EW, 4), dtype=torch.float32, device="cuda")
        ids = torch.full((EH, EW), -7, dtype=torch.int32, device="cuda")
        actx.draw(frame, 1, EW, EH, img, mode=libs.MODE_FAST)
        actx.draw_aovs(frame, 1, EW, EH, ids=ids)
        got = decode(img.cpu().numpy().reshape(-1, 4)).reshape(EH, EW)
        assert (got >= -1).all() and (got == ids.cpu().numpy()).all(), (variant, frame)
    for rows in ((1, 29, 3, 0), (17, 40, 1, 1)):
        h = rows[1] if rows[3] else EH
        img = torch.zeros((h, EW, 4), dtype=torch.float32, device="cuda")
        ids = torch.full((h, EW), -7, dtype=torch.int32, device="cuda")
        actx.draw(4, 1, EW, EH, img, mode=libs.MODE_FAST, rows=rows)
        actx.draw_aovs(4, 1, EW, EH, ids=ids, rows=rows)
        sel = slice(None) if rows[3] else slice(rows[0], rows[0] + rows[1] * rows[2], rows[2])
        got = decode(img.cpu().numpy()[sel].reshape(-1, 4)).reshape(-1, EW)
        assert (got >= -1).all() and (got == ids.cpu().numpy()[sel]).all(), (variant, rows)


@pytest.mark.parametrize("variant", [3, 8])
def test_coverage_is_the_draws_coverage(actx, libs, variant):
    """spp 4 over 3 progressive frames: the draw's green channel is 8 cov + 0.21 (1 - cov) with cov the blended coverage."""
    emission_ctx(actx, 4)
    actx.set_option("fast_variant", variant)
    img = torch.zeros((EH, EW, 4), dtype=torch.float32, device="cuda")
    alb = torch.zeros((EH, EW, 4), dtype=torch.float32, device="cuda")
    for f in range(3):
        actx.draw(f, 1, EW, EH, img, flags=PROG, mode=libs.MODE_FAST)
        actx.draw_aovs(f, 1, EW, EH, albedo=alb, flags=PROG)
    g = img.cpu().numpy()[..., 1].astype(np.float64)
    cov = alb.cpu().numpy()[..., 3].astype(np.float64)
    assert 0.2 < (cov > 0.999).mean() < 0.95 and ((cov > 0) & (cov < 1)).any()
    assert np.abs(g - (8.0 * cov + 0.21 * (1.0 - cov))).max() < 2e-5


# ---- 3. pixel footprints of scene A ----------------------------------------------------------------------------------
def test_pixel_footprints(actx, libs):
    w = h = 64
    s, m, c, em = F.furnace_scene(w, h)
    actx.set_scene(s, m, c, em)
    actx.set_spp(16)
    B = 16
    albs, nrms, idss = [], [], []
    for b in range(B):
        alb, nrm, ids = dev_buffers(h, w)
        assert actx.draw_aovs(b, 1, w, h, alb, nrm, ids) == w * h * 16
        a_, n_, i_ = np_(alb, nrm, ids)
        albs.append(a_); nrms.append(n_); idss.append(i_)
    albs, nrms, idss = np.array(albs), np.array(nrms, np.float64), np.array(idss)
    assert (albs[..., 3] == 1).all() and (idss == 0).all()
    assert np.allclose(albs[..., :3], m["albedo"][0], rtol=2 ** -20, atol=0)
    # each pixel's mean lies within the range of its footprint (a dense grid, plus the grid's distance to the corners)
    p, wq, _ = F.footprint_hits(c, w, h, nq=12)
    o = c["origin"][0].astype(np.float64)
    depth = np.linalg.norm(p - o, axis=-1)
    normal = p / F.RECEIVER_R
    for val, got in ((depth[..., None], nrms[..., 3:]), (normal, nrms[..., :3])):
        lo, hi = val.min(2), val.max(2)
        marg = 0.05 * (hi - lo) + 2e-6
        assert ((got >= lo - marg) & (got <= hi + marg)).all()
    p4, wq4, _ = F.footprint_hits(c, w, h)
    e_depth = (np.linalg.norm(p4 - o, axis=-1) * wq4).sum(-1)
    e_normal = (p4 / F.RECEIVER_R * wq4[:, None]).sum(-2)
    bins = F.bins_by(None, key=e_depth)
    F.check_bins(nrms[..., 3:], e_depth[..., None], bins)
    F.check_bins(nrms[..., :3], e_normal, bins)


# ---- 4. lens coverage of scene B5 ------------------------------------------------------------------------------------
def test_lens_coverage(actx, libs):
    s, m, c, em, w, h, e, bins, mitsuba, ls = F.b_case("b5")
    _, cov = F.b5_expect(s, m, c, w, h)
    actx.set_scene(s, m, c, em)
    actx.set_spp(16)
    batches = []
    for b in range(16):
        alb = torch.zeros((h, w, 4), dtype=torch.float32, device="cuda")
        actx.draw_aovs(b, 1, w, h, albedo=alb)
        batches.append(alb.cpu().numpy()[..., 3:].astype(np.float64))
    batches = np.array(batches)
    F.check_bins(batches, cov[..., None], bins)
    assert (batches[:, cov == 0] == 0).all() and (batches[:, cov == 1] == 1).all()
    assert (cov == 0).sum() > 1000 and (cov == 1).sum() > 1000


# ---- 5. blend and regions --------------------------------------------------------------------------------------------
RW, RH = 160, 90


def ref_ctx(ctx, libs):
    sph, mats, cam, em = libs.reference_scene(RW, RH)
    ctx.set_scene(sph, mats, cam, em)
    ctx.set_spp(4)


def test_progressive_calls_match_one_call(actx, libs):
    ref_ctx(actx, libs)
    k = 4
    one = dev_buffers(RH, RW)
    actx.draw_aovs(0, k, RW, RH, *one, flags=PROG)
    step = dev_buffers(RH, RW)
    for f in range(k):
        actx.draw_aovs(f, 1, RW, RH, *step, flags=PROG)
    a1, n1, i1 = np_(*one)
    a2, n2, i2 = np_(*step)
    assert np.allclose(a1, a2, rtol=1e-5, atol=1e-6) and np.allclose(n1, n2, rtol=1e-5, atol=1e-5)
    assert ((a1[..., 3] > 0) & (a1[..., 3] < 1)).any()       # partly covered pixels: the blend is exercised
    # ids are sample 0 of frame frameCount: the one-call ids are the ids of the first single-frame call
    first = dev_buffers(RH, RW)
    actx.draw_aovs(0, 1, RW, RH, *first, flags=PROG)
    assert (np_(first[2])[0] == i1).all() and (np_(step[2])[0] != i1).any()


def test_zero_prev_weight_ignores_nan(actx, libs):
    ref_ctx(actx, libs)
    for frame, flags in ((0, PROG), (5, 0)):
        alb, nrm, ids = dev_buffers(RH, RW)
        alb.fill_(float("nan")); nrm.fill_(float("nan"))
        actx.draw_aovs(frame, 1, RW, RH, alb, nrm, ids, flags=flags)
        assert torch.isfinite(alb).all() and torch.isfinite(nrm).all()
        ha, hn = np.full((RH, RW, 4), np.nan, np.float32), np.full((RH, RW, 4), np.nan, np.float32)
        actx.draw_aovs(frame, 1, RW, RH, ha, hn, flags=flags)
        assert not bits_differ(ha, alb.cpu().numpy()).any() and not bits_differ(hn, nrm.cpu().numpy()).any()


def test_regions_and_shards(actx, libs):
    ref_ctx(actx, libs)
    full = dev_buffers(RH, RW)
    actx.draw_aovs(3, 2, RW, RH, *full, flags=PROG)
    fa, fn, fi = np_(*full)
    # rows outside the region are untouched
    alb, nrm, ids = dev_buffers(RH, RW)
    alb.fill_(7.0); nrm.fill_(-3.0); ids.fill_(12345)
    actx.draw_aovs(3, 2, RW, RH, alb, nrm, ids, flags=PROG, rows=(1, 29, 3, 0))
    a, n, i = np_(alb, nrm, ids)
    inside = np.zeros(RH, bool); inside[1:88:3] = True
    assert (a[~inside] == 7).all() and (n[~inside] == -3).all() and (i[~inside] == 12345).all()
    # strided shards assemble bitwise into the full image; zero prev weight, so the fill does not matter
    shard = dev_buffers(RH, RW)
    for k in range(3):
        assert actx.draw_aovs(3, 2, RW, RH, *shard, flags=PROG, rows=(k, len(range(k, RH, 3)), 3, 0)) == \
            len(range(k, RH, 3)) * RW * 4 * 2
    sa, sn, si = np_(*shard)
    assert not bits_differ(sa, fa).any() and not bits_differ(sn, fn).any() and (si == fi).all()
    # a packed band holds the band's rows
    band = dev_buffers(40, RW)
    actx.draw_aovs(3, 2, RW, RH, *band, flags=PROG, rows=(17, 40, 1, 1))
    ba, bn, bi = np_(*band)
    assert not bits_differ(ba, fa[17:57]).any() and not bits_differ(bn, fn[17:57]).any() and (bi == fi[17:57]).all()
    # two identical calls, identical bits
    again = dev_buffers(RH, RW)
    actx.draw_aovs(3, 2, RW, RH, *again, flags=PROG)
    ga, gn, gi = np_(*again)
    assert not bits_differ(ga, fa).any() and not bits_differ(gn, fn).any() and (gi == fi).all()


# ---- 6. buffers, accounting, ordering --------------------------------------------------------------------------------
def test_trace_buffer_kinds_and_subsets(actx, libs):
    ref_ctx(actx, libs)
    sph, mats, cam, em = libs.reference_scene(RW, RH)
    rays = libs.camera_rays(cam, RW, RH, per_pixel=2, seed=4)
    n = len(rays)
    (ra, rn, ri), traced = actx.trace_aovs(rays)
    assert isinstance(ra, np.ndarray) and ra.shape == (n, 4) and rn.shape == (n, 4) and ri.shape == (n,) and ri.dtype == np.int32
    assert traced == n and ((ri >= 0).mean() > 0.3) and (ri == -1).any()

    def same(a, nrm, ids, want=(True, True, True)):
        for got, ref, w in ((a, ra, want[0]), (nrm, rn, want[1]), (ids, ri, want[2])):
            if w:
                got = got.cpu().numpy() if hasattr(got, "cpu") else got
                assert not bits_differ(got.reshape(n, -1)[None], ref.reshape(n, -1)[None]).any()

    pin = torch.empty((n, 6), dtype=torch.float32, pin_memory=True); pin.numpy()[...] = rays
    (a, nrm, ids), t = actx.trace_aovs(pin)
    assert not a.is_cuda and t == traced
    same(a, nrm, ids)
    base = torch.zeros((n + 1, 6), dtype=torch.float32, device="cuda"); base[1:] = torch.from_numpy(rays).cuda()
    side = torch.cuda.Stream()
    torch.cuda.synchronize()
    a, nrm, ids = actx.trace_aovs(base[1:], stream=side.cuda_stream, want_rays=False)
    side.synchronize()
    assert a.is_cuda
    same(a, nrm, ids)
    rp, ap, np_p, ip = actx.mem_alloc(n * 24), actx.mem_alloc(n * 16), actx.mem_alloc(n * 16), actx.mem_alloc(n * 4)
    try:
        actx.mem_from_host(rp, rays)
        _, t = actx.trace_aovs(rp, albedo=ap, normal=np_p, ids=ip, n=n)
        same(actx.mem_to_host(ap, np.empty((n, 4), np.float32)), actx.mem_to_host(np_p, np.empty((n, 4), np.float32)),
             actx.mem_to_host(ip, np.empty(n, np.int32)))
        assert t == traced
    finally:
        for p in (rp, ap, np_p, ip):
            actx.mem_free(p)
    for host in (True, False):
        for want in itertools.product((True, False), repeat=3):
            if not any(want):
                continue
            mk = (lambda shp, dt: np.full(shp, 5, dt)) if host else \
                 (lambda shp, dt: torch.full(shp, 5, dtype=getattr(torch, np.dtype(dt).name), device="cuda"))
            bufs = [mk((n, 4), np.float32) if want[0] else None, mk((n, 4), np.float32) if want[1] else None,
                    mk((n,), np.int32) if want[2] else None]
            r = rays if host else torch.from_numpy(rays).cuda()
            (a, nrm, ids), t = actx.trace_aovs(r, *bufs)
            assert t == traced and [b is None for b in (a, nrm, ids)] == [not x for x in want]
            same(a, nrm, ids, want)


def test_draw_buffer_kinds_and_subsets(actx, libs):
    ref_ctx(actx, libs)
    ref = dev_buffers(RH, RW)
    actx.draw_aovs(2, 1, RW, RH, *ref)
    ref = np_(*ref)
    for want in itertools.product((True, False), repeat=3):
        if not any(want):
            continue
        host = [np.zeros((RH, RW, 4), np.float32), np.zeros((RH, RW, 4), np.float32), np.zeros((RH, RW), np.int32)]
        dev = list(dev_buffers(RH, RW))
        hb = [b if w else None for b, w in zip(host, want)]
        db = [b if w else None for b, w in zip(dev, want)]
        assert actx.draw_aovs(2, 1, RW, RH, *hb) == RW * RH * 4
        actx.draw_aovs(2, 1, RW, RH, *db)
        for k in range(3):
            if want[k]:
                assert (host[k].view(np.uint32) == ref[k].view(np.uint32)).all()
                assert (dev[k].cpu().numpy().view(np.uint32) == ref[k].view(np.uint32)).all()
    # a progressive host draw uploads `prev` and matches the device draw
    hb = [np.array(r) for r in ref]
    db = [torch.from_numpy(np.array(r)).cuda() for r in ref]
    actx.draw_aovs(3, 1, RW, RH, *hb, flags=PROG)
    actx.draw_aovs(3, 1, RW, RH, *db, flags=PROG)
    for h_, d_ in zip(hb, db):
        assert not bits_differ(h_.reshape(RH, RW, -1), d_.cpu().numpy().reshape(RH, RW, -1)).any()


def test_refusals(actx, libs):
    ref_ctx(actx, libs)
    L, h = actx._L, actx._h
    rays = torch.zeros((70, 6), dtype=torch.float32, device="cuda")
    f4 = torch.zeros((RH * RW, 4), dtype=torch.float32, device="cuda")
    i1 = torch.zeros(RH * RW, dtype=torch.int32, device="cuda")
    vp = ctypes.c_void_p
    R, A, I = vp(rays.data_ptr()), vp(f4.data_ptr()), vp(i1.data_ptr())
    cnt = ctypes.c_longlong(-1)

    def trace(r, ron, n, a, nrm, ids, oon=1):
        return L.tpt_trace_aovs(h, r, ron, n, a, nrm, ids, oon, ctypes.byref(cnt), None)

    def draw(nf, a, nrm, ids, rows=(0, RH, 1, 0), width=RW):
        return L.tpt_draw_aovs(h, 0, nf, width, RH, *rows, a, nrm, ids, 1, 0, ctypes.byref(cnt), None)

    def refused(text, rc):
        assert rc != 0
        assert text in L.tpt_last_error(h).decode(), (text, L.tpt_last_error(h).decode())

    refused("albedo4, normal4 and ids are all null", trace(R, 1, 4, None, None, None))
    refused("albedo4, normal4 and ids are all null", draw(1, None, None, None))
    refused("null rays6", trace(None, 1, 4, A, None, None))
    refused("n < 0", trace(R, 1, -1, A, None, None))
    refused("n > 2^32 - 1", trace(R, 1, 1 << 32, A, None, None))
    refused("rays6 is not 4-byte aligned", trace(vp(rays.data_ptr() + 2), 1, 4, A, None, None))
    refused("albedo4 is not 16-byte aligned", trace(R, 1, 4, vp(f4.data_ptr() + 4), None, None))
    refused("normal4 is not 16-byte aligned", draw(1, None, vp(f4.data_ptr() + 8), None))
    refused("ids is not 4-byte aligned", trace(R, 1, 4, None, None, vp(i1.data_ptr() + 2)))
    host = np.zeros((4, 6), np.float32)
    refused("rays6 is not CUDA memory", trace(vp(host.ctypes.data), 1, 4, A, None, None))
    refused("ids is not CUDA memory", draw(1, None, None, vp(host.ctypes.data)))
    refused("numFrames > 256", draw(257, A, None, None))
    refused("rows outside the image", draw(1, A, None, None, rows=(1, RH, 1, 0)))
    if torch.cuda.device_count() > 1:
        other = torch.zeros((4, 4), dtype=torch.float32, device="cuda:1")
        refused("lives on device 1", trace(R, 1, 4, vp(other.data_ptr()), None, None))
        refused("lives on device 1", draw(1, A, vp(other.data_ptr()), None))
    # n == 0 and numRows == 0: nothing launched, no rays
    cnt.value = -1
    assert trace(vp(host.ctypes.data), 0, 0, vp(host.ctypes.data), None, None, 0) == 0 and cnt.value == 0
    assert actx.last_launch_count() == 0
    cnt.value = -1
    assert draw(1, A, None, None, rows=(0, 0, 1, 0)) == 0 and cnt.value == 0 and actx.last_launch_count() == 0


def test_accounting(actx, libs):
    s, m, c, em = F.furnace_scene(64, 64)
    actx.set_scene(s, m, c, em)
    actx.set_spp(3)
    actx.read_ray_count()
    alb = torch.zeros((64, 64, 4), dtype=torch.float32, device="cuda")
    drawn = actx.draw_aovs(0, 5, 64, 64, albedo=alb, flags=PROG, rows=(2, 20, 3, 0))
    assert drawn == 20 * 64 * 3 * 5
    assert actx.last_launch_count() == 2 and actx.last_kernel_ms() > 0
    rays = libs.camera_rays(c, 64, 64, per_pixel=1, seed=2)[:1000]
    bad = [(3, 0.0), (3, np.nan), (4, np.inf), (5, -np.inf), (0, np.nan), (1, np.inf)]
    for i in range(0, 1000, 3):
        col, val = bad[(i // 3) % len(bad)]
        if col == 3 and val == 0.0:
            rays[i, 3:] = 0.0
        else:
            rays[i, col] = val
    rays[1, 3:] = (1e-30, -1e-30, 1e-30)                    # does not normalise
    (a, nrm, ids), traced = actx.trace_aovs(rays)
    valid = np.isfinite(rays).all(1) & (np.abs(rays[:, 3:]).max(1) > 0)
    valid[1] = False
    assert traced == int(valid.sum()) and actx.last_launch_count() == 2
    assert (a[~valid] == 0).all() and (nrm[~valid] == 0).all() and (ids[~valid] == -1).all()
    assert (ids[valid] == 0).all() and (a[valid, 3] == 1).all()
    assert actx.read_ray_count() == drawn + traced


@pytest.mark.parametrize("mode", ["exact", "fast"])
def test_draws_around_aovs_are_unchanged(actx, libs, mode):
    ref_ctx(actx, libs)
    md = libs.MODE_EXACT if mode == "exact" else libs.MODE_FAST
    alone = torch.zeros((RH, RW, 4), dtype=torch.float32, device="cuda")
    actx.draw(0, 1, RW, RH, alone, flags=PROG, mode=md)
    actx.draw(1, 1, RW, RH, alone, flags=PROG, mode=md)
    side = torch.cuda.Stream()
    mixed = torch.zeros((RH, RW, 4), dtype=torch.float32, device="cuda")
    aovs = dev_buffers(RH, RW)
    actx.draw(0, 1, RW, RH, mixed, flags=PROG, mode=md, want_rays=False)
    actx.draw_aovs(0, 2, RW, RH, *aovs, flags=PROG, stream=side.cuda_stream, want_rays=False)
    actx.draw(1, 1, RW, RH, mixed, flags=PROG, mode=md, stream=side.cuda_stream, want_rays=False)
    torch.cuda.synchronize()
    a, b = alone.cpu().numpy(), mixed.cpu().numpy()
    if mode == "exact":
        assert not bits_differ(a, b).any()
    else:
        assert rel_l2(b, a) < 1e-5
