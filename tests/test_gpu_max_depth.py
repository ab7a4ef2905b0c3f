"""The fast mode's per-call path depth cap ("max_depth") and its Russian roulette past depth 10, on the GPU.

1. Default equality: max_depth set to 10, or to 37 and back to 10, is a context that never set it: bits, ray counts and
   kernels through every fast call, on the 46- and 4096-sphere scenes, light sampling on and off.
2. Mirror corridor through the cap: mirror_chain's all-mirror corridor (roughness 0: no draw that matters, so every
   chain is deterministic) against sample_replay's float64 replay with its cap set to n, values and ray counts, for n in
   {1, 2, 5, 9, 10}, and for n in {11, 32, 256} with every mirror's red albedo 1 (q = 1: the roll never ends a chain).
3. Roulette on the same corridor with every albedo channel below 1: per ray, the mean of trace_samples against the
   replay's cap-n value, and the rays per sample against their closed form from the chain's throughputs.
4. Dense media: the white furnace of test_gpu_media at cap 256 recovers L (1 - p_cap(256)); with light absorption the
   roll really ends paths, and the mean is the roll-free float64 model's at cap 256 (unbiasedness).
5. Float64 replay of single samples at n in {3, 24}, light sampling on and off: Lambert, rough Metal and glass through
   sample_replay with its cap set to n (at 24 the samples that never reach a hit at depth 10, which draw exactly what
   the replay draws), and a scattering medium in glass through a replay in this file that also draws the roll.
6. Contract: refusals keep the value, routing, calls in flight keep their cap, nothing is uploaded, AOVs do not change,
   and the option combines with media, textures and both sampling options."""
import numpy as np
import pytest
import torch

import mirror_chain as mc
import sample_replay as sr
import test_gpu_media as gm
from test_gpu_media import GLASS46, L_ENV, SCENES, _kinds, _reference_form_only, _same
from test_gpu_textures import TEX_KERNELS, _const_layers, _draw, _every_call
from toypathtracer_b200 import MODE_EXACT, MODE_FAST, MODE_REFGPU, MODE_REFGPU_FAST, Context, TptError, scenes

pytestmark = pytest.mark.gpu

REF_DEPTH = 10           # TPT_MAX_DEPTH: the default, and the depth the roll starts at


def capped_replay(monkeypatch, sc, rays, seeds, n):
    """sample_replay.replay with its depth cap (the module's MAX_DEPTH, read when a hit is shaded) set to n. It draws no
    roll: its samples are the kernel's wherever no path ray hits at depth >= 10 (nvert <= 10), or where nothing the path
    draws after its first roll matters and every roll has q = 1."""
    monkeypatch.setattr(sr, "MAX_DEPTH", n)
    return sr.replay(sc, seeds, rays=rays)


@pytest.fixture
def dctx(gpu_ctx):
    yield gpu_ctx
    gpu_ctx.set_media(None)
    gpu_ctx.set_textures(None)
    gpu_ctx.set_emission_textures(None)
    gpu_ctx.set_environment(None)
    for k, v in (("max_depth", 10), ("fast_variant", -1), ("fast_kform", 2), ("light_sampling", 1),
                 ("environment_sampling", 0), ("emission_texture_sampling", 0), ("mitsuba_compare", 0),
                 ("scene_upload_always", 0)):
        gpu_ctx.set_option(k, v)
    gpu_ctx.set_spp(4)


# ---- 1. default equality ---------------------------------------------------------------------------------------------
def _all_calls(ctx, which, ls, kform):
    make, w, h, variants = SCENES[which]
    s, m, c, em = make()
    ctx.set_option("light_sampling", ls)
    ctx.set_option("fast_kform", kform)
    ctx.set_scene(s, m, c, em)
    res = _every_call(ctx, w, h, c, s, (-1, 3, 9) if which == "46" else variants)
    _draw(ctx, w, h)
    return res, ctx.last_kernels()


@pytest.mark.parametrize("kform", [2, 0])
@pytest.mark.parametrize("ls", [1, 0])
@pytest.mark.parametrize("which", sorted(SCENES))
def test_default_is_the_context_that_never_set_it(dctx, which, ls, kform):
    """Also with "fast_kform" 0, which runs the reference-form instances that take the call's cap."""
    fresh = Context(0)
    try:
        ref, kern = _all_calls(fresh, which, ls, kform)
    finally:
        fresh.close()
    dctx.set_option("max_depth", 10)
    got, k = _all_calls(dctx, which, ls, kform)
    assert k == kern
    _same(got, ref)
    dctx.set_option("max_depth", 37)
    dctx.set_option("max_depth", 10)
    got, k = _all_calls(dctx, which, ls, kform)
    assert k == kern
    _same(got, ref)


# ---- 2./3. the mirror corridor -----------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def corridor():
    s, m, em = mc.corridor(6, "compact")                     # few small spheres: chains between floor and ceiling
    rays = mc.candidate_rays(s, 1500, seed=57)
    return s, m, em, rays


def _set_corridor(ctx, s, m, em, n):
    """max_depth n; at n = 10 with "fast_kform" 0, so that the default cap is checked in the instances that take the
    call's cap (every other n runs them anyway)."""
    ctx.set_option("fast_kform", 0)
    ctx.set_option("max_depth", n)
    ctx.set_scene(s, m, mc.point_camera(mc.CAMERA_O, (0, 0, -1))[0], em)


def _chains(monkeypatch, s, m, em, rays, n, ls):
    """The corridor's chains under cap n: values, rays (= segments), the hit of each segment, well-conditioned."""
    res = capped_replay(monkeypatch, sr.Scene(s, m, em, ls=bool(ls)), rays, sr.ray_seeds(np.arange(len(rays)), 1, 0, 0), n)
    return res


@pytest.mark.parametrize("n,red_one", [(1, False), (2, False), (5, False), (9, False), (10, False), (11, True),
                                       (32, True), (256, True)])
def test_mirror_corridor_through_the_cap(dctx, monkeypatch, corridor, n, red_one):
    s, m, em, rays = corridor
    m = m.copy()
    if red_one:
        m["albedo"][:, 0] = 1.0                              # q = 1 at every roll: the chains stay deterministic
    for ls in (1, 0):
        res = _chains(monkeypatch, s, m, em, rays, n, ls)
        sel = np.nonzero(res["well"])[0]
        assert len(sel) >= 40
        if n > REF_DEPTH:
            assert (res["rays"][sel] > REF_DEPTH + 1).sum() >= 5, "too few chains past the reference's cap"
        if n < REF_DEPTH:
            assert res["flags"]["cap"][sel].sum() >= 5
        v, tol = res["v"][sel], res["tol"][sel] + 4 * 2.0 ** -23 * np.abs(res["v"][sel]).max(1)
        dctx.set_option("light_sampling", ls)
        _set_corridor(dctx, s, m, em, n)
        out, traced = dctx.trace_rays(torch.from_numpy(rays[sel]).cuda(), spp=2, frame=n)
        err = np.abs(out.cpu().numpy()[:, :3] - v).max(1)
        bad = err > tol
        assert not bad.any(), (n, ls, int(bad.sum()), res["rays"][sel][bad][:5], (err / tol)[bad][:5])
        assert traced == 2 * int(res["rays"][sel].sum()), (n, ls, traced, 2 * int(res["rays"][sel].sum()))
        assert all(k.startswith(TEX_KERNELS) for k in _kinds(dctx)), dctx.last_kernels()


def expected_rays(ids, seg, alb):
    """Distribution of the rays one sample of a deterministic mirror chain traces under the roll: ids the chain's hits
    (segment k hits ids[k]), seg its segments under the cap. Segment k + 1 is traced when hit k continues and, from hit
    10 on, survives its roll with q_k = min(1, max channel of thr_k), thr_k the albedo product of hits 0 .. k-1 divided
    by the q of every earlier roll. Returns (mean, variance)."""
    thr = np.ones(3)
    surv = [1.0]                                             # P(segment k traced)
    for k in range(seg - 1):
        q = 1.0
        if k >= REF_DEPTH:
            q = min(1.0, thr.max())
            thr = thr / q
        thr = thr * alb[ids[k]]
        surv.append(surv[-1] * q)
    surv = np.array(surv)
    p = surv - np.append(surv[1:], 0.0)                      # P(rays = k + 1)
    r = np.arange(1, seg + 1)
    mean = (p * r).sum()
    return mean, (p * r * r).sum() - mean ** 2


@pytest.mark.parametrize("n", [16, 64, 256])
def test_roulette_on_a_deterministic_chain(dctx, monkeypatch, corridor, n):
    s, m, em, rays = corridor                                # albedos k / 64 <= 63 / 64: the roll ends chains
    assert (m["albedo"] < 1).all()
    res = _chains(monkeypatch, s, m, em, rays, n, 1)         # without the roll: the cap-n value, every segment traced
    long_ = np.nonzero(res["well"] & (res["rays"] >= REF_DEPTH + 2))[0]        # at least one roll decides a segment
    assert len(long_) >= 4, len(long_)
    pick = np.random.default_rng(n).choice(long_, min(6, len(long_)), replace=False)
    _set_corridor(dctx, s, m, em, n)
    dev = torch.from_numpy(rays).cuda()
    spp = 8192
    ended = 0
    alb = m["albedo"].astype(np.float64)
    for i in pick:
        (s4, q4), traced = dctx.trace_samples(dev, entries=torch.tensor([i], dtype=torch.int32).cuda(), spp=spp, frame=3)
        s4, q4 = s4.cpu().numpy().astype(np.float64)[0], q4.cpu().numpy().astype(np.float64)[0]
        assert s4[3] == spp
        mean = s4[:3] / spp
        se = np.sqrt(np.maximum(q4[:3] / spp - mean ** 2, 0) / spp)
        v = res["v"][i]
        assert (np.abs(mean - v) <= 5 * se + res["tol"][i] + 1e-6 * np.abs(v)).all(), (i, mean, v, se)
        ids = [int(x) for x in res["trail"][i] if x != -3]     # segment k's hit (one path ray per step: no lights hit)
        er, var = expected_rays(ids, int(res["rays"][i]), alb)
        rse = np.sqrt(var / spp)
        assert abs(traced / spp - er) <= 5 * rse + 1e-9, (i, traced / spp, er, rse)
        ended += traced < spp * res["rays"][i]
    assert ended == len(pick)                                # the roll really ended paths (q < 1 on every chain)


# ---- 4. dense media ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("g", [-0.6, 0.0, 0.8])
def test_white_furnace_recovers_its_energy(dctx, monkeypatch, g):
    monkeypatch.setattr(gm, "MAX_DEPTH", 256)
    radius, ri, sigma_s = 1.0, 1.5, 4.0
    dctx.set_scene(*gm.glass_scene(radius, ri))
    dctx.set_environment(np.broadcast_to(L_ENV, (4, 8, 3)).copy())
    dctx.set_media(np.float32([[0.0, 0.0, 0.0, sigma_s, g]]))
    dctx.set_option("max_depth", 256)
    val, capped = gm.mc_model(200_000, (0, 0, 0), sigma_s, g, radius, ri, seed=int(g * 100) & 0xffff)
    p_cap = capped.mean()
    p_se = np.sqrt(max(p_cap * (1 - p_cap), 1.0 / capped.size) / capped.size)
    mean, se, _ = gm._per_sample_stats(dctx, gm._centre_rays(4096, 5), 16, 1)
    want = L_ENV * (1 - p_cap)
    tol = 5 * np.sqrt(se ** 2 + (L_ENV * p_se) ** 2)
    print(f"g {g}: p_cap(256) {p_cap:.2e}, kernel {mean / L_ENV}")
    assert (np.abs(mean - want) <= tol).all(), (g, p_cap, mean / L_ENV, se)


@pytest.mark.parametrize("ls", [1, 0])
def test_absorbing_dense_medium_is_unbiased(dctx, monkeypatch, ls):
    """sigma_a > 0: thr < 1, so the roll ends paths; the mean must be the roll-free model's at the same cap."""
    monkeypatch.setattr(gm, "MAX_DEPTH", 256)
    radius, ri = 1.0, 1.5
    sa, ss, g = (0.02, 0.06, 0.15), 4.0, 0.3
    dctx.set_option("light_sampling", ls)
    dctx.set_scene(*gm.glass_scene(radius, ri))
    dctx.set_environment(np.broadcast_to(L_ENV, (4, 8, 3)).copy())
    dctx.set_media(np.float32([[*sa, ss, g]]))
    dctx.set_option("max_depth", 256)
    val, _ = gm.mc_model(200_000, sa, ss, g, radius, ri, seed=13 + ls)
    want = L_ENV * val.mean(0)
    want_se = L_ENV * val.std(0) / np.sqrt(val.shape[0])
    rays = gm._centre_rays(4096, 9)
    mean, se, _ = gm._per_sample_stats(dctx, rays, 16, 1)
    assert (np.abs(mean - want) <= 5 * np.sqrt(se ** 2 + want_se ** 2)).all(), (mean, want, se, want_se)
    dctx.set_option("max_depth", 10)                         # the higher cap gives back what the default's takes
    mean10, se10, _ = gm._per_sample_stats(dctx, rays, 16, 1)
    assert (mean - mean10 > 5 * np.sqrt(se ** 2 + se10 ** 2)).all(), (mean, mean10)


# ---- 5. float64 replay ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def mixed():
    s, m, em = sr.mixed_corridor(40, "compact", n_lights=4)
    rays = np.concatenate([sr.candidate_rays(s, 1600, seed=44), sr.inside_glass_rays(s, m, 200, seed=40)])
    return s, m, em, rays


@pytest.mark.parametrize("ls", [1, 0])
@pytest.mark.parametrize("n", [3, 24])
def test_samples_replay_in_float64(dctx, monkeypatch, mixed, n, ls):
    """At n <= 10 nothing new is drawn: every well-conditioned sample is the replay's with its cap at n. At n > 10 a
    sample whose path rays never hit at depth >= 10 draws exactly what the replay draws, and must be its sample; the
    roll's own draw is replayed by test_medium_samples_replay_in_float64 and checked in distribution above."""
    s, m, em, rays = mixed
    dctx.set_option("light_sampling", ls)
    dctx.set_option("max_depth", n)
    dctx.set_scene(s, m, sr.lens_camera(), em)
    sc = sr.Scene(s, m, em, ls=bool(ls))
    frame = 5 + n + ls
    res = capped_replay(monkeypatch, sc, rays, sr.ray_seeds(np.arange(len(rays)), 1, 0, frame), n)
    well = res["well"] & (res["nvert"] <= REF_DEPTH)       # no path-ray hit at depth >= 10: no roll
    assert well.sum() >= 300, int(well.sum())
    if n > REF_DEPTH:
        assert (well & (res["nvert"] > 3)).sum() >= 10         # paths that n = 3 would have ended
    else:
        assert (res["flags"]["cap"][well]).sum() >= 5
    dev = torch.from_numpy(rays).cuda()
    out, traced = dctx.trace_rays(dev, spp=1, frame=frame)
    out = out.cpu().numpy()
    v, tol = res["v"], res["tol"] + 4 * 2.0 ** -23 * np.abs(res["v"]).max(1)
    err = np.abs(out[:, :3] - v).max(1)
    bad = np.nonzero(well & ~(err <= tol))[0]
    assert not len(bad), [(int(i), sr.describe(res, i), out[i, :3], v[i]) for i in bad[:6]]
    idx = np.nonzero(well)[0].astype(np.int32)
    _, n_well = dctx.trace_samples(dev, entries=torch.from_numpy(idx).cuda(), spp=1, frame=frame)
    assert n_well == int(res["rays"][idx].sum())


def replay_medium(ray, seed, sph, max_depth):
    """test_gpu_media.replay_one with the call's cap and the roll: before anything else at a path ray's hit at depth
    >= 10 (when max_depth > 10), u against q = min(1, max channel of thr)."""
    st = sr.Stream(np.array([seed], np.uint32))
    draw = lambda: float(sr.u01(st.draw(np.array([0]))[0]))  # noqa: E731
    cen = sph["center"].astype(np.float64)
    rad = sph["radius"].astype(np.float64)
    o = ray[:3].astype(np.float64)
    d = ray[3:].astype(np.float64)
    d /= np.linalg.norm(d)
    thr, depth, rays, err = np.ones(3), 0, 0, 1e-6
    ok = True
    k_margin = 16.0
    zero = lambda: (np.zeros(3), rays, ok, np.full(3, 1e-6))  # noqa: E731
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
                ok &= abs(t - gm.TMIN) > 1e-5
                if t > gm.TMIN:
                    ts_all.append(t)
                    if t < best:
                        best, bid = t, k
                    break
        if bid < 0:
            return thr, rays, ok, 1e-6 + (k_margin * err * 4 + 1e-5 + 1e-6 * depth) * np.abs(thr)
        ts_all.sort()
        if len(ts_all) > 1:
            ok &= ts_all[1] - ts_all[0] > k_margin * err
        t = best
        if max_depth > REF_DEPTH and depth >= REF_DEPTH:
            u = draw()
            q = min(1.0, thr.max())
            ok &= abs(u - q) > 1e-5
            if u >= q:
                return zero()
            thr = thr / q
        pos = o + d * t
        nrm = (pos - cen[bid]) / rad[bid]
        dn = d @ nrm
        ok &= abs(dn) > k_margin * err
        ri = gm.REPLAY_SPHERES[bid][2]
        med = gm.REPLAY_MEDIA[bid]
        sa, ss, g = med[:3].astype(np.float64), float(med[3]), float(med[4])
        if dn > 0:
            if ss > 0:
                t_s = -np.log(1 - draw()) / ss
                ok &= abs(t_s - t) > k_margin * err * max(t, 1.0)
                if t_s < t:
                    if depth >= max_depth:
                        return zero()
                    thr = thr * np.exp(-sa * t_s)
                    o = o + d * t_s
                    xi1, xi2 = draw(), draw()
                    ok &= abs(d[2]) > k_margin * err
                    d = gm.hg_dirs(d[None, :], g, np.array([xi1]), np.array([xi2]))[0]
                    depth += 1
                    err = err * 1.5 + 1e-5
                    continue
            thr = thr * np.exp(-sa * t)
        if depth >= max_depth:
            return zero()
        if dn > 0:
            out_n, nint, cosine = -nrm, ri, ri * dn
        else:
            out_n, nint, cosine = nrm, 1.0 / ri, -dn
        dt = d @ out_n
        discr = 1.0 - nint * nint * (1.0 - dt * dt)
        ok &= abs(discr) > k_margin * err
        refl_p = gm.schlick(cosine, ri) if discr > 0 else 1.0
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
@pytest.mark.parametrize("n", [3, 24])
def test_medium_samples_replay_in_float64(dctx, n, ls):
    dctx.set_option("light_sampling", ls)
    sph, mats, cam, em = gm.replay_scene()
    dctx.set_scene(sph, mats, cam, em)
    dctx.set_environment(np.ones((4, 8, 3), np.float32))
    dctx.set_media(gm.REPLAY_MEDIA)
    dctx.set_option("max_depth", n)
    rng = np.random.default_rng(31 + ls + n)
    n_out, n_in = 300, 300
    aim = sph["center"][rng.integers(0, len(sph), n_out)] + rng.normal(scale=0.4, size=(n_out, 3))
    orig = rng.normal(size=(n_out, 3))
    orig = 6.0 * orig / np.linalg.norm(orig, axis=1, keepdims=True)
    outside = np.concatenate([orig, aim - orig], 1).astype(np.float32)
    rays = np.concatenate([outside, sr.inside_glass_rays(sph, mats, n_in, seed=7 + ls)])
    frame = 4
    (s4, _q4), _ = dctx.trace_samples(rays, spp=1, frame=frame)
    seeds = sr.ray_seeds(np.arange(len(rays)), 1, 0, frame)
    good, deep, bad = 0, 0, []
    for i in range(len(rays)):
        val, nr, ok, tol = replay_medium(rays[i], seeds[i], sph, n)
        if not ok:
            continue
        good += 1
        deep += nr > REF_DEPTH + 1
        (_one, _), kr = dctx.trace_samples(rays, entries=np.array([i], np.int32), spp=1, frame=frame)
        if kr != nr or s4[i, 3] != 1 or (np.abs(s4[i, :3] - val) > tol).any():
            bad.append((i, kr, nr, s4[i].tolist(), val.tolist()))
    print(f"medium replay n {n}: {good} of {len(rays)} well-conditioned, {deep} past depth 10, {len(bad)} differ")
    assert not bad, bad[:8]
    assert good >= 0.85 * len(rays), good                   # deeper paths than test_gpu_media's: more ill-conditioned
    if n > REF_DEPTH:
        assert deep >= 5


# ---- 6. contract ------------------------------------------------------------------------------------------------------
def test_refusals_keep_the_value(dctx):
    w, h = 64, 36
    s, m, c, em = scenes.reference_scene(w, h)
    dctx.set_scene(s, m, c, em)
    dctx.set_spp(1)
    dctx.set_option("max_depth", 40)
    ref, rr = _draw(dctx, w, h)
    L = dctx._L
    for bad in (0, -1, 257, 1 << 20):
        assert L.tpt_set_option(dctx._h, b"max_depth", bad) != 0
        assert L.tpt_last_error(dctx._h).decode() == "max_depth: 1..256"
    with pytest.raises(TptError, match="max_depth: 1..256"):
        dctx.set_option("max_depth", 0)
    got, gr = _draw(dctx, w, h)
    assert gr == rr and got.tobytes() == ref.tobytes()        # still 40
    for v in (0, 1, 2, 4, 5, 6, 7, 8):
        dctx.set_option("fast_variant", v)
        with pytest.raises(TptError, match=f'tpt_draw: "max_depth" is 40, and fast_variant {v} keeps the depth cap at 10: '
                                           r'use -1 \(auto\), 3 or 9'):
            _draw(dctx, w, h)
    for v in (3, 9):
        dctx.set_option("fast_variant", v)
        _draw(dctx, w, h)
    dctx.set_option("fast_variant", -1)
    for mode in (MODE_EXACT, MODE_REFGPU, MODE_REFGPU_FAST):
        with pytest.raises(TptError, match=r'tpt_draw: "max_depth" is 40, and only TPT_MODE_FAST draws use it \(set it '
                                           r'back to 10 for exact and reference-GPU draws\)'):
            _draw(dctx, w, h, mode=mode)
    # every existing refusal keeps its text and comes first
    dctx.set_media(gm._media(len(s), {GLASS46: (0.5, 0.5, 0.5, 2.0, 0.3)}))
    with pytest.raises(TptError, match="the scene has media, and only TPT_MODE_FAST"):
        _draw(dctx, w, h, mode=MODE_EXACT)
    dctx.set_option("fast_variant", 5)
    with pytest.raises(TptError, match=r"the scene has media \(tpt_set_media\), and fast_variant 5"):
        _draw(dctx, w, h)
    dctx.set_option("fast_variant", -1)
    dctx.set_media(None)
    dctx.set_option("max_depth", 10)
    _draw(dctx, w, h, mode=MODE_EXACT)                       # allowed again
    dctx.set_option("fast_variant", 5)
    _draw(dctx, w, h)


@pytest.mark.parametrize("which,inst", [("46", "<128, 6, 0>"), ("4096", "<768, 1, 0>")])
def test_route_to_the_reference_form_instances(dctx, which, inst):
    make, w, h, _v = SCENES[which]
    s, m, c, em = make()
    dctx.set_scene(s, m, c, em)
    _draw(dctx, w, h)
    default = dctx.last_kernels()
    for n in (1, 64):
        dctx.set_option("max_depth", n)
        for v in (-1, 3, 9):
            dctx.set_option("fast_variant", v)
            _draw(dctx, w, h)
            k = _kinds(dctx)
            assert _reference_form_only(k, inst) and all(x.startswith(TEX_KERNELS) for x in k), (n, v, k)
        dctx.set_option("fast_variant", -1)
        host = np.zeros((h, w, 4), np.float32)
        dctx.draw(0, 1, w, h, host, mode=MODE_FAST)
        assert _reference_form_only(_kinds(dctx), inst), dctx.last_kernels()
        rays = scenes.camera_rays(c, w, h)
        pts = np.concatenate([np.zeros((8, 3)), np.tile([0, 1, 0], (8, 1))], 1).astype(np.float32)
        for call in (lambda: dctx.trace_rays(rays, spp=2), lambda: dctx.draw_samples(0, w, h, spp=2),
                     lambda: dctx.trace_samples(rays, spp=2), lambda: dctx.trace_irradiance(pts, spp=2)):
            call()
            assert _reference_form_only(_kinds(dctx), inst), dctx.last_kernels()
    dctx.set_option("max_depth", 10)
    _draw(dctx, w, h)
    assert dctx.last_kernels() == default


def test_draw_issued_before_a_change_keeps_its_cap(dctx):
    w, h = 1280, 720
    s, m, c, em = scenes.reference_scene(w, h)
    dctx.set_scene(s, m, c, em)
    dctx.set_spp(1)                                          # one sample per pixel: a draw is bitwise reproducible
    dctx.set_option("max_depth", 64)
    ref, _ = _draw(dctx, w, h)
    buf = torch.zeros((h, w, 4), dtype=torch.float32, device="cuda")
    dctx.draw(0, 1, w, h, buf, mode=MODE_FAST, want_rays=False)     # asynchronous: still in flight
    dctx.set_option("max_depth", 1)
    torch.cuda.synchronize()
    assert buf.cpu().numpy().tobytes() == ref.tobytes()
    after, _ = _draw(dctx, w, h)
    assert after.tobytes() != ref.tobytes()


def test_nothing_is_uploaded(dctx):
    w, h = 64, 36
    s, m, c, em = scenes.reference_scene(w, h)
    dctx.set_scene(s, m, c, em)
    first = dctx.last_scene_upload_bytes()
    for n in (1, 37, 256, 10):
        dctx.set_option("max_depth", n)
        assert dctx.last_scene_upload_bytes() == first
        _draw(dctx, w, h)
        dctx.set_scene(s, m, c, em)                          # the resident bytes: nothing to copy
        assert dctx.last_scene_upload_bytes() == 0


def test_aovs_do_not_change(dctx):
    w, h = 64, 36
    s, m, c, em = scenes.reference_scene(w, h)
    dctx.set_scene(s, m, c, em)
    rays = scenes.camera_rays(c, w, h, seed=1)

    def aovs():
        (a, nn, i), r = dctx.trace_aovs(rays)
        alb, nm, ii = (torch.zeros((h, w, 4), device="cuda"), torch.zeros((h, w, 4), device="cuda"),
                       torch.zeros((h, w), dtype=torch.int32, device="cuda"))
        r2 = dctx.draw_aovs(0, 2, w, h, alb, nm, ii)
        return [np.asarray(x).tobytes() for x in (a, nn, i, alb.cpu(), nm.cpu(), ii.cpu())] + [r, r2]

    ref = aovs()
    for n in (1, 200):
        dctx.set_option("max_depth", n)
        assert aovs() == ref


def test_combines_with_media_textures_and_sampling(dctx):
    w, h = 160, 90
    s, m, c, em = scenes.reference_scene(w, h)
    dctx.set_scene(s, m, c, em)
    dctx.set_environment(np.random.default_rng(6).uniform(0.0, 1.5, (16, 32, 3)).astype(np.float32))
    dctx.set_option("environment_sampling", 1)
    dctx.set_textures(_const_layers(0.8), np.zeros(len(s), np.int32))
    layers = np.zeros(len(s), np.int32) - 1
    layers[em] = 0
    dctx.set_emission_textures(_const_layers(1.0), layers)
    dctx.set_option("emission_texture_sampling", 1)
    dctx.set_media(gm._media(len(s), {GLASS46: (0.1, 0.2, 0.3, 4.0, 0.6)}))
    rays = scenes.camera_rays(c, w, h, seed=2)
    (_a, _n, ids), _ = dctx.trace_aovs(rays)
    glass = ids == GLASS46
    assert glass.sum() >= 50
    means, counts = {}, {}
    for n in (10, 64):
        dctx.set_option("max_depth", n)
        img, r = _draw(dctx, w, h, spp=8)
        assert np.isfinite(img).all() and all(k.startswith(TEX_KERNELS) for k in _kinds(dctx))
        acc = np.zeros((len(rays), 3))
        for f in range(8):
            out, _ = dctx.trace_rays(rays[glass], spp=16, frame=f)
            acc[glass] += out[:, :3]
        means[n] = acc[glass].mean(0) / 8
        counts[n] = r
    # the dense medium in the glass sphere gives back what the cap at 10 took
    assert (means[64] > means[10]).all(), means
    assert counts[64] > counts[10]
