"""Every fast kernel instance against the sample replay of tests/sample_replay.py: Lambert, rough-metal and glass vertices
and light-sampled shadow rays, sample by sample. Caller rays (trace_rays at spp 1 under every fast_kform, light sampling
on and off, the sky, mitsuba_compare and a lat-long map; launches long enough for the 8-CTA instances; trace_samples
lists for exact per-sample ray counts), surface points (trace_irradiance, trace_samples(points=True), with and without
ids), and draws of a lens camera in every fast variant (spp 1; progressive draws with spp 2, two frames and a weighted
prev, variant 0's carried stream included; draw_samples lists). Every well-conditioned sample's value must lie within the
replay's tolerance, and ray counts must equal the replay's over count-certain samples plus what a list call over the
rest reports (exactly where the list call sweeps like the draw, bounded below elsewhere). Through
Context.last_kernels() the module asserts which instance ran, and the union must equal the fast (k_fast_*) part of
mirror_chain.COVERAGE that the mirror chains drive. Every replayed batch must also hold a minimum share of
well-conditioned samples (WELL_MIN), so that no check passes on an empty selection."""
import numpy as np
import pytest
import torch

import furnace as F
import mirror_chain as mc
import sample_replay as sr
import test_sweep_oracle as so
from test_gpu_mirror_chains import LONG_SLABS_PER_WARP, SLAB_PIX, image_instances, queue_instance, ran

pytestmark = pytest.mark.gpu

FAST_DRIVEN = {k for k, v in mc.COVERAGE.items() if not v.startswith("excluded") and k.startswith("k_fast_")}
# scene key -> (sphere count, layout, lights, caller rays replayed). c700: past 36 KB of staged arrays, so the 768-thread
# instances run for every form the gate allows; s400: fails the gate and takes form 3 at 768 threads; L1000: 300 lights,
# a blob past 64 KB with at most 1024 spheres (the group queue's kform 2 and its unstaged-material instances).
SCENES = {"c40": (40, "compact", 4, 1500), "s40": (40, "spread", 4, 1500), "c120": (120, "compact", 6, 600),
          "c700": (700, "compact", 6, 120), "s400": (400, "spread", 6, 300), "L1000": (1000, "compact", 300, 48)}
SMALL_SCENE = 120                    # scenes up to this size fit the 128-thread CTAs: the 8-CTA (long launch) instances
# The least share of well-conditioned samples in any replayed batch of a scene: half of the least share the replay
# decides over the module's batches of that scene (c40 0.198, s40 0.204, c120 0.148, c700 0.078, s400 0.240). The
# 300-light scene has its own floors in counts (L1000_MIN, measured 2 of 54 caller rays with light sampling, 7 without,
# 9 of 48 draw pixels without).
WELL_MIN = {"c40": 0.1, "s40": 0.1, "c120": 0.07, "c700": 0.035, "s400": 0.12}
L1000_MIN = {"rays1": 2, "rays0": 4, "draw0": 4}
MAP = np.random.default_rng(3).uniform(0.05, 1.5, (16, 32, 3)).astype(np.float32)


@pytest.fixture(scope="module")
def scenes():
    cache = {}

    def get(key):
        if key not in cache:
            count, layout, nl, nr = SCENES[key]
            s, m, em = sr.mixed_corridor(count, layout, n_lights=nl)
            rays = np.concatenate([sr.candidate_rays(s, nr, seed=count + nl), sr.inside_glass_rays(s, m, nr // 8, seed=count)])
            cache[key] = (s, m, em, rays)
        return cache[key]
    return get


@pytest.fixture(scope="module")
def seen():
    return set()


@pytest.fixture
def rctx(gpu_ctx):
    yield gpu_ctx
    gpu_ctx.set_environment(None)
    for k, v in (("fast_kform", 2), ("mitsuba_compare", 0), ("light_sampling", 1), ("fast_variant", -1)):
        gpu_ctx.set_option(k, v)
    gpu_ctx.set_spp(4)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def check(got, res, sel, scale=1.0, extra=0.0, what=""):
    """got [n, >= 3] against scale x the replay's values on the samples `sel`; a failure lists each bad sample's path."""
    v, tol = res["v"] * scale, res["tol"] * scale + 4 * 2.0 ** -23 * np.abs(res["v"] * scale).max(1) + extra
    err = np.abs(got[:, :3] - v).max(1)
    bad = np.nonzero(sel & ~(err <= tol))[0]
    assert not len(bad), "\n".join([f"{what}: {len(bad)} of {int(sel.sum())} well samples off"] + [
        f"  {sr.describe(res, i)}: gpu {got[i, :3]}, replay {v[i]}, |err| {err[i]:.3g} > tol {tol[i]:.3g}" for i in bad[:8]])


def _floor(res, key, what, n_min=None):
    """A replayed batch holds its scene's least share of well-conditioned samples (or n_min of them)."""
    k = int(res["well"].sum())
    want = n_min if n_min is not None else int(np.ceil(WELL_MIN[key] * len(res["well"])))
    assert k >= want, f"{key} {what}: {k} of {len(res['well'])} samples well conditioned, want >= {want}"


def _kq(kopt):
    """fast_kform 4 runs what 2 runs (form 4 where <= 64 padded spheres fit the kernel parameter), but with the FP32
    pass 1 instead of the half-precision one: the instance names the pick rules give for 2."""
    return 2 if kopt == 4 else kopt


def _set(ctx, s, m, em, kopt, ls, sky, cam=None):
    ctx.set_option("fast_kform", kopt)
    ctx.set_option("light_sampling", ls)
    ctx.set_option("mitsuba_compare", int(sky == "mitsuba"))
    ctx.set_scene(s, m, sr.lens_camera() if cam is None else cam, em)
    ctx.set_environment(MAP if sky == "env" else None)
    return sr.Scene(s, m, em, mitsuba=sky == "mitsuba", env=MAP if sky == "env" else None, ls=bool(ls))


def _counts(ctx, inputs, res, frame, spp=1, points=False, ids=None):
    """trace_samples over the well samples (their rays are certain: exactly the replay's) and over the rest."""
    well = np.nonzero(res["well"])[0].astype(np.int32)
    rest = np.nonzero(~res["well"])[0].astype(np.int32)
    _, n_well = ctx.trace_samples(inputs, ids=ids, points=points, entries=torch.from_numpy(well).cuda(), spp=spp, frame=frame)
    assert n_well == int(res["rays"][well].sum()), (n_well, int(res["rays"][well].sum()))
    n_rest = 0
    if len(rest):
        _, n_rest = ctx.trace_samples(inputs, ids=ids, points=points, entries=torch.from_numpy(rest).cuda(), spp=spp,
                                      frame=frame)
    return n_well + n_rest


# ---- 1. caller rays ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key", list(SCENES))
def test_caller_rays(rctx, scenes, seen, key):
    """trace_rays at spp 1 under every fast_kform, light sampling on and off, with the sky, mitsuba_compare and a map:
    well-conditioned samples within tolerance, ray counts exact (trace_samples lists with squares); then a launch of
    >= 48 slabs per warp (the 8-CTA instances) checked on a subset of its rays."""
    s, m, em, rays = scenes(key)
    n = len(s)
    gate = so.gate_passes(s)
    dev = torch.from_numpy(rays).cuda()
    combos = [(k, ls, "sky") for k in (0, 1, 2, 3) for ls in (1, 0)] + [(2, 1, "mitsuba"), (2, 0, "env"), (3, 1, "env")]
    if n <= 64:
        combos += [(4, 1, "sky"), (4, 0, "sky")]              # form 4 with its FP32 pass 1
    if key in ("c700", "s400"):
        combos = combos[:8]
    if key == "L1000":
        combos = [(2, 1, "sky"), (2, 0, "sky")]
    for frame, (kopt, ls, sky) in enumerate(combos):
        sc = _set(rctx, s, m, em, kopt, ls, sky)
        res = sr.replay(sc, sr.ray_seeds(np.arange(len(rays)), 1, 0, frame), rays=rays)
        _floor(res, key, f"caller rays kform {kopt} ls {ls} {sky}", L1000_MIN[f"rays{ls}"] if key == "L1000" else None)
        out, traced = rctx.trace_rays(dev, spp=1, frame=frame)
        ran(rctx, queue_instance("rays", n, len(em), _kq(kopt), gate and kopt != 0, ls), seen)
        out = out.cpu().numpy()
        check(out, res, res["well"], what=f"{key} kform {kopt} ls {ls} {sky}")
        assert (out[:, 3] == 0).all()
        assert traced == _counts(rctx, dev, res, frame), (key, kopt, ls, sky)
        if sky == "sky" and kopt in (0, 2, 4):
            # squares: a sample's v and v^2 through trace_samples
            idx = np.nonzero(res["well"])[0][:200]
            s4 = torch.zeros((len(idx), 4), device="cuda")
            q4 = torch.zeros((len(idx), 4), device="cuda")
            (s4, q4), _ = rctx.trace_samples(dev, entries=torch.from_numpy(idx.astype(np.int32)).cuda(), spp=1,
                                             frame=frame, sum4=s4, sq4=q4)
            sub = {k: (v[idx] if not isinstance(v, dict) else {a: b[idx] for a, b in v.items()}) for k, v in res.items()}
            g = s4.cpu().numpy()
            check(g, sub, np.ones(len(idx), bool), what=f"{key} trace_samples sums")
            assert (g[:, 3] == 1).all()
            g2 = q4.cpu().numpy()[:, :3]
            v = sub["v"]
            assert (np.abs(g2 - v * v).max(1) <= 2.01 * np.abs(v).max(1) * sub["tol"] + 2.0 ** -21 * (v * v).max(1) + 1e-9).all()
        if n <= SMALL_SCENE and sky == "sky":
            # >= 48 slabs of 64 rays per warp on every SM; a random subset of the tiled rays is replayed
            rep = -(-LONG_SLABS_PER_WARP * _sms() * 32 * SLAB_PIX // len(rays)) + 1
            big = np.tile(rays, (rep, 1))
            out, _ = rctx.trace_rays(torch.from_numpy(big).cuda(), spp=1, frame=frame + 50)
            ran(rctx, queue_instance("rays", n, len(em), _kq(kopt), gate and kopt != 0, ls, long=True), seen)
            pick = np.random.default_rng(frame).choice(len(big), 1200, replace=False)
            r2 = sr.replay(sc, sr.ray_seeds(pick, 1, 0, frame + 50), rays=big[pick])
            _floor(r2, key, f"long launch kform {kopt} ls {ls}")
            check(out.cpu().numpy()[pick], r2, r2["well"], what=f"{key} kform {kopt} ls {ls} long")


# ---- 2. points -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key", ["c40", "c120", "c700", "s400"])
def test_points(rctx, scenes, seen, key):
    """trace_irradiance (pi x the sample) and trace_samples(points=True), with ids and without (points off the lights)."""
    s, m, em, _ = scenes(key)
    n = len(s)
    gate = so.gate_passes(s)
    for with_ids in (True, False):
        pts, self_ = sr.surface_points(s, m, em, 600 if n < 500 else 200, seed=n + with_ids, with_ids=with_ids)
        ids = self_ if with_ids else None
        dev = torch.from_numpy(pts).cuda()
        dids = torch.from_numpy(ids).cuda() if with_ids else None
        for frame, (kopt, ls) in enumerate([(2, 1), (0, 1), (3, 0)]):
            sc = _set(rctx, s, m, em, kopt, ls, "sky")
            res = sr.replay(sc, sr.ray_seeds(np.arange(len(pts)), 1, 0, frame), points=pts, point_ids=ids, point_self=self_)
            _floor(res, key, f"points ids {with_ids} kform {kopt} ls {ls}")
            out, traced = rctx.trace_irradiance(dev, ids=dids, spp=1, frame=frame)
            ran(rctx, queue_instance("rays", n, len(em), kopt, gate and kopt != 0, ls), seen)
            check(out.cpu().numpy(), res, res["well"], scale=sr.PI32, what=f"{key} irradiance ids {with_ids} kform {kopt}")
            assert traced == _counts(rctx, dev, res, frame, points=True, ids=dids)
            s4 = torch.zeros((len(pts), 4), device="cuda")
            (s4, _), _ = rctx.trace_samples(dev, ids=dids, points=True, spp=1, frame=frame, sum4=s4)
            g = s4.cpu().numpy()
            check(g, res, res["well"], scale=sr.PI32, what=f"{key} trace_samples points ids {with_ids}")
            assert (g[:, 3] == 1).all()


# ---- 3. draws ------------------------------------------------------------------------------------------------------
W, H = 40, 24
SMALL = {"c700": (12, 8), "s400": (16, 12), "L1000": (8, 6)}        # slow replays: smaller images
# Only the slab queue (variants 3 and 9) sweeps with draw_samples' arithmetic, so only there does a list call over the
# ill-conditioned pixels trace exactly the draw's paths; elsewhere those pixels may take other paths (that is what ill
# conditioned means), and the count is only bounded below by one ray per sample.
SAME_SWEEP = (3, 9)


def _pixels(w, h):
    y, x = np.divmod(np.arange(w * h), w)
    return x, y


@pytest.mark.parametrize("key", ["c40", "s40", "c120", "c700", "s400", "L1000"])
def test_draws(rctx, scenes, seen, key):
    """A lens camera at spp 1, one frame, in every fast variant x the sweep forms each allows (fast_kform 4, the FP32
    pass 1, for the slab queue's variants 3 and 9): every well pixel is its one sample; the ray count is the replay's over
    well pixels plus draw_samples' over the rest. The 300-light scene draws with variant 8 only (the group queue past
    64 KB of blob, kform 0 - 2)."""
    s, m, em, _ = scenes(key)
    n = len(s)
    gate = so.gate_passes(s)
    W, H = SMALL.get(key, (40, 24))
    x, y = _pixels(W, H)
    rctx.set_spp(1)
    cache = {}
    for v in ((8,) if key == "L1000" else range(10)):
        kopts = (0, 1, 2, 3, 4) if v in (3, 9) else ((0, 1, 2, 3) if v in (4, 5, 8) else (2,))
        for kopt in kopts:
            for ls in ((1, 0) if v in (3, 4, 8, 9) or kopt == 2 else (1,)):
                frame = 7
                sc = _set(rctx, s, m, em, kopt, ls, "sky")
                if key == "L1000" and ls:
                    # With 300 lights every Lambert vertex traces 299 shadow rays and the replay decides no camera path
                    # that meets one (0 of 48 pixels, after 55 s of replay): the draw is checked for its instance and
                    # its ray count's lower bound only; the instance's sweep and shading are the light-free draw's.
                    rctx.set_option("fast_variant", v)
                    total = rctx.draw(frame, 1, W, H, torch.zeros((H, W, 4), device="cuda"), flags=0, mode=1)
                    ran(rctx, image_instances("fast", v, n, len(em), kopt, gate and kopt != 0, ls), seen)
                    assert total >= W * H
                    continue
                if ls not in cache:
                    cache[ls] = sr.replay(sc, sr.draw_seeds(x, y, W, 1, 0, frame), camera=(sr.lens_camera(), W, H, x, y))
                    _floor(cache[ls], key, f"draw ls {ls}", L1000_MIN["draw0"] if key == "L1000" else None)
                res = cache[ls]
                rctx.set_option("fast_variant", v)
                buf = torch.zeros((H, W, 4), device="cuda")
                total = rctx.draw(frame, 1, W, H, buf, flags=0, mode=1)
                want = image_instances("fast", v, n, len(em), _kq(kopt), gate and kopt != 0, ls)
                got = rctx.last_kernels()
                seen.update(got)
                assert got == [want], (v, kopt, ls, got, want)
                img = buf.cpu().numpy().reshape(-1, 4)
                check(img, res, res["well"], what=f"{key} variant {v} kform {kopt} ls {ls}")
                rest = np.nonzero(~res["well"])[0].astype(np.int32)
                n_well = int(res["rays"][res["well"]].sum())
                if v in SAME_SWEEP:
                    _, n_rest = rctx.draw_samples(frame, W, H, torch.from_numpy(rest).cuda(), 1) if len(rest) else (None, 0)
                    assert total == n_well + n_rest, (key, v, kopt, ls, total, n_well, n_rest)
                else:
                    assert total >= n_well + len(rest), (key, v, kopt, ls, total, n_well, len(rest))


@pytest.mark.parametrize("key", ["c40"])
def test_progressive_draws(rctx, scenes, seen, key):
    """spp 2, two frames, a weighted prev: pixel = prev W + sum_f w_f mean_s v; variant 0 carries one stream per pixel
    and frame across its samples, the others seed every sample."""
    s, m, em, _ = scenes(key)
    x, y = _pixels(W, H)
    spp, f0, nf, flags = 2, 3, 2, 2
    Wp, w = F.frame_weights(f0, nf, flags)
    prev = np.random.default_rng(1).uniform(0, 1, (H, W, 4)).astype(np.float32)
    rctx.set_spp(spp)
    for v in (0, 1, 3, 6, 8, 9):
        sc = _set(rctx, s, m, em, 2, 1, "sky")
        rctx.set_option("fast_variant", v)
        acc, tol, well, rays = np.zeros((W * H, 3)), np.zeros(W * H), np.ones(W * H, bool), np.zeros(W * H, int)
        for fi in range(nf):
            state = sr.mega_seed(x, y, W, f0 + fi)
            for smp in range(spp):
                st = state if v == 0 else sr.draw_seeds(x, y, W, spp, smp, f0 + fi)
                r = sr.replay(sc, st, camera=(sr.lens_camera(), W, H, x, y))
                state = r["state"]
                acc += w[fi] / spp * r["v"]
                tol += w[fi] / spp * r["tol"]
                well &= r["well"]
                rays += r["rays"]
        buf = torch.from_numpy(prev.copy()).cuda()
        total = rctx.draw(f0, nf, W, H, buf, flags=flags, mode=1)
        seen.update(rctx.last_kernels())
        got = buf.cpu().numpy().reshape(-1, 4)
        exp = prev.reshape(-1, 4)[:, :3].astype(np.float64) * Wp + acc
        err = np.abs(got[:, :3] - exp).max(1)
        lim = tol + 2.0 ** -21 * np.abs(exp).max(1) + 1e-7
        bad = np.nonzero(well & (err > lim))[0]
        assert not len(bad), (key, v, bad[:5], err[bad[:5]], lim[bad[:5]])
        assert well.mean() >= WELL_MIN[key] / 2, (key, v, well.mean())
        if v in SAME_SWEEP:
            rest = np.nonzero(~well)[0].astype(np.int32)
            n_rest = 0
            for fi in range(nf):
                if len(rest):
                    _, k = rctx.draw_samples(f0 + fi, W, H, torch.from_numpy(rest).cuda(), spp)
                    n_rest += k
            assert total == int(rays[well].sum()) + n_rest, (key, v)


@pytest.mark.parametrize("key", ["c40", "s40", "c120", "c700", "s400"])
def test_pixel_lists(rctx, scenes, seen, key):
    """draw_samples: a pixel list (spp 1) under every fast_kform, light sampling on and off, with and without squares;
    sums equal the replay's samples, counts 1, exact ray counts for well pixels; and a whole image long enough for the
    8-CTA instances, checked on a subset."""
    s, m, em, _ = scenes(key)
    n = len(s)
    gate = so.gate_passes(s)
    W, H = SMALL.get(key, (40, 24))
    x, y = _pixels(W, H)
    for kopt in (0, 1, 2, 3):
        for ls in (1, 0):
            sc = _set(rctx, s, m, em, kopt, ls, "sky")
            frame = 11 + kopt
            res = sr.replay(sc, sr.draw_seeds(x, y, W, 1, 0, frame), camera=(sr.lens_camera(), W, H, x, y))
            _floor(res, key, f"pixel list kform {kopt} ls {ls}")
            well = np.nonzero(res["well"])[0].astype(np.int32)
            for moments in (False, True):
                s4 = torch.zeros((len(well), 4), device="cuda")
                q4 = torch.zeros((len(well), 4), device="cuda") if moments else None
                (s4, q4), traced = rctx.draw_samples(frame, W, H, torch.from_numpy(well).cuda(), 1, s4, q4)
                ran(rctx, queue_instance("samples", n, len(em), kopt, gate and kopt != 0, ls, moments=moments), seen)
                sub = {k: (v[well] if not isinstance(v, dict) else {a: b[well] for a, b in v.items()}) for k, v in res.items()}
                check(s4.cpu().numpy(), sub, np.ones(len(well), bool), what=f"{key} list kform {kopt} ls {ls}")
                assert (s4.cpu().numpy()[:, 3] == 1).all()
                assert traced == int(sub["rays"].sum())
            if n <= SMALL_SCENE and kopt >= 2 and gate:
                WW = 512
                HH = -(-LONG_SLABS_PER_WARP * _sms() * 32 * SLAB_PIX // WW) + 1
                pick = np.random.default_rng(kopt).choice(WW * HH, 800, replace=False)
                py, px = np.divmod(pick, WW)
                r2 = sr.replay(sc, sr.draw_seeds(px, py, WW, 1, 0, frame), camera=(sr.lens_camera(), WW, HH, px, py))
                _floor(r2, key, f"long list kform {kopt} ls {ls}")
                for moments in (False, True):
                    s4 = torch.zeros((WW * HH, 4), device="cuda")
                    q4 = torch.zeros((WW * HH, 4), device="cuda") if moments else None
                    (s4, _), _ = rctx.draw_samples(frame, WW, HH, None, 1, s4, q4)
                    ran(rctx, queue_instance("samples", n, len(em), kopt, True, ls, long=True, moments=moments), seen)
                    check(s4.cpu().numpy()[pick], r2, r2["well"], what=f"{key} long list kform {kopt} ls {ls}")


# ---- 4. coverage ---------------------------------------------------------------------------------------------------
def test_coverage_is_complete(request, seen):
    """The union of the instances the module launched equals the fast part of the mirror chains' driven table. Only
    complete when every test of the module ran before this one; otherwise skipped."""
    mine = [it for it in request.session.items if getattr(it, "module", None) is request.module]
    total = sum(len(f.pytestmark[0].args[1]) for f in (test_caller_rays, test_points, test_draws, test_progressive_draws,
                                                       test_pixel_lists)) + 1
    if len(mine) != total or mine[-1] is not request.node:
        pytest.skip(f"needs all {total} tests of the module, this one last ({len(mine)} selected)")
    missing = sorted(FAST_DRIVEN - seen)
    extra = sorted(k for k in seen - FAST_DRIVEN)
    assert not missing and not extra, (missing, extra)
