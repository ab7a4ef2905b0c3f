"""The fast kernels' sphere sweeps (tpt_debug_hit, forms 0-3 of tpt_fast.cu's prepare_sweep) against the float64
nearest-hit oracle of test_sweep_oracle.py, at every padded sphere count mod 64, around the group kernels' 1024-sphere
limit, past the 64 KB all-staged blob and up to the largest scene tpt_debug_hit can stage; then the production kernels
end to end at one count per tail class, against exact mode (statistically) and exact mode against the CPU restatement
(bit for bit)."""
import numpy as np
import pytest

from conftest import bits_differ, rel_l2
from test_gpu_fast import surface_rays
from test_sweep_oracle import (T_MAX, aimed_rays, degenerate_rays, gate_passes, make_scene, near_tangent_rays,
                               nearest_hit, pad_aimed_rays, pad_possible, tmin_rays)

pytestmark = pytest.mark.gpu

TAILS = list(range(4, 65, 4))                                         # padded count mod 64: 4, 8, ..., 60, 0
BELOW = [p - (i % 4) for i, p in enumerate(TAILS)]                    # 4 .. 64, some padded
ABOVE = [64 * (1 + i % 4) + p - (i % 3) for i, p in enumerate(TAILS)]  # the same classes after 1-4 full chunks
SWEEP_COUNTS = [1, 2, 3] + BELOW + ABOVE + [1023, 1024, 1025, 1028, 1536, 2048]
FORMS = {"compact": (0, 1, 2), "spread": (0, 3)}


def _simd(count):
    return (count + 3) // 4 * 4


def _geom_bytes(count, n_lights):
    """Spheres + inverse radii + light table (tpt_scene_pack.h scene_blob_layout); tpt_set_scene refuses > 200 KB."""
    a16 = lambda x: (x + 15) // 16 * 16
    simd = _simd(count)
    return a16(simd * 16) + a16(simd * 4) + a16(max(n_lights, 1) * 32)


def _debug_hit_smem(count, n_lights, kform):
    """Dynamic shared memory launch_debug_hit asks for (tpt_scene_pack.h scene_blob_layout + fast_smem)."""
    a16 = lambda x: (x + 15) // 16 * 16
    simd = _simd(count)
    geom = _geom_bytes(count, n_lights)
    total = geom + 2 * a16((count + 1) * 16) + a16((count + 1) * 4)
    staged = total if total <= 64 * 1024 else geom
    return (staged + 127) // 128 * 128 + (simd * 16 if kform >= 2 else 0)


def max_debug_count(kform, n_lights):
    c = 4
    while _debug_hit_smem(c + 4, n_lights, kform) <= 200 * 1024 and _geom_bytes(c + 4, n_lights) <= 200 * 1024:
        c += 4
    return c


def _lights(mats):
    return int((mats["emissive"] > 0).any(axis=1).sum())


def check_sweeps(ctx, sph, dup, forms, seed, tag, min_frac=0.9, min_aimed=1.0):
    """All assertions of one scene through tpt_debug_hit. Returns the well-conditioned fraction of the surface rays."""
    count = len(sph)
    simd = _simd(count)
    n = int(np.clip(300_000 / count, 64, 3000))
    surf = surface_rays(sph, 4 * n, seed)
    sets = {"surface": surf[np.isfinite(surf).all(1)],
            "tangent": near_tangent_rays(sph, n, seed + 1)[0],
            "tmin": tmin_rays(sph, n, seed + 2)[0],
            "degenerate": degenerate_rays(sph, seed + 3),
            "pad": pad_aimed_rays(max(16, n // 4), seed + 4)}
    aimed, target = aimed_rays(sph, seed + 5)
    sets["aimed"] = aimed
    if dup >= 0:
        # many rays at the duplicate pair from all sides: the pair's position in the candidate list (and so whether the two
        # land in one trip of a two-candidates-per-trip pass 2) varies from ray to ray
        rng = np.random.default_rng(seed + 6)
        c = sph["center"][dup].astype(np.float64); r = float(sph["radius"][dup])
        nrm = rng.normal(size=(256, 3)); nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
        o = c + nrm * (r + rng.uniform(0.01, 0.3, (256, 1)))
        d = -nrm + rng.normal(size=(256, 3)) * 0.3 * r
        d /= np.linalg.norm(d, axis=1, keepdims=True)
        sets["dup"] = np.concatenate([o, d], 1).astype(np.float32)
    frac = None
    for name, rays in sets.items():
        res = {k: ctx.debug_hit(k, rays) for k in forms}
        for k, (ids, t) in res.items():
            assert (ids >= -1).all() and (ids < simd).all(), (tag, name, k)
            pad = ids >= count
            if k != 0 or name != "pad":
                assert not pad.any(), (tag, name, k, np.unique(ids[pad]))
            else:
                assert pad_possible(rays[pad], count).all(), (tag, name)
            if dup >= 0:
                assert not (ids == dup + 1).any(), (tag, name, k, "the higher id of an exact duplicate pair won")
        if 0 in res and 3 in res:
            # form 0 sweeps the padding like the reference (DESIGN.md 1.1); form 3's pass 1 never makes a pad a candidate
            # (-1e30), so where form 0 met the padding point form 3 answers with the real spheres alone
            real = res[0][0] < count
            assert (res[3][0] == res[0][0])[real].all() and \
                (res[3][1].view(np.uint32) == res[0][1].view(np.uint32))[real].all(), \
                (tag, name, "form 3 != form 0", int((res[3][0] != res[0][0])[real].sum()))
        if 1 in res and 2 in res:
            assert (res[2][0] == res[1][0]).all() and (res[2][1].view(np.uint32) == res[1][1].view(np.uint32)).all(), \
                (tag, name, "form 2 != form 1", int((res[2][0] != res[1][0]).sum()))
        if name == "aimed":
            for k, (ids, t) in res.items():
                assert (ids == target).all(), (tag, k, "aimed", target[ids != target][:8], ids[ids != target][:8])
            if count > 2048:
                continue                 # the geometric construction alone decides these; spare the oracle 10^8 pairs
        if name == "dup":
            continue
        ora = nearest_hit(rays, sph)
        well = ora["well"]
        for k, (ids, t) in res.items():
            w = well.copy()
            if k == 0 and name == "pad":
                w &= ~((ora["id"] == -1) & (ids >= count))          # form 0 may meet the padding point behind everything
            bad = w & (ids != ora["id"])
            assert not bad.any(), (tag, name, k, int(bad.sum()), ids[bad][:8], ora["id"][bad][:8])
            hit = w & (ids >= 0)
            tt = t.astype(np.float64)
            assert ((tt[hit] >= ora["tlo"][hit]) & (tt[hit] <= ora["thi"][hit])).all(), (tag, name, k)
            assert (t[w & (ids < 0)] == np.float32(T_MAX)).all()
        if name == "surface":
            frac = float(well.mean())
    print(f"{tag}: well-conditioned {frac:.4f} of {len(sets['surface'])} surface/camera rays")
    assert frac >= min_frac, (tag, frac)
    # every real sphere (the higher id of the duplicate pair stands for the lower) is hit by its aimed ray
    expect = set(range(count)) - ({dup + 1} if dup >= 0 else set())
    assert set(target) <= expect and len(set(target)) >= min_aimed * len(expect), (tag, sorted(expect - set(target))[:8])
    return frac


@pytest.mark.parametrize("layout", ["compact", "spread"])
@pytest.mark.parametrize("count", SWEEP_COUNTS)
def test_sweep_forms_against_oracle(gpu_ctx, count, layout):
    sph, mats, cam, dup = make_scene(count, layout)
    assert gate_passes(sph) == (layout == "compact")
    gpu_ctx.set_scene(sph, mats, cam, None)
    check_sweeps(gpu_ctx, sph, dup, FORMS[layout], 100 + count, f"{layout}{count}")


@pytest.mark.parametrize("layout", ["compact", "spread"])
def test_sweep_forms_at_the_staging_limit(gpu_ctx, layout):
    """The largest scene tpt_debug_hit stages for each form, and one sphere more: that must fail with an error, never
    sweep a truncated array (launch_debug_hit refuses more than 200 KB of shared memory; past 200 KB of geometry
    tpt_set_scene already refuses the scene)."""
    import toypathtracer_b200 as tpt
    forms = FORMS[layout]
    limits = sorted({max_debug_count(k, 4) for k in forms})
    for cap in limits:
        sph, mats, cam, dup = make_scene(cap, layout, seed=1)
        assert _lights(mats) == 4
        gpu_ctx.set_scene(sph, mats, cam, None)
        ok = tuple(k for k in forms if max_debug_count(k, 4) >= cap)
        # 5 680 / 10 232 spheres inside the gate's |s| <= 11 ball are packed densely: more rays start on a sphere and
        # graze its neighbours, and a few spheres lie wholly inside the union of others (no origin outside them is free)
        check_sweeps(gpu_ctx, sph, dup, ok, 7 + cap, f"{layout}{cap}", min_frac=0.8, min_aimed=0.995)
        sph, mats, cam, dup = make_scene(cap + 1, layout, seed=1)
        if _geom_bytes(cap + 1, _lights(mats)) > 200 * 1024:
            with pytest.raises(tpt.TptError, match="too many spheres"):      # refused before any kernel sees it
                gpu_ctx.set_scene(sph, mats, cam, None)
            continue
        gpu_ctx.set_scene(sph, mats, cam, None)
        ray = np.array([[0, 6, 14, 0, 0, -1]], np.float32)
        for k in forms:
            if max_debug_count(k, _lights(mats)) < cap + 1:
                with pytest.raises(tpt.TptError):
                    gpu_ctx.debug_hit(k, ray)


# ---- end to end ------------------------------------------------------------------------------------------------------
E2E = [(c, lay) for c in ABOVE for lay in ("compact", "spread")] + [(1025, "compact"), (2048, "compact"), (4600, "spread")]
W, H = 192, 108


@pytest.mark.parametrize("count,layout", E2E)
def test_production_kernels_end_to_end(gpu_ctx, oracle, libs, count, layout):
    """Fast variants 3, 8, 5 and 7 (automatic sweep form) against exact mode, and the reference-GPU mode's native
    instance against its strict twin, with the bars of test_gpu_fast.test_statistical_parity (the ray-count bar scaled to
    this image's sample count); then exact mode bit for bit against the CPU restatement."""
    sph, mats, cam, dup = make_scene(count, layout)
    gpu_ctx.set_scene(sph, mats, cam, None)
    try:
        gpu_ctx.set_option("exact_lanes", 0)
        samples = W * H * 64
        ray_tol = 2e-3 * np.sqrt(640 * 360 / (W * H))

        def pair(mode):
            a = np.zeros((H, W, 4), np.float32); b = np.zeros((H, W, 4), np.float32)
            ra = gpu_ctx.draw(0, 16, W, H, a, flags=2, mode=mode)
            rb = gpu_ctx.draw(16, 16, W, H, b, flags=2, mode=mode)
            return a, ra, b, rb

        def parity(img, rays, ref, what):
            a, ra, b, rb = ref
            floor = rel_l2(b, a)
            assert np.isfinite(img).all(), what
            r = rel_l2(img, a)
            assert r < 1.25 * floor, (what, r, floor)
            assert abs(rays / ra - 1) < ray_tol, (what, rays / samples, ra / samples)
            ma, mb, mi = (x[..., :3].reshape(-1, 3).astype(np.float64).mean(0) for x in (a, b, img))
            assert (np.abs(mi - ma) < 3 * np.abs(ma - mb) + 2e-3 * ma).all(), (what, mi, ma)

        exact = pair(libs.MODE_EXACT)
        for variant in (3, 8, 5, 7):
            gpu_ctx.set_option("fast_variant", variant)
            img = np.zeros((H, W, 4), np.float32)
            rays = gpu_ctx.draw(0, 16, W, H, img, flags=2, mode=libs.MODE_FAST)
            parity(img, rays, exact, f"{layout}{count} variant {variant}")
        strict = pair(libs.MODE_REFGPU)
        img = np.zeros((H, W, 4), np.float32)
        rays = gpu_ctx.draw(0, 16, W, H, img, flags=2, mode=libs.MODE_REFGPU_FAST)
        parity(img, rays, strict, f"{layout}{count} refgpu fast")
        # exact mode: bit for bit the CPU restatement, every lane layout
        w, h = 64, 36
        obuf, orays, pads = oracle.orc_render(sph, mats, cam, w, h, 0, 2, flags=2)
        for lanes in (32, 8, 1, 65):
            gpu_ctx.set_option("exact_lanes", lanes)
            buf = np.zeros((h, w, 4), np.float32)
            total, pf = gpu_ctx.draw(0, 2, w, h, buf, flags=2, mode=libs.MODE_EXACT, per_frame=True)
            assert pf == orays, (layout, count, lanes)
            assert not bits_differ(buf, obuf, pads).any(), (layout, count, lanes)
    finally:
        gpu_ctx.set_option("exact_lanes", 0)
        gpu_ctx.set_option("fast_variant", 3)
