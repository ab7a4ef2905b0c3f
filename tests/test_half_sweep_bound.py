"""Sweep form 5's half-precision pass 1 on the CPU (toypathtracer_b200/half_sweep.py, the model of FastHitterKH's pass
in csrc/tpt_fast.cu and of build_half_pairs in csrc/tpt_scene_pack.h): the binary16 emulation is exact, the observed
error of xu and xv stays within the derived bound E, and for every ray inside the bound's premises the candidate set
contains every sphere form 4's FP32 pass 1 and an exact float64 intersection accept. No GPU needed."""
from fractions import Fraction

import numpy as np
import pytest

import test_sweep_oracle as so
from toypathtracer_b200 import half_sweep as hs
from toypathtracer_b200 import scenes


def _scene(spheres):
    raw = np.asarray(spheres).view(np.float32).reshape(-1, 5)
    pad = (len(raw) + 3) // 4 * 4 - len(raw)
    c = np.concatenate([raw[:, :3], np.full((pad, 3), 10000, np.float32)])
    r2 = np.concatenate([(raw[:, 3] * raw[:, 3]).astype(np.float32), np.zeros(pad, np.float32)])
    return c, r2, np.arange(len(c)) < len(raw)


def _unit(v):
    return v / np.linalg.norm(v, axis=1, keepdims=True)


def _bench_rays(n, seed=3):
    sp, _, cam, _ = scenes.reference_scene(1280, 720)
    cr = scenes.camera_rays(cam, 1280, 720, 1, seed)
    rng = np.random.default_rng(seed)
    cr = cr[rng.choice(len(cr), n, replace=False)]
    # secondary-like rays: origins on sphere surfaces, random directions
    raw = np.asarray(sp).view(np.float32).reshape(-1, 5).astype(np.float64)
    k = rng.integers(0, len(raw), n)
    nrm = _unit(rng.normal(size=(n, 3)))
    o = raw[k, :3] + nrm * raw[k, 3:4] * 1.0001
    o = np.where(np.linalg.norm(o, axis=1, keepdims=True) < 15.9, o, raw[k, :3] * 0)   # keep |o| inside the bound
    d = _unit(nrm + rng.normal(size=(n, 3)))
    return sp, np.concatenate([cr, np.concatenate([o, d], 1).astype(np.float32)])


def _edge_rays(c, r2, real, n, seed, margins=3.0):
    """Rays whose line passes sphere k at a distance R + delta, delta within +-margins times k's widening R' - R, from
    origins 2..14 away (|o| <= 16): the edge of the half test."""
    rng = np.random.default_rng(seed)
    ids = np.nonzero(real & (r2 < 1e3))[0]
    k = rng.choice(ids, n)
    _, Rp2, _, _, _ = hs.sphere_constants(c, r2)
    R = np.sqrt(r2[k].astype(np.float64))
    widen = np.sqrt(Rp2[k]) - R
    dist = R + rng.uniform(-margins, margins, n) * widen
    d = _unit(rng.normal(size=(n, 3)))
    side = _unit(np.cross(d, rng.normal(size=(n, 3))))
    foot = c[k].astype(np.float64) + side * dist[:, None]
    o = foot - d * rng.uniform(2, 14, n)[:, None]
    keep = np.linalg.norm(o, axis=1) < 15.9
    return np.concatenate([o, d], 1)[keep].astype(np.float32)


def _limit_rays(n, seed):
    """Origins on the sphere |o| = 16 (in float32, a hair inside or outside), aimed at the scene's centre region."""
    rng = np.random.default_rng(seed)
    o = _unit(rng.normal(size=(n, 3))) * 16.0 * (1 + rng.uniform(-1e-7, 1e-7, (n, 1)))
    d = _unit(rng.uniform(-4, 4, (n, 3)) - o)
    return np.concatenate([o, d], 1).astype(np.float32)


def _check_superset(c, r2, real, rays, tag):
    o, d = rays[:, :3], rays[:, 3:]
    ok = hs.in_bound(o, d)
    cand = hs.half_pass(c, r2, o, d)[0]
    need = (hs.fp32_candidates(c, r2, o, d) | hs.exact_accepts(c, r2, o, d)) & real
    # form 4's pass 1 also passes spheres wholly behind the origin only when the origin is inside them; the half pass has
    # no behind test, so every line it passes is a candidate. What matters: nothing form 4 needs is missing.
    miss = need & ~cand & ok[:, None]
    assert not miss.any(), (tag, int(miss.sum()), np.argwhere(miss)[:5].tolist())
    return int(ok.sum())


def test_half_fma_emulation_is_exact():
    rng = np.random.default_rng(0)
    vals = hs.round_half(np.concatenate([rng.normal(0, 1, 4000) * 2.0 ** rng.integers(-16, 8, 4000),
                                         rng.uniform(-64, 64, 4000)]))
    a, b, cc = (rng.choice(vals, 4000) for _ in range(3))
    got = hs.hfma(a, b, cc)

    def rn(fr):
        """Round a Fraction to binary16 (nearest, ties to even) by exact arithmetic."""
        if fr == 0:
            return 0.0
        x = float(fr)
        lo, hi = hs.round_half(x, -1), hs.round_half(x, 1)
        lo_f, hi_f = Fraction(float(lo)), Fraction(float(hi))
        lo_f, hi_f = (lo_f, hi_f) if lo_f <= fr else (hi_f - (hi_f - lo_f) * 2, hi_f)
        while hi_f < fr:
            lo_f, hi_f = hi_f, Fraction(float(hs.round_half(np.nextafter(float(hi_f), np.inf), 1)))
        if lo_f == fr or hi_f == fr:
            return float(fr)
        dl, dh = fr - lo_f, hi_f - fr
        if dl != dh:
            return float(lo_f if dl < dh else hi_f)
        q = float(hi_f - lo_f)
        return float(lo_f) if (float(lo_f) / q) % 2 == 0 else float(hi_f)
    for i in range(len(a)):
        want = rn(Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(cc[i])))
        assert got[i] == want or (got[i] == 0 and want == 0), (a[i], b[i], cc[i], got[i], want)


@pytest.mark.parametrize("which", ["bench", "compact-48", "edge", "limit"])
def test_emulated_error_within_bound(which):
    if which == "bench":
        sp, rays = _bench_rays(3000)
        c, r2, real = _scene(sp)
    else:
        sph, _, _, _ = so.make_scene(46, "compact", seed=1)
        c, r2, real = _scene(sph)
        rays = {"compact-48": lambda: so.near_tangent_rays(sph, 3000, 5)[0], "edge": lambda: _edge_rays(c, r2, real, 3000, 6),
                "limit": lambda: _limit_rays(3000, 7)}[which]()
    o, d = rays[:, :3], rays[:, 3:]
    ok = hs.in_bound(o, d)
    o, d = o[ok], d[ok]
    assert len(o) > 1000
    _, xu, xv, _ = hs.half_pass(c, r2, o, d)
    eu, ev = hs.exact_xuv(c, o, d)
    E = hs.sphere_constants(c, r2)[3]
    ratio = max(float((np.abs(xu - eu)[:, real] / E[real]).max()), float((np.abs(xv - ev)[:, real] / E[real]).max()))
    print(f"{which}: largest |xu, xv error| / E = {ratio:.3f}")
    assert 0.05 < ratio <= 1.0, ratio


@pytest.mark.parametrize("count", list(range(4, 65, 4)))
def test_candidates_contain_every_fp32_accept(count):
    sph, _, _, dup = so.make_scene(count, "compact", seed=count)
    c, r2, real = _scene(sph)
    assert hs.scene_ok(c[real], r2[real])
    n = 800
    sets = {"tangent": so.near_tangent_rays(sph, n, 10 + count)[0], "tmin": so.tmin_rays(sph, n, 20 + count)[0],
            "aimed": so.aimed_rays(sph, 30 + count)[0], "edge": _edge_rays(c, r2, real, n, 40 + count),
            "limit": _limit_rays(n, 50 + count), "degenerate": so.degenerate_rays(sph, 60 + count)}
    inside = sum(_check_superset(c, r2, real, rays, (count, name)) for name, rays in sets.items())
    assert inside > 3 * n
    if dup >= 0:
        # an exact duplicate pair: both ids are candidates for a ray aimed at them (pass 2 then keeps the lower id)
        o = np.array([[0.0, 6.0, 14.0]], np.float32)
        d = _unit(c[dup:dup + 1].astype(np.float64) - o).astype(np.float32)
        cand = hs.half_pass(c, r2, o, d)[0][0]
        assert cand[dup] and cand[dup + 1]


def test_bench_scene_passes_and_ground_is_kept():
    sp, rays = _bench_rays(2000, seed=9)
    c, r2, real = _scene(sp)
    assert hs.scene_ok(c[real], r2[real])
    _check_superset(c, r2, real, rays, "bench")
    # straight-down rays onto the r = 100 ground (sphere 0) from |o| <= 16
    rng = np.random.default_rng(4)
    o = np.stack([rng.uniform(-10, 10, 500), rng.uniform(0.1, 5, 500), rng.uniform(-10, 5, 500)], 1)
    d = _unit(np.stack([rng.uniform(-0.5, 0.5, 500), -np.ones(500), rng.uniform(-0.5, 0.5, 500)], 1))
    g = np.concatenate([o, d], 1).astype(np.float32)
    assert hs.half_pass(c, r2, g[:, :3], g[:, 3:])[0][:, 0].all()
    _check_superset(c, r2, real, g, "ground")


def test_scenes_outside_the_half_range_are_refused():
    sph, _, _, _ = so.make_scene(40, "spread")          # ground r = 1000 at (0, -1000, 0)
    c, r2, real = _scene(sph)
    assert not hs.scene_ok(c[real], r2[real])
    sph, _, _, _ = so.make_scene(65, "compact")         # 68 padded spheres: more than the parameter holds
    c, r2, real = _scene(sph)
    assert not hs.scene_ok(c[real], r2[real])
    sph, _, _, _ = so.make_scene(64, "compact")
    c, r2, real = _scene(sph)
    assert hs.scene_ok(c[real], r2[real])
