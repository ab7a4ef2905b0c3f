"""Emission texture sampling ("emission_texture_sampling") on the GPU.

1. Replay: trace_irradiance at spp 1 under a light with a heavy-tailed layer, a black occluder beside it, a light with layer -1
   and one with an all-zero layer, from ground points and from points on the textured light itself, against a float64
   replay of each sample's stream (bounce, cone, six texture draws, alias choice, sampled point, visibility, both MIS
   weights); the call's ray count equals the replayed count.
2. Unbiasedness: irradiance under the half-textured and the hot-spot light, option on and off, against the float64
   quadrature of the visible cap.
3. Variance: on the hot-spot light the per-sample variance matches a numpy simulation of the same estimator, and beats
   the cone alone by the factor the simulation predicts.
4. The 46-sphere scene with checker emission layers: on against off per entry, also with environment sampling.
5. Inactive is bitwise off: no emission textures, light sampling off, only all-zero layers, layers only on non-emitters.
6. Ordering, boolean coercion and AOVs."""
import numpy as np
import pytest
import torch

import furnace as F
from conftest import rel_l2
from sample_replay import Exact, pixel_seed, u01, unit_vector, xorshift32
from test_environment_sampling_api import build_tables, sample_cells, split_tables, tables_lib  # noqa: F401
from test_gpu_emission_textures import GROUND_R, LIGHT_C, LIGHT_E, LIGHT_R, _cap_integral, _half_texture, _scene
from test_gpu_environment import env_lookup, lat_long_dir, lookup_tolerance
from test_gpu_environment_sampling import random_map
from test_gpu_textures import _every_call
from toypathtracer_b200 import MODE_FAST, scenes

pytestmark = pytest.mark.gpu


@pytest.fixture
def xctx(gpu_ctx):
    yield gpu_ctx
    gpu_ctx.set_emission_textures(None)
    gpu_ctx.set_textures(None)
    gpu_ctx.set_environment(None)
    for k, v in (("fast_variant", -1), ("fast_kform", 2), ("light_sampling", 1), ("environment_sampling", 0),
                 ("emission_texture_sampling", 0)):
        gpu_ctx.set_option(k, v)
    gpu_ctx.set_spp(4)


def replay_layer(w=32, h=16):
    """Heavy-tailed texels: cell probabilities over several decades, so that both weights take every value."""
    return (np.random.default_rng(12).exponential(1.0, (1, h, w, 3)) ** 3).astype(np.float32)


def hot_layer(w=32, h=16):
    """Dark, with a 2 x 2 patch of bright texels on the light's lower half, towards the receivers."""
    t = np.full((1, h, w, 3), 0.02, np.float32)
    t[0, 11:13, 15:17] = (60.0, 45.0, 30.0)
    return t


class LayerTables:
    def __init__(self, lib, layer):
        self.m = layer
        self.h, self.w = layer.shape[:2]
        ok, tex, rows, cols, _w = build_tables(lib, layer)
        assert ok
        self.P = tex[..., 3].astype(np.float64)
        self.rp, self.ra, self.cp, self.ca = split_tables(self.w, self.h, rows, cols)

    def sample(self, x):
        """Six raw draws -> unit normal, sin theta, P, and the distance of (u, v) to a cell edge."""
        i, j = sample_cells((x[0] & 0xFFFFFF).astype(np.int64), u01(x[1]).astype(np.float32),
                            (x[2] & 0xFFFFFF).astype(np.int64), u01(x[3]).astype(np.float32),
                            self.w, self.h, self.rp, self.ra, self.cp, self.ca)
        u, v = i + u01(x[4]), j + u01(x[5])
        return lat_long_dir(u, v, self.w, self.h), np.sin(v * np.pi / self.h), self.P[j, i]

    def cell_p(self, n):
        u = (np.arctan2(n[:, 0], -n[:, 2]) + np.pi) / (2 * np.pi) * self.w
        v = np.arccos(np.clip(n[:, 1], -1, 1)) / np.pi * self.h
        i = np.floor(u).astype(np.int64) % self.w
        j = np.clip(np.floor(v).astype(np.int64), 0, self.h - 1)
        edge = np.minimum(np.minimum(u % 1, 1 - u % 1), np.minimum(v % 1, 1 - v % 1))
        return self.P[j, i], edge


def _draws(state, n):
    out = []
    for _ in range(n):
        state = xorshift32(state)
        out.append(state)
    return out, state


def _hit(o, d, c, r):
    """Nearest t > 1e-3 along unit d from o with sphere (c, r), inf on a miss; and the test's margin."""
    oc = o - c
    b = (oc * d).sum(-1)
    disc = b * b - ((oc * oc).sum(-1) - r * r)
    sq = np.sqrt(np.maximum(disc, 0.0))
    t0, t1 = -b - sq, -b + sq
    t = np.where(t0 > 1e-3, t0, np.where(t1 > 1e-3, t1, np.inf))
    return np.where(disc > 0, t, np.inf), np.abs(disc) / (r * r)


def cone_sample(o, c, r, e1, e2):
    """sample_light_cone in float64: the direction, omega."""
    pc = c - o
    sw = pc / np.linalg.norm(pc, axis=1, keepdims=True)
    sgn = np.where(np.signbit(sw[:, 2]), -1.0, 1.0)
    oa = -1.0 / (sgn + sw[:, 2])
    ob = sw[:, 0] * sw[:, 1] * oa
    su = np.stack([1.0 + sgn * sw[:, 0] ** 2 * oa, sgn * ob, -sgn * sw[:, 0]], 1)
    sv = np.stack([ob, sgn + sw[:, 1] ** 2 * oa, -sw[:, 1]], 1)
    cmax = np.sqrt(1.0 - r * r / (pc * pc).sum(1))
    cosA = 1.0 - e1 + e1 * cmax
    sinA = np.sqrt(1.0 - cosA ** 2)
    ph = 2 * np.pi * e2
    l = su * (np.cos(ph) * sinA)[:, None] + sv * (np.sin(ph) * sinA)[:, None] + sw * cosA[:, None]
    return l, 2 * np.pi * (1.0 - cmax), np.abs(sw[:, 2])


def pt_of(T, P, s, r, ox):
    """pt(x) in solid angle at o, ox = o - x, for the layer cell probability P and sin theta s at x."""
    d2 = (ox * ox).sum(1)
    return P * T.w * T.h / (2 * np.pi ** 2 * s) / (r * r) * d2


# ---- 1. replay -------------------------------------------------------------------------------------------------------
OCC_C, OCC_R = np.array([1.1, 1.7, 0.2]), 0.45
L1_C, L1_R, L1_E = np.array([-3.0, 2.5, -1.0]), 0.5, np.float32([0.5, 0.7, 0.9])
L2_C, L2_R, L2_E = np.array([3.0, 2.5, -1.0]), 0.4, np.float32([0.9, 0.9, 0.9])


def replay_scene():
    return _scene([LIGHT_C, OCC_C, L1_C, L2_C], [LIGHT_R, OCC_R, L1_R, L2_R], [F.LAMBERT] * 4, [(0, 0, 0)] * 4,
                  [LIGHT_E, (0, 0, 0), L1_E, L2_E])


SPHERES = [(LIGHT_C, LIGHT_R), (OCC_C, OCC_R), (L1_C, L1_R), (L2_C, L2_R)]


def _first_hit(o, d):
    """Index of the first sphere hit (-1: none), its t, and the smallest margin over all spheres."""
    ts, ms = zip(*[_hit(o, d, c, r) for c, r in SPHERES])
    ts, ms = np.stack(ts, 1), np.stack(ms, 1)
    k = np.argmin(ts, 1)
    t = ts[np.arange(len(o)), k]
    return np.where(np.isfinite(t), k, -1), t, ms.min(1)


def _points(n, frame, rng):
    """Ground points and points on the textured light (id 0), each index's point chosen so that its bounce (drawn
    first) leaves the scene with a margin: every ray after the vertex's shadow rays is then one escaping ray."""
    seeds = pixel_seed(np.arange(n, dtype=np.uint64), frame)
    x, _ = _draws(seeds, 2)
    uv = unit_vector(Exact(), x[0], x[1])
    pts, ids = np.zeros((n, 6), np.float32), np.full(n, -1, np.int32)
    left = np.arange(n)
    on_light = np.arange(n) % 8 == 0
    for _ in range(200):
        if not len(left):
            break
        m = len(left)
        g = np.stack([rng.uniform(-2.5, 2.5, m), np.zeros(m), rng.uniform(-2.5, 1.5, m)], 1)
        gn = rng.normal(size=(m, 3)) * 0.4 + np.array([0, 1.0, 0])
        gn /= np.linalg.norm(gn, axis=1, keepdims=True)
        ln = rng.normal(size=(m, 3))
        ln /= np.linalg.norm(ln, axis=1, keepdims=True)
        ol = on_light[left][:, None]
        p = np.where(ol, LIGHT_C + LIGHT_R * ln, g)
        nn = np.where(ol, ln, gn)
        cand = np.concatenate([p, nn], 1).astype(np.float32)
        o, nl = cand[:, :3].astype(np.float64), cand[:, 3:].astype(np.float64)
        b = nl + uv[left]
        b /= np.linalg.norm(b, axis=1, keepdims=True)
        k, _t, mg = _first_hit(o + 1e-4 * nl, b)
        ok = (k < 0) & (mg > 1e-3)
        pts[left[ok]] = cand[ok]
        ids[left[ok]] = np.where(on_light[left[ok]], 0, -1)
        left = left[~ok]
    assert not len(left)
    return pts, ids


def replay(T, pts, ids, frame):
    """Per point: value (3), ray count, well-conditioned flag, whether the texture ray was traced, the two weights."""
    n = len(pts)
    o, nl = pts[:, :3].astype(np.float64), pts[:, 3:].astype(np.float64)
    state = pixel_seed(np.arange(n, dtype=np.uint64), frame)
    _x, state = _draws(state, 2)
    val = np.zeros((n, 3))
    ltol = np.zeros(n)                                # the lookups' sensitivity to the float32 hit normals
    count = np.ones(n, np.int64)                      # the bounce
    well = np.ones(n, bool)
    traced = np.zeros(n, bool)
    wc = np.full(n, np.nan)
    wt = np.full(n, np.nan)
    own = ids == 0
    L0 = LIGHT_E.astype(np.float64)

    def shadow(li, l, target):
        k, t, mg = _first_hit(o[li], l)
        return k == target, t, mg

    # light 0 (textured, hot spot): cone, then the texture sample
    li = np.nonzero(~own)[0]
    (e1, e2), st2 = _draws(state[li], 2)
    l, omega, swz = cone_sample(o[li], LIGHT_C, LIGHT_R, u01(e1), u01(e2))
    count[li] += 1
    reach, t, mg = shadow(li, l, 0)
    x = o[li] + l * np.where(reach, t, 0)[:, None]
    nx = (x - LIGHT_C) / LIGHT_R
    P, edge = T.cell_p(nx)
    s = np.sqrt(np.maximum(1 - nx[:, 1] ** 2, 0))
    ox = o[li] - x
    with np.errstate(divide="ignore", invalid="ignore"):
        cosx = (nx * ox).sum(1) / np.linalg.norm(ox, axis=1)
        pt = np.where(reach, pt_of(T, P, s, LIGHT_R, ox) / cosx, 0.0)
        w = np.where(pt > 0, (1 / omega) ** 2 / ((1 / omega) ** 2 + pt ** 2), 1.0)
    m = np.maximum((l * nl[li]).sum(1), 0)
    val[li] += np.where(reach[:, None], L0 * env_lookup(T.m, nx) * (m * omega / np.pi * w)[:, None], 0.0)
    # (the float32 cone direction carries the sampler's cosA / sinA rounding, which the hit point magnifies by d / r)
    ltol[li] += np.where(reach, lookup_tolerance(T.m, nx, eps=1e-4) * m * omega / np.pi * w, 0.0)
    wc[li] = np.where(reach, w, np.nan)
    # a hit near the light's silhouette moves its normal, and the steep layer's lookup, far for a small change of l
    well[li] &= (swz > 1e-4) & (mg > 1e-4) & (((edge > 1e-4) & (mg > 1e-2)) | ~reach)
    e, st8 = _draws(st2, 6)
    ns, s_t, P_t = T.sample(e)
    xs = LIGHT_C + LIGHT_R * ns
    ox = o[li] - xs
    dist = np.linalg.norm(ox, axis=1)
    lt = -ox / dist[:, None]
    cx = (ns * ox).sum(1) / dist
    mt = (lt * nl[li]).sum(1)
    tr = (cx > 0) & (mt > 0) & (s_t > 0)
    traced[li] = tr
    count[li] += tr
    with np.errstate(divide="ignore", invalid="ignore"):
        ptt = pt_of(T, P_t, np.where(s_t > 0, s_t, 1), LIGHT_R, ox) / cx
        pend = np.where(tr, mt / np.pi * ptt / (ptt ** 2 + (1 / omega) ** 2), 0.0)
    reach_t, t2, mg2 = shadow(li, lt, 0)
    nh = (o[li] + lt * np.where(reach_t, t2, 0)[:, None] - LIGHT_C) / LIGHT_R
    val[li] += np.where((tr & reach_t)[:, None], L0 * env_lookup(T.m, nh) * pend[:, None], 0.0)
    ltol[li] += np.where(tr & reach_t, lookup_tolerance(T.m, nh, eps=1e-5) * pend, 0.0)
    wt[li] = np.where(tr, ptt ** 2 / (ptt ** 2 + (1 / omega) ** 2), np.nan)
    well[li] &= ~tr | ((mg2 > 1e-4) & ((mg2 > 1e-2) | ~reach_t) & (np.abs(cx) > 1e-4) & (np.abs(mt) > 1e-4))
    state = state.copy()
    state[li] = st8
    # light 1 (layer -1) and light 2 (all-zero layer): a cone each, nothing drawn after it; light 2 adds e x 0
    for c, r, E, target in ((L1_C, L1_R, L1_E, 2), (L2_C, L2_R, L2_E * 0, 3)):
        (e1, e2), state = _draws(state, 2)
        l, omega, swz = cone_sample(o, c, r, u01(e1), u01(e2))
        count += 1
        reach, t, mg = shadow(np.arange(n), l, target)
        m = np.maximum((l * nl).sum(1), 0)
        val += np.where(reach[:, None], E.astype(np.float64) * (m * omega / np.pi)[:, None], 0.0)
        well &= (swz > 1e-4) & (mg > 1e-4)
    return val * np.pi, ltol * np.pi, count, well, traced, wc, wt


@pytest.mark.parametrize("frame", [3, 11])
def test_replay_of_irradiance_samples(xctx, tables_lib, frame):
    layer = replay_layer()
    T = LayerTables(tables_lib, layer[0])
    xctx.set_scene(*replay_scene())
    xctx.set_environment(np.zeros((4, 8, 3), np.float32))        # a black map: an escaping ray adds nothing
    xctx.set_emission_textures(np.concatenate([layer, np.zeros_like(layer)]), [0, -1, -1, 1])
    xctx.set_option("emission_texture_sampling", 1)
    n = 16384
    pts, ids = _points(n, frame, np.random.default_rng(frame))
    out, rays = xctx.trace_irradiance(pts, ids, spp=1, frame=frame)
    val, ltol, count, well, traced, wc, wt = replay(T, pts, ids, frame)
    assert rays == int(count.sum()), (rays, int(count.sum()))
    assert well.mean() > 0.9, well.mean()
    got = out[:, :3].astype(np.float64)
    tol = 2e-3 * np.abs(val) + 2e-3 * np.abs(val).max(1, keepdims=True) + 1e-6 + 2.0 * ltol[:, None]
    bad = well[:, None] & (np.abs(got - val) > tol)
    assert not bad.any(), (int(bad.any(1).sum()), np.nonzero(bad.any(1))[0][:5], got[bad.any(1)][:3], val[bad.any(1)][:3])
    # what the replay is about happens: texture rays traced and not, both weights away from 0 and 1, own-light points
    assert traced.sum() > n // 4 and (~traced & (ids != 0)).sum() > 100
    assert ((wc > 0.05) & (wc < 0.95)).sum() > 20 and ((wt > 0.05) & (wt < 0.95)).sum() > 20, (np.nanpercentile(wc, [5, 50, 95]), np.nanpercentile(wt, [5, 50, 95]))
    assert (ids == 0).sum() > n // 10
    # the option off: the same points trace one texture ray fewer wherever one was traced
    xctx.set_option("emission_texture_sampling", 0)
    _out, rays_off = xctx.trace_irradiance(pts, ids, spp=1, frame=frame)
    assert rays_off == rays - int(traced.sum())


# ---- 2. unbiasedness ---------------------------------------------------------------------------------------------------
def _cap_scene():
    return _scene([LIGHT_C, (0.0, -GROUND_R, 0.0)], [LIGHT_R, GROUND_R], [F.LAMBERT, F.LAMBERT], [(0, 0, 0), (1, 1, 1)],
                  [LIGHT_E, (0, 0, 0)])


def _ground_point(x):
    y = GROUND_R * np.cos(np.arcsin(x / GROUND_R)) - GROUND_R
    return np.concatenate([[x, y, 0.0], np.array([x, y + GROUND_R, 0.0]) / GROUND_R]).astype(np.float32)


def _samples_at(ctx, pt, copies, spp=1, frame=1):
    out, _ = ctx.trace_irradiance(np.tile(pt, (copies, 1)), np.ones(copies, np.int32), spp=spp, frame=frame)
    return out[:, :3].astype(np.float64)


@pytest.mark.parametrize("which", ["half", "hot", "hot_second_layer"])
@pytest.mark.parametrize("on", [0, 1])
def test_irradiance_is_the_cap_integral(xctx, which, on):
    """hot_second_layer: the light takes layer 1 of a set whose layer 0 is another sampleable image (its hot spot on
    the far side), so the texture sample must read its own layer's tables."""
    tex = _half_texture() if which == "half" else hot_layer()
    if which == "hot_second_layer":
        other = hot_layer()[:, ::-1].copy()
        xctx.set_emission_textures(np.concatenate([other, tex]), [1, -1])
    else:
        xctx.set_emission_textures(tex, [0, -1])
    xctx.set_scene(*_cap_scene())
    xctx.set_environment(np.zeros((4, 8, 3), np.float32))
    xctx.set_option("emission_texture_sampling", on)
    copies = 1 << 15
    for x in (0.0, 1.3, 2.6):
        pt = _ground_point(x)
        want = _cap_integral(pt[:3].astype(np.float64), pt[3:].astype(np.float64), tex)
        e = _samples_at(xctx, pt, copies, spp=16)
        mean, se = e.mean(0), e.std(0) / np.sqrt(copies)
        assert (np.abs(mean - want) < 5.0 * se + 1e-6 * want).all(), (which, on, x, mean, want, se)


# ---- 3. variance -------------------------------------------------------------------------------------------------------
def simulate(T, pt, n, rng):
    """Per-sample irradiance values at ground point pt under the hot-spot light, cone alone and cone + texture sample with
    the power heuristic, in float64 with numpy's generator."""
    o = np.broadcast_to(pt[:3].astype(np.float64), (n, 3))
    nl = pt[3:].astype(np.float64)
    l, omega, _ = cone_sample(o, LIGHT_C, LIGHT_R, rng.random(n), rng.random(n))
    t, _ = _hit(o, l, LIGHT_C, LIGHT_R)
    x = o + l * t[:, None]
    nx = (x - LIGHT_C) / LIGHT_R
    le = LIGHT_E.astype(np.float64) * env_lookup(T.m, nx)
    m = np.maximum(l @ nl, 0)
    P, _ = T.cell_p(nx)
    ox = o - x
    with np.errstate(divide="ignore", invalid="ignore"):
        cosx = (nx * ox).sum(1) / np.linalg.norm(ox, axis=1)
        ptc = pt_of(T, P, np.sqrt(np.maximum(1 - nx[:, 1] ** 2, 0)), LIGHT_R, ox) / cosx
        w = np.where(ptc > 0, 1.0 / (1.0 + (ptc * omega) ** 2), 1.0)
    off = np.pi * le * (m * omega / np.pi)[:, None]
    draws = [rng.integers(0, 1 << 24, n).astype(np.uint32) for _ in range(6)]
    ns, s, Pt = T.sample(draws)
    xs = LIGHT_C + LIGHT_R * ns
    ox = o - xs
    dist = np.linalg.norm(ox, axis=1)
    lt = -ox / dist[:, None]
    cx = (ns * ox).sum(1) / dist
    mt = lt @ nl
    tr = (cx > 0) & (mt > 0) & (s > 0)
    with np.errstate(divide="ignore", invalid="ignore"):
        ptt = pt_of(T, Pt, np.where(s > 0, s, 1), LIGHT_R, ox) / cx
        pend = np.where(tr, mt / np.pi * ptt / (ptt ** 2 + (1 / omega) ** 2), 0.0)
    th, _ = _hit(o, lt, LIGHT_C, LIGHT_R)
    nh = (o + lt * np.where(np.isfinite(th), th, 0)[:, None] - LIGHT_C) / LIGHT_R
    on = off * w[:, None] + np.pi * np.where((tr & np.isfinite(th))[:, None], LIGHT_E * env_lookup(T.m, nh) * pend[:, None], 0)
    return off, on


def _var_and_rel_se(v):
    """Per-channel variance of the samples v and the relative standard error of that estimate."""
    c = v - v.mean(0)
    m2, m4 = (c ** 2).mean(0), (c ** 4).mean(0)
    return m2, np.sqrt(np.maximum(m4 / m2 ** 2 - 1, 0) / len(v))


def test_variance_matches_the_model_and_beats_the_cone(xctx, tables_lib):
    layer = hot_layer()
    T = LayerTables(tables_lib, layer[0])
    pt = _ground_point(1.3)
    sim_off, sim_on = simulate(T, pt, 1 << 21, np.random.default_rng(2))
    vs_off, rs_off = _var_and_rel_se(sim_off)
    vs_on, rs_on = _var_and_rel_se(sim_on)
    xctx.set_scene(*_cap_scene())
    xctx.set_environment(np.zeros((4, 8, 3), np.float32))
    xctx.set_emission_textures(layer, [0, -1])
    got = {}
    for on in (0, 1):
        xctx.set_option("emission_texture_sampling", on)
        got[on] = _var_and_rel_se(_samples_at(xctx, pt, 1 << 20))
    (vg_off, rg_off), (vg_on, rg_on) = got[0], got[1]
    # each measured variance is the model's
    assert (np.abs(vg_on / vs_on - 1) < 5 * np.hypot(rg_on, rs_on)).all(), (vg_on, vs_on, rg_on, rs_on)
    assert (np.abs(vg_off / vs_off - 1) < 5 * np.hypot(rg_off, rs_off)).all(), (vg_off, vs_off, rg_off, rs_off)
    # and the gain is at least the model's, less its statistical margin
    ratio_sim = vs_off / vs_on
    margin = 5 * np.sqrt(rs_off ** 2 + rs_on ** 2 + rg_off ** 2 + rg_on ** 2)
    assert (vg_off / vg_on >= ratio_sim * (1 - margin)).all(), (vg_off / vg_on, ratio_sim, margin)
    assert (ratio_sim > 2).all(), ratio_sim                 # the case is one where the technique matters
    print(f"per-sample variance, off/on: measured {vg_off / vg_on}, simulated {ratio_sim}")


# ---- 4. the 46-sphere scene ---------------------------------------------------------------------------------------------
def checker_layers(w=16, h=8):
    t = np.full((1, h, w, 3), 0.2, np.float32)
    ii, jj = np.meshgrid(np.arange(w), np.arange(h))
    t[0][(ii + jj) % 2 == 0] = (3.0, 2.5, 2.0)
    return t


def _mean_se(ctx, rays, spp):
    (s4, q4), _r = ctx.trace_samples(rays, spp=spp)
    s4, q4 = np.asarray(s4, np.float64), np.asarray(q4, np.float64)
    k = s4[:, 3:4]
    mean = s4[:, :3] / k
    var = np.maximum(q4[:, :3] / k - mean ** 2, 0) * k / (k - 1)
    return mean, np.sqrt(var / k)


@pytest.mark.parametrize("env", [0, 1])
def test_reference_scene_on_and_off_agree(xctx, env):
    w, h = 48, 27
    s, mats, cam, em = scenes.reference_scene(w, h)
    xctx.set_scene(s, mats, cam, em)
    if env:
        xctx.set_environment(random_map(32, 16, seed=4))
        xctx.set_option("environment_sampling", 1)
    emitters = (mats["emissive"] != 0).any(1)
    xctx.set_emission_textures(checker_layers(), np.where(emitters, 0, -1).astype(np.int32))
    rays = scenes.camera_rays(cam, w, h, seed=3)
    spp = 1024
    res = {}
    for on in (0, 1):
        xctx.set_option("emission_texture_sampling", on)
        res[on] = _mean_se(xctx, rays, spp)
    (m0, s0), (m1, s1) = res[0], res[1]
    z = np.abs(m1 - m0) / (np.hypot(s0, s1) + 1e-5 * np.abs(m0) + 1e-9)
    assert (z < 5).all(), (float(z.max()), np.unravel_index(np.argmax(z), z.shape))
    assert rel_l2(m1, m0) > 0                      # the estimators differ


# ---- 5. inactive is bitwise off -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["no_textures", "light_sampling_off", "all_zero_layers", "non_emitters_only"])
def test_inactive_is_bitwise_off(xctx, case):
    w, h = 32, 18
    s, mats, cam, em = scenes.reference_scene(w, h)
    emitters = (mats["emissive"] != 0).any(1)
    if case == "light_sampling_off":
        xctx.set_option("light_sampling", 0)
    xctx.set_scene(s, mats, cam, em)
    if case == "light_sampling_off":
        xctx.set_emission_textures(checker_layers(), np.where(emitters, 0, -1).astype(np.int32))
    if case == "all_zero_layers":
        xctx.set_emission_textures(np.zeros((2, 4, 8, 3), np.float32), np.where(emitters, 0, 1).astype(np.int32))
    if case == "non_emitters_only":
        xctx.set_emission_textures(checker_layers(), np.where(emitters, -1, 0).astype(np.int32))
    ref = _every_call(xctx, w, h, cam, s, (-1, 3))
    xctx.set_option("emission_texture_sampling", 1)
    got = _every_call(xctx, w, h, cam, s, (-1, 3))
    for k in ref:
        (ga, gr), (ra, rr) = got[k], ref[k]
        assert gr == rr, (case, k, gr, rr)
        assert np.asarray(ga).tobytes() == np.asarray(ra).tobytes(), (case, k)


# ---- 6. ordering, coercion, AOVs ---------------------------------------------------------------------------------------
def test_textures_set_during_a_sampled_draw_are_not_seen_by_it(xctx):
    """One sample per pixel, so each pixel is written once and the outputs are bitwise reproducible."""
    w, h, spp = 1280, 720, 1
    s, mats, cam, em = scenes.reference_scene(w, h)
    xctx.set_scene(s, mats, cam, em)
    xctx.set_spp(spp)
    xctx.set_option("emission_texture_sampling", 1)
    emitters = np.where((mats["emissive"] != 0).any(1), 0, -1).astype(np.int32)
    a, b = checker_layers(), hot_layer(16, 8)
    bufs = [torch.zeros((h, w, 4), dtype=torch.float32, device="cuda") for _ in range(2)]
    torch.cuda.synchronize()
    xctx.set_emission_textures(a, emitters)
    xctx.draw(0, 1, w, h, bufs[0], flags=0, mode=MODE_FAST, want_rays=False)
    xctx.set_emission_textures(b, emitters)
    xctx.draw(0, 1, w, h, bufs[1], flags=0, mode=MODE_FAST, want_rays=False)
    torch.cuda.synchronize()
    got = [t.cpu().numpy() for t in bufs]
    refs = []
    for t in (a, b):
        xctx.set_emission_textures(t, emitters)
        buf = torch.zeros((h, w, 4), dtype=torch.float32, device="cuda")
        xctx.draw(0, 1, w, h, buf, flags=0, mode=MODE_FAST)
        refs.append(buf.cpu().numpy())
    assert got[0].tobytes() == refs[0].tobytes() and got[1].tobytes() == refs[1].tobytes()
    assert rel_l2(refs[1], refs[0]) > 0.05


def test_option_is_boolean_and_aovs_are_unaffected(xctx):
    w, h = 32, 18
    s, mats, cam, em = scenes.reference_scene(w, h)
    xctx.set_scene(s, mats, cam, em)
    xctx.set_emission_textures(checker_layers(), np.where((mats["emissive"] != 0).any(1), 0, -1).astype(np.int32))
    res = {}
    for v in (0, 1, 7, -3):
        xctx.set_option("emission_texture_sampling", v)
        res[v] = _every_call(xctx, w, h, cam, s, (-1,))
    for v in (7, -3):
        for k in res[1]:
            assert np.asarray(res[v][k][0]).tobytes() == np.asarray(res[1][k][0]).tobytes() and res[v][k][1] == res[1][k][1], (v, k)
    for k in ("daovs", "taovs"):
        assert np.asarray(res[1][k][0]).tobytes() == np.asarray(res[0][k][0]).tobytes(), k
    # the option is active: the sampled estimate differs and traces more rays
    assert res[1]["irr"][1] > res[0]["irr"][1]
