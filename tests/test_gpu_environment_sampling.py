"""Environment importance sampling ("environment_sampling") on the GPU.

1. Replay: trace_samples points at spp 1 beside a black occluder, and caller rays that meet a Lambert vertex from inside
   its sphere, against a float64 replay of each sample's stream (bounce, six environment draws, alias choice, in-cell
   direction, pdf, shadow-ray visibility, lookup, MIS weights); the call's ray count equals the replayed sum.
2. Unbiasedness: the irradiance at points facing a random map and a sun map, sampling on and off, against a float64
   quadrature of the bilinear map times the cosine.
3. Efficiency: the per-sample variance on the sun map against a numpy simulation of the same estimator on the same tables.
4. Whole scenes: the 46-sphere scene under sky_environment, sampling on against off, per entry within Monte-Carlo error;
   draws, trace_rays and trace_irradiance equal the sample sums of the same streams; under the sun map, sampling on is
   closer to a high-spp reference at equal spp.
5. Inactive is identical: option on without a map, with light sampling off, and with an all-black map.
6. Ordering, refusals and scope: in-flight calls keep their map, explicit variants are refused, only the sampling
   instances run, AOVs are unchanged, parity modes stay refused."""
import numpy as np
import pytest
import torch

from conftest import rel_l2
from sample_replay import Exact, pixel_seed, u01, unit_vector, xorshift32
from test_environment_sampling_api import build_tables, sample_cells, split_tables, tables_lib  # noqa: F401
from test_gpu_environment import env_lookup, far_scene, lat_long_dir
from toypathtracer_b200 import MATERIAL_DTYPE, MODE_EXACT, MODE_FAST, MODE_REFGPU, SPHERE_DTYPE, TptError, scenes
import furnace as F

pytestmark = pytest.mark.gpu

SAMPLING_KERNELS = ("k_fast_queue<128, 6, 0>", "k_fast_queue<768, 1, 0>", "k_fast_rays<128, 6, 0>", "k_fast_rays<768, 1, 0>",
                    "k_fast_samples<128, 6, 0,", "k_fast_samples<768, 1, 0,")


def _sampling_only(ctx):
    """The call's trace kernels are environment-sampling instances only (and there is one)."""
    kinds = [k for k in ctx.last_kernels() if k.startswith("k_fast")]
    return bool(kinds) and all(k.startswith(SAMPLING_KERNELS) for k in kinds)


@pytest.fixture
def sctx(gpu_ctx):
    yield gpu_ctx
    gpu_ctx.set_environment(None)
    for k, v in (("environment_sampling", 0), ("fast_variant", -1), ("fast_kform", 2), ("light_sampling", 1),
                 ("host_zero_copy", 1)):
        gpu_ctx.set_option(k, v)
    gpu_ctx.set_spp(4)


# ---- maps ------------------------------------------------------------------------------------------------------------
SUN_ELEV = np.radians(30.0)
SUN_RADIUS = np.radians(0.53) / 2
SUN_DIR = np.array([0.3 * np.cos(SUN_ELEV), np.sin(SUN_ELEV), -np.sqrt(1 - 0.09) * np.cos(SUN_ELEV)])


def sun_map(w, h, sky=None):
    """sky_environment(w, h) plus a 0.53 degree disc 30 degrees above the horizon, rasterised by 8 x 8 supersampled
    coverage, bright enough to give most of the horizontal irradiance (the sky's is ~ pi * 0.8)."""
    m = (scenes.sky_environment(w, h) if sky is None else sky.copy())[..., :3].astype(np.float64)
    s = SUN_DIR / np.linalg.norm(SUN_DIR)
    theta_s = np.arccos(s[1])
    j0 = int(theta_s / np.pi * h)
    span = int(np.ceil(4 * SUN_RADIUS / np.pi * h)) + 2
    phi_s = np.arctan2(s[0], -s[2])
    i0 = int((phi_s + np.pi) / (2 * np.pi) * w)
    spanu = int(np.ceil(4 * SUN_RADIUS / (2 * np.pi) * w / max(np.sin(theta_s), 1e-3))) + 2
    sub = (np.arange(8) + 0.5) / 8
    radiance = 4.0 / (np.pi * SUN_RADIUS ** 2 * s[1])        # E_sun = L * omega * cos = 4 on a horizontal receiver
    for j in range(j0 - span, j0 + span + 1):
        for i in range(i0 - spanu, i0 + spanu + 1):
            uu, vv = np.meshgrid(i + sub, j + sub)
            d = lat_long_dir(uu, vv, w, h).reshape(-1, 3)
            cov = float((d @ s > np.cos(SUN_RADIUS)).mean())
            m[j % h, i % w] += radiance * cov
    return m.astype(np.float32)


def random_map(w=64, h=32, seed=7):
    return np.random.default_rng(seed).exponential(1.0, (h, w, 3)).astype(np.float32)


def irradiance_quadrature(m, normals, sub=4):
    """E(n) = integral of the bilinear map times max(0, d.n) over the sphere: midpoint rule on a sub x sub grid per texel
    in (phi, theta), weighted by sin theta."""
    h, w = m.shape[:2]
    uu, vv = np.meshgrid((np.arange(w * sub) + 0.5) / sub, (np.arange(h * sub) + 0.5) / sub)
    d = lat_long_dir(uu, vv, w, h).reshape(-1, 3)
    L = env_lookup(m, d)
    dA = (2 * np.pi / (w * sub)) * (np.pi / (h * sub)) * np.sin(vv.ravel() * np.pi / h)
    out = []
    for n in normals:
        c = np.maximum(d @ n, 0.0) * dA
        out.append((L * c[:, None]).sum(0))
    return np.array(out)


def _samples(ctx, inputs, points, spp, frame, ids=None):
    (s4, q4), r = ctx.trace_samples(inputs, ids=ids, points=points, spp=spp, frame=frame,
                                    sum4=np.zeros((len(inputs), 4), np.float32), sq4=np.zeros((len(inputs), 4), np.float32))
    return s4.astype(np.float64), q4.astype(np.float64), r


def mean_se(s4, q4):
    n = s4[:, 3:4]
    mean = s4[:, :3] / n
    var = np.maximum(q4[:, :3] / n - mean ** 2, 0.0) * n / (n - 1)
    return mean, np.sqrt(var / n), var


# ---- 1. replay -------------------------------------------------------------------------------------------------------
def _sphere_hit(o, d, c, r):
    """Nearest t > 1e-3 of rays o + t d (d unit) with one sphere, or inf; and the margin |b^2 - q| / r^2 of the test."""
    oc = o - c
    b = (oc * d).sum(-1)
    q = (oc * oc).sum(-1) - r * r
    disc = b * b - q
    sq = np.sqrt(np.maximum(disc, 0.0))
    t0, t1 = -b - sq, -b + sq
    t = np.where(t0 > 1e-3, t0, np.where(t1 > 1e-3, t1, np.inf))
    t = np.where(disc > 0, t, np.inf)
    return t, np.abs(disc) / (r * r)


class EnvTables:
    def __init__(self, lib, m):
        h, w = m.shape[:2]
        ok, tex, rows, cols, _w = build_tables(lib, m)
        assert ok
        self.w, self.h, self.m = w, h, m
        self.P = tex[..., 3].astype(np.float64)
        self.rp, self.ra, self.cp, self.ca = split_tables(w, h, rows, cols)

    def sample(self, x):
        """The six draws x[0..5] (raw uint32) -> direction, sin theta, cell probability, and cell-edge margins."""
        k1, k3 = (x[0] & 0xFFFFFF).astype(np.int64), (x[2] & 0xFFFFFF).astype(np.int64)
        i, j = sample_cells(k1, u01(x[1]).astype(np.float32), k3, u01(x[3]).astype(np.float32),
                            self.w, self.h, self.rp, self.ra, self.cp, self.ca)
        u, v = i + u01(x[4]), j + u01(x[5])
        d = lat_long_dir(u, v, self.w, self.h)
        return d, np.sin(v * np.pi / self.h), self.P[j, i]

    def pdf(self, d):
        """pdf_e(d) and the distance of d's (u, v) to the nearest cell edge (a lookup near an edge may take either cell)."""
        phi = np.arctan2(d[:, 0], -d[:, 2])
        theta = np.arccos(np.clip(d[:, 1], -1, 1))
        u = (phi + np.pi) / (2 * np.pi) * self.w
        v = theta / np.pi * self.h
        i = np.floor(u).astype(np.int64) % self.w
        j = np.clip(np.floor(v).astype(np.int64), 0, self.h - 1)
        s = np.sin(theta)
        with np.errstate(divide="ignore", invalid="ignore"):
            pe = self.P[j, i] * self.w * self.h / (2 * np.pi ** 2 * s)
        edge = np.minimum(np.minimum(u % 1, 1 - u % 1), np.minimum(v % 1, 1 - v % 1))
        return pe, edge


def _unit(x1, x2):
    return unit_vector(Exact(), x1, x2)


def _power(pa, pb):
    a2, b2 = pa * pa, pb * pb
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(b2 > 0, a2 / (a2 + b2), 1.0)


def _draws(state, n):
    out = []
    for _ in range(n):
        state = xorshift32(state)
        out.append(state)
    return out, state


def test_replay_points_beside_a_black_occluder(sctx, tables_lib):
    m = random_map(64, 32, seed=3)
    T = EnvTables(tables_lib, m)
    centre, radius = np.array([0.0, 0.3, -2.0]), 1.2
    sph = np.zeros(1, SPHERE_DTYPE)
    sph[0] = (centre, radius, 1.0 / radius)
    mats = np.zeros(1, MATERIAL_DTYPE)                 # black Lambert, not emissive
    sctx.set_scene(sph, mats, F.furnace_camera(8, 8), np.zeros(0, np.int32))
    sctx.set_environment(m)
    sctx.set_option("environment_sampling", 1)
    rng = np.random.default_rng(21)
    n = 8192
    nrm = rng.normal(size=(n, 3))
    nrm[:, 2] -= 1.0                                   # mostly towards the occluder
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    pts = np.concatenate([np.zeros((n, 3)), nrm], 1).astype(np.float32)
    frame = 5
    s4, q4, rays = _samples(sctx, pts, True, 1, frame)
    assert (s4[:, 3] == 1).all()
    assert _sampling_only(sctx)

    o = pts[:, :3].astype(np.float64)
    nl = pts[:, 3:].astype(np.float64)
    state = pixel_seed(np.arange(n, dtype=np.uint64), frame)
    x, state = _draws(state, 2)
    nxt = nl + _unit(x[0], x[1])
    nxt /= np.linalg.norm(nxt, axis=1, keepdims=True)
    e, state = _draws(state, 6)
    l, s, P = T.sample(e)
    c = (l * nl).sum(1)
    traced = (c > 0) & (s > 0)
    pe = P * T.w * T.h / (2 * np.pi ** 2 * np.where(s > 0, s, 1))
    pb = c / np.pi
    with np.errstate(invalid="ignore", divide="ignore"):
        pend = np.where(traced, pb * pe / (pe * pe + pb * pb), 0.0)
    ts, ms = _sphere_hit(o, l, centre, radius)
    val = np.where((traced & ~np.isfinite(ts))[:, None], env_lookup(m, l) * pend[:, None], 0.0)
    count = traced.astype(np.int64) + 1
    tb, mb = _sphere_hit(o, nxt, centre, radius)
    pe_b, edge = T.pdf(nxt)
    wb = _power(np.maximum((nxt * nl).sum(1), 0) / np.pi, pe_b)
    miss = ~np.isfinite(tb)
    val += np.where(miss[:, None], env_lookup(m, nxt) * wb[:, None], 0.0)
    # a bounce that hits the black sphere: a Lambert vertex from outside (bounce draws, six environment draws, a shadow
    # ray when traced, then a bounce that leaves the convex sphere); nothing it adds is non-zero
    hit = ~miss
    p2 = o + nxt * np.where(hit, tb, 0)[:, None]
    n2 = (p2 - centre) / radius
    _x2, state2 = _draws(state, 2)
    e2, _ = _draws(state2, 6)
    l2, s2, _P2 = T.sample(e2)
    traced2 = ((l2 * n2).sum(1) > 0) & (s2 > 0)
    count += np.where(hit, traced2.astype(np.int64) + 1, 0)
    val *= np.pi

    assert rays == int(count.sum()), (rays, int(count.sum()))
    well = (np.abs(c) > 1e-4) & (s > 1e-4) & (ms > 1e-4) & (mb > 1e-4) & (edge > 1e-4) & ((np.abs((l2 * n2).sum(1)) > 1e-4) | miss)
    assert well.mean() > 0.9
    got = s4[:, :3]
    tol = 2e-3 * np.abs(val) + 2e-3 * np.abs(val).max(1, keepdims=True) + 1e-6
    bad = well[:, None] & (np.abs(got - val) > tol)
    assert not bad.any(), (int(bad.any(1).sum()), np.nonzero(bad.any(1))[0][:5])
    # the squares are the sample's
    assert np.allclose(q4[:, :3], got ** 2, rtol=1e-6, atol=0)
    # the features the replay is about are exercised
    assert traced.sum() > n // 4 and (traced & np.isfinite(ts)).sum() > 100 and hit.sum() > 500 and (wb < 0.99).sum() > 100


def test_replay_lambert_vertex_hit_from_inside(sctx, tables_lib):
    """Rays from inside a grey Lambert sphere meet it from inside: that vertex takes no environment sample (the pinned
    choice: its bounce is drawn about the outward normal while nl faces in), so its bounce keeps full weight and each
    sample traces exactly two rays."""
    m = random_map(32, 16, seed=9)
    radius = 2.0
    sph = np.zeros(1, SPHERE_DTYPE)
    sph[0] = ((0, 0, 0), radius, 1.0 / radius)
    mats = np.zeros(1, MATERIAL_DTYPE)
    mats[0]["albedo"] = (0.5, 0.25, 0.75)
    sctx.set_scene(sph, mats, F.furnace_camera(8, 8), np.zeros(0, np.int32))
    sctx.set_environment(m)
    sctx.set_option("environment_sampling", 1)
    rng = np.random.default_rng(8)
    n = 4096
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    rays = np.concatenate([np.zeros((n, 3)), d], 1).astype(np.float32)
    frame = 2
    s4, q4, count = _samples(sctx, rays, False, 1, frame)
    assert count == 2 * n
    normal = d                                           # hit at radius * d, outward normal d
    state = pixel_seed(np.arange(n, dtype=np.uint64), frame)
    x, _ = _draws(state, 2)
    b = normal + _unit(x[0], x[1])
    b /= np.linalg.norm(b, axis=1, keepdims=True)
    val = env_lookup(m, b) * np.array([0.5, 0.25, 0.75])
    tol = 2e-3 * np.abs(val).max(1, keepdims=True) + 1e-6
    assert (np.abs(s4[:, :3] - val) <= tol).mean() > 0.995


# ---- 2. unbiasedness ---------------------------------------------------------------------------------------------------
NORMALS = np.array([[0, 1, 0], [0, -1, 0], [1, 0, 0], [0, 0, -1], [0.6, 0.8, 0]] + [list(SUN_DIR)], np.float64)
NORMALS /= np.linalg.norm(NORMALS, axis=1, keepdims=True)


@pytest.fixture(scope="module")
def sun_1k():
    return sun_map(1024, 512)


@pytest.mark.parametrize("which", ["random", "sun"])
@pytest.mark.parametrize("on", [0, 1])
def test_irradiance_is_unbiased(sctx, sun_1k, which, on):
    m = random_map() if which == "random" else sun_1k
    sctx.set_scene(*far_scene()[:3], None)
    sctx.set_environment(m)
    sctx.set_option("environment_sampling", on)
    rep = 256
    pts = np.concatenate([np.zeros((len(NORMALS) * rep, 3)), np.repeat(NORMALS, rep, 0)], 1).astype(np.float32)
    spp = 4096
    s4, q4, _r = _samples(sctx, pts, True, spp, 1)
    S = s4.reshape(len(NORMALS), rep, 4).sum(1)
    Q = q4.reshape(len(NORMALS), rep, 4).sum(1)
    mean, se, _v = mean_se(S, Q)
    ref = irradiance_quadrature(m, NORMALS, sub=4 if which == "random" else 2)
    # the quadrature's own error (midpoint rule on sin theta cos, O(h^2)) is allowed for at 1e-4 relative
    z = (mean - ref) / np.maximum(se + 1e-4 * np.abs(ref) / 4.5, 1e-12)
    assert (np.abs(z) < 4.5).all(), (z, mean, ref, se)
    # trace_irradiance runs the same streams: its mean equals the sums'
    # (float32 sums in another order: the bound scales with the samples' magnitudes, which a sun hit makes large)
    E, _rays = sctx.trace_irradiance(pts, spp=spp, frame=1)
    tol = 2e-5 * np.abs(s4[:, :3]) / spp + 1e-5 * np.sqrt(q4[:, :3] * spp) / spp + 1e-6
    assert (np.abs(E[:, :3] - s4[:, :3] / spp) <= tol).all()


# ---- 3. efficiency ---------------------------------------------------------------------------------------------------
def simulate(T, normal, n, rng):
    """Per-sample values of the sampled estimator (and of the bounce alone) at a white point facing `normal` with
    nothing in view, in float64 with numpy's generator."""
    z = rng.uniform(-1, 1, n)
    a = rng.uniform(0, 2 * np.pi, n)
    r = np.sqrt(1 - z * z)
    b = normal + np.stack([r * np.cos(a), r * np.sin(a), z], -1)
    b /= np.linalg.norm(b, axis=1, keepdims=True)
    Lb = env_lookup(T.m, b)
    off = np.pi * Lb
    pe_b, _ = T.pdf(b)
    wb = _power(np.maximum(b @ normal, 0) / np.pi, pe_b)
    x = [rng.integers(0, 1 << 24, n, dtype=np.int64).astype(np.uint32) for _ in range(6)]
    l, s, P = T.sample(x)
    c = l @ normal
    ok = (c > 0) & (s > 0)
    pe = P * T.w * T.h / (2 * np.pi ** 2 * np.where(s > 0, s, 1))
    pb = c / np.pi
    with np.errstate(invalid="ignore", divide="ignore"):
        pend = np.where(ok, pb * pe / (pe * pe + pb * pb), 0.0)
    on = np.pi * (Lb * wb[:, None] + env_lookup(T.m, l) * pend[:, None])
    return off, on


def test_variance_matches_the_model_and_beats_the_bounce(sctx, tables_lib, sun_1k):
    T = EnvTables(tables_lib, sun_1k)
    normal = np.array([0.0, 1.0, 0.0])
    rng = np.random.default_rng(1)
    offs, ons = [], []
    for _ in range(4):
        o, s = simulate(T, normal, 1 << 20, rng)
        offs.append(o); ons.append(s)
    off, on = np.concatenate(offs), np.concatenate(ons)
    v_on_model = on.var(0, ddof=1).sum()
    v_off_model = off.var(0, ddof=1).sum()
    ratio = v_off_model / v_on_model
    print(f"sun map, horizontal receiver: model variance off {v_off_model:.4g}, on {v_on_model:.4g}, ratio {ratio:.4g}")
    assert ratio > 100

    sctx.set_scene(*far_scene()[:3], None)
    sctx.set_environment(sun_1k)
    sctx.set_option("environment_sampling", 1)
    rep = 1024
    pts = np.concatenate([np.zeros((rep, 3)), np.tile(normal, (rep, 1))], 1).astype(np.float32)
    s4, q4, _r = _samples(sctx, pts, True, 4096, 3)
    _m, _se, var = mean_se(s4.sum(0, keepdims=True), q4.sum(0, keepdims=True))
    v_gpu = var.sum()
    assert abs(v_gpu / v_on_model - 1) < 0.10, (v_gpu, v_on_model)


# ---- 4. whole scenes -------------------------------------------------------------------------------------------------
def _z(a4, aq, b4, bq):
    """z of the per-entry means; the floor on the standard error covers entries without variance (a caller ray that
    reaches the map through smooth metal), where the two sweep forms' float rounding is all that differs."""
    ma, sa, _ = mean_se(a4, aq)
    mb, sb, _ = mean_se(b4, bq)
    return (ma - mb) / (np.sqrt(sa ** 2 + sb ** 2) + 1e-5 * np.abs(mb) + 1e-7)


def _check_z(z, what):
    z = z[np.isfinite(z)]
    assert (np.abs(z) > 5).mean() <= 1e-3, (what, float((np.abs(z) > 5).mean()))
    assert abs(float(z.mean())) < 0.05, (what, float(z.mean()))


def test_reference_scene_on_and_off_agree(sctx):
    w, h, spp = 96, 54, 64
    s, mats, cam, em = scenes.reference_scene(w, h)
    sctx.set_scene(s, mats, cam, em)
    sctx.set_environment(scenes.sky_environment(512, 256))
    rays = scenes.camera_rays(cam, w, h)
    rng = np.random.default_rng(2)
    nrm = rng.normal(size=(3000, 3))
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    pts = np.concatenate([np.broadcast_to(cam["origin"][0], (3000, 3)), nrm], 1).astype(np.float32)
    res = {}
    for on in (0, 1):
        sctx.set_option("environment_sampling", on)
        (d4, dq), dr = sctx.draw_samples(0, w, h, spp=spp, sum4=np.zeros((w * h, 4), np.float32),
                                         sq4=np.zeros((w * h, 4), np.float32))
        r4, rq, rr = _samples(sctx, rays, False, spp, 0)
        p4, pq, pr = _samples(sctx, pts, True, spp, 0)
        res[on] = dict(draw=(d4.astype(np.float64), dq.astype(np.float64)), rays=(r4, rq), pts=(p4, pq))
        if on:
            assert dr > res[0]["draw_rays"] and rr > res[0]["rays_rays"]
            assert _sampling_only(sctx)
        res[on].update(draw_rays=dr, rays_rays=rr)
        # draws (variant 3 and auto, device and host buffers), trace_rays and trace_irradiance run the same streams
        sctx.set_spp(spp)
        mean_draw = (d4[:, :3] / d4[:, 3:4]).reshape(h, w, 3)
        for variant in (3, -1):
            sctx.set_option("fast_variant", variant)
            dev = torch.zeros((h, w, 4), dtype=torch.float32, device="cuda")
            r_dev = sctx.draw(0, 1, w, h, dev, flags=0, mode=MODE_FAST)
            host = np.zeros((h, w, 4), np.float32)
            r_host = sctx.draw(0, 1, w, h, host, flags=0, mode=MODE_FAST)
            assert r_dev == r_host == dr, (variant, r_dev, r_host, dr)
            assert rel_l2(dev.cpu().numpy(), mean_draw) < 1e-5
            assert rel_l2(host, mean_draw) < 1e-5
            if on:
                assert _sampling_only(sctx)
        sctx.set_option("fast_variant", -1)
        out, trr = sctx.trace_rays(rays, spp=spp)
        assert trr == rr and rel_l2(out, r4[:, :3] / spp) < 1e-5
        E, tpr = sctx.trace_irradiance(pts, spp=spp)
        assert tpr == pr and rel_l2(E, p4[:, :3] / spp) < 1e-5
    for k in ("draw", "rays", "pts"):
        _check_z(_z(*res[1][k], *res[0][k]), k)


def test_sun_map_sampling_on_is_closer_to_the_reference(sctx, sun_1k):
    w, h = 96, 54
    s, mats, cam, em = scenes.reference_scene(w, h)
    sctx.set_scene(s, mats, cam, em)
    sctx.set_environment(sun_1k)
    sctx.set_option("environment_sampling", 1)
    (r4, _q), _ = sctx.draw_samples(100, w, h, spp=4096, sum4=np.zeros((w * h, 4), np.float32))
    ref = r4[:, :3] / r4[:, 3:4]
    err = {}
    for on in (0, 1):
        sctx.set_option("environment_sampling", on)
        (d4, _q), _ = sctx.draw_samples(0, w, h, spp=16, sum4=np.zeros((w * h, 4), np.float32))
        err[on] = rel_l2(d4[:, :3] / d4[:, 3:4], ref)
    print(f"sun map, 16 spp: relative L2 off {err[0]:.4g}, on {err[1]:.4g}")
    assert err[1] < err[0]


# ---- 5. inactive is identical ----------------------------------------------------------------------------------------
def _outputs(ctx, w, h, rays):
    """One sample per entry, so that every output is a single sum (multi-sample atomic sums are not bitwise repeatable)."""
    ctx.set_spp(1)
    buf = torch.zeros((h, w, 4), dtype=torch.float32, device="cuda")
    r1 = ctx.draw(0, 1, w, h, buf, flags=0, mode=MODE_FAST)
    out, r2 = ctx.trace_rays(rays, spp=1)
    return [buf.cpu().numpy(), out], (r1, r2)


@pytest.mark.parametrize("case", ["no_map", "light_sampling_off", "black_map"])
def test_inactive_sampling_is_bitwise_off(sctx, case):
    w, h = 64, 36
    s, mats, cam, em = scenes.reference_scene(w, h)
    if case == "light_sampling_off":
        sctx.set_option("light_sampling", 0)
        sctx.set_environment(random_map())
    if case == "black_map":
        sctx.set_environment(np.zeros((16, 32, 3), np.float32))
    sctx.set_scene(s, mats, cam, em)
    rays = scenes.camera_rays(cam, w, h)
    ref, rref = _outputs(sctx, w, h, rays)
    sctx.set_option("environment_sampling", 1)
    got, rgot = _outputs(sctx, w, h, rays)
    assert rgot == rref
    for a, b in zip(got, ref):
        assert np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32))


# ---- 6. ordering, refusals, scope ------------------------------------------------------------------------------------
def test_a_map_set_during_a_sampled_draw_is_not_seen_by_it(sctx):
    w, h, spp = 1280, 720, 8
    s, mats, cam, em = scenes.reference_scene(w, h)
    sctx.set_scene(s, mats, cam, em)
    sctx.set_spp(spp)
    sctx.set_option("environment_sampling", 1)
    a, b = random_map(seed=1), random_map(seed=2) * 0.01
    bufs = [torch.zeros((h, w, 4), dtype=torch.float32, device="cuda") for _ in range(2)]
    torch.cuda.synchronize()
    sctx.set_environment(a)
    sctx.draw(0, 1, w, h, bufs[0], flags=0, mode=MODE_FAST, want_rays=False)
    sctx.set_environment(b)
    sctx.draw(0, 1, w, h, bufs[1], flags=0, mode=MODE_FAST, want_rays=False)
    torch.cuda.synchronize()
    got = [t.cpu().numpy() for t in bufs]
    refs = []
    for mp in (a, b):
        sctx.set_environment(mp)
        buf = torch.zeros((h, w, 4), dtype=torch.float32, device="cuda")
        sctx.draw(0, 1, w, h, buf, flags=0, mode=MODE_FAST)
        refs.append(buf.cpu().numpy())
    assert rel_l2(got[0], refs[0]) < 1e-5 and rel_l2(got[1], refs[1]) < 1e-5
    assert rel_l2(refs[1], refs[0]) > 0.1


def test_explicit_variants_are_refused_and_auto_runs_the_slab_queue(sctx):
    w, h = 64, 36
    s, mats, cam, em = scenes.reference_scene(w, h)
    sctx.set_scene(s, mats, cam, em)
    sctx.set_environment(random_map())
    sctx.set_option("environment_sampling", 1)
    buf = torch.zeros((h, w, 4), dtype=torch.float32, device="cuda")
    for v in (0, 1, 2, 4, 5, 6, 7, 8):
        sctx.set_option("fast_variant", v)
        with pytest.raises(TptError, match="environment_sampling"):
            sctx.draw(0, 1, w, h, buf, flags=0, mode=MODE_FAST)
    for v in (3, 9, -1):
        sctx.set_option("fast_variant", v)
        assert sctx.draw(0, 1, w, h, buf, flags=0, mode=MODE_FAST) > 0
        assert _sampling_only(sctx), (v, sctx.last_kernels())
        host = np.zeros((h, w, 4), np.float32)
        assert sctx.draw(0, 1, w, h, host, flags=0, mode=MODE_FAST) > 0
        assert _sampling_only(sctx), (v, sctx.last_kernels())
    # with the option off every variant runs again
    sctx.set_option("environment_sampling", 0)
    for v in (0, 8):
        sctx.set_option("fast_variant", v)
        assert sctx.draw(0, 1, w, h, buf, flags=0, mode=MODE_FAST) > 0


def test_aovs_and_parity_refusals_are_unchanged(sctx):
    w, h = 64, 36
    s, mats, cam, em = scenes.reference_scene(w, h)
    sctx.set_scene(s, mats, cam, em)
    rays = scenes.camera_rays(cam, w, h)
    sctx.set_environment(random_map())

    def aovs():
        alb, nrm, ids = (torch.zeros((h, w, 4), device="cuda"), torch.zeros((h, w, 4), device="cuda"),
                         torch.zeros((h, w), dtype=torch.int32, device="cuda"))
        r1 = sctx.draw_aovs(0, 1, w, h, alb, nrm, ids)
        (ra, rn, ri), r2 = sctx.trace_aovs(rays)
        return [t.cpu().numpy() for t in (alb, nrm, ids)] + [ra, rn, ri], (r1, r2)

    ref, rr = aovs()
    sctx.set_option("environment_sampling", 1)
    got, rg = aovs()
    assert rg == rr
    for a, b in zip(got, ref):
        assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))
    buf = torch.zeros((h, w, 4), dtype=torch.float32, device="cuda")
    for mode in (MODE_EXACT, MODE_REFGPU):
        with pytest.raises(TptError, match="only TPT_MODE_FAST draws use one"):
            sctx.draw(0, 1, w, h, buf, flags=0, mode=mode)


def test_option_is_accepted_and_boolean(sctx):
    for v in (0, 1, 7, -3):
        sctx.set_option("environment_sampling", v)
