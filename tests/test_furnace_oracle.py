"""The furnace scenes' closed-form answers (tests/furnace.py) checked against the CPU restatements before they judge any
kernel: scene A bit for bit with exact ray counts, scenes B1-B5 statistically, and the quadrature behind them."""
import os

import numpy as np
import pytest

import furnace as F


@pytest.fixture(scope="module")
def oracles(oracle):
    """name -> (render function, light sampling on): the CPU path's and the GPU shader's restatements, each also
    compiled with DO_LIGHT_SAMPLING 0."""
    from oracle import nolight
    if not (os.path.exists(nolight.pyoracle.ORC_SO) and os.path.exists(nolight.pyoracle.RGO_SO)):
        nolight.build()
    return {"orc": (oracle.orc_render, True), "rgo": (oracle.rgo_render, True),
            "orc_nolight": (nolight.pyoracle.orc_render, False), "rgo_nolight": (nolight.pyoracle.rgo_render, False)}


def _render(fn, s, m, c, w, h, f0, n, flags, spp, mitsuba, buf):
    out = fn(s, m, c, w, h, f0, n, flags=flags, spp=spp, mitsuba=mitsuba, buf=buf)
    return out[0], out[1]


@pytest.mark.parametrize("K,metal", [(0, False), (3, False), (40, False), (255, False), (256, False), (300, False),
                                     (5, True)])
@pytest.mark.parametrize("which", ["orc", "rgo", "orc_nolight", "rgo_nolight"])
def test_furnace_a_is_exact_in_every_restatement(oracles, which, K, metal):
    """Every sample is albedo * sky: the pixel is the closed-form blend within a quarter of one sample's weight, and
    every frame traces exactly w*h*spp*(2 + K) rays (2 for Metal or without light sampling). The CPU path never writes
    alpha; the GPU shader's restatement writes 1."""
    fn, ls = oracles[which]
    w, h, spp = 48, 40, 3
    s, m, c, em = F.furnace_scene(w, h, K, metal)
    v = F.furnace_value(m)
    rng = np.random.default_rng(K)
    for f0, n, flags in ((0, 3, 2), (4, 2, 2), (2, 2, 0), (3, 3, 3)):
        prev = rng.uniform(0, 1, (h, w, 4)).astype(np.float32)
        buf, rays = _render(fn, s, m, c, w, h, f0, n, flags, spp, True, prev.copy())
        exp, tol = F.furnace_expect(prev[..., :3], v, f0, n, flags, spp)
        err = np.abs(buf[..., :3] - exp)
        assert (err <= tol).all(), (which, K, f0, flags, float((err / tol).max()))
        assert rays == [w * h * spp * F.furnace_rays_per_sample(m, K, ls)] * n, (which, K, rays)
        alpha = np.ones((h, w), np.float32) if which.startswith("rgo") else prev[..., 3]
        assert np.array_equal(buf[..., 3], alpha)


def test_furnace_tolerance_sees_one_sample():
    """The bar is a quarter of one sample: a pixel missing one of its samples (the rest of its frame's mean unchanged) is
    off by 4 tolerances, at the heaviest and the lightest frame weight."""
    v = np.array([0.12, 0.126, 0.12], np.float64)
    for f0, n, flags, spp in ((0, 257, 2, 1), (3, 5, 2, 7), (0, 1, 0, 4), (2, 5, 0, 3), (3, 4, 3, 2)):
        W, w = F.frame_weights(f0, n, flags)
        assert abs(W + w.sum() - 1) < 1e-12
        exp, tol = F.furnace_expect(np.zeros(3), v, f0, n, flags, spp)
        lost = exp - v * w[w > 0].min() / spp
        assert (np.abs(lost - exp) > 3.9 * tol).all()


def test_light_phi_matches_cone_quadrature():
    """Phi = cos(beta) sin^2(alpha) against a float64 Gauss-Legendre integral of max(0, n.w)/pi over the cone."""
    rng = np.random.default_rng(3)
    xs, ws = np.polynomial.legendre.leggauss(48)
    for _ in range(20):
        n = rng.normal(size=3); n /= np.linalg.norm(n)
        axis = rng.normal(size=3); axis /= np.linalg.norm(axis)
        if axis.dot(n) < 0.2:
            axis = axis + 2 * n; axis /= np.linalg.norm(axis)
        dist = rng.uniform(0.8, 3.0)
        r = dist * rng.uniform(0.02, 0.95) * axis.dot(n)           # sin(alpha) < cos(beta): wholly above the horizon
        sin2a = r * r / dist ** 2
        phi = F.light_phi(np.zeros((1, 3)), n[None], axis * dist, r)[0]
        cosmax = np.sqrt(1 - sin2a)
        u = np.cross(axis, [1.0, 0, 0] if abs(axis[0]) < 0.9 else [0, 1.0, 0]); u /= np.linalg.norm(u)
        vv = np.cross(axis, u)
        ct = cosmax + (1 - cosmax) * 0.5 * (xs + 1)            # cos(theta) over [cos alpha, 1]
        ph = np.pi * (xs + 1)                                 # azimuth over [0, 2 pi)
        CT, PH = np.meshgrid(ct, ph, indexing="ij")
        ST = np.sqrt(1 - CT ** 2)
        d = CT[..., None] * axis + ST[..., None] * (np.cos(PH)[..., None] * u + np.sin(PH)[..., None] * vv)
        integ = np.maximum(d @ n, 0) * np.outer(ws * 0.5 * (1 - cosmax), ws * np.pi)
        assert abs(integ.sum() / np.pi - phi) < 1e-10 * max(phi, 1e-3), (phi, integ.sum() / np.pi)


def test_cosine_lobe_mean_is_two_thirds_n():
    """The mean direction of the cosine lobe about n is (2/3) n (float64 quadrature of cos-weighted directions)."""
    xs, ws = np.polynomial.legendre.leggauss(32)
    ct = 0.5 * (xs + 1)                                        # cos(theta) in [0, 1]
    ph = np.pi * (xs + 1)
    CT, PH = np.meshgrid(ct, ph, indexing="ij")
    W = np.outer(ws * 0.5, ws * np.pi) * CT / np.pi             # pdf cos/pi over the hemisphere
    ST = np.sqrt(1 - CT ** 2)
    mean = np.array([(W * ST * np.cos(PH)).sum(), (W * ST * np.sin(PH)).sum(), (W * CT).sum()])
    assert abs(W.sum() - 1) < 1e-13
    assert np.allclose(mean, [0, 0, 2 / 3], atol=1e-13)


def test_b_expectations_resolve_the_footprint():
    """The per-pixel quadrature has converged (4x4 vs 8x8 nodes), and the B1 lights matter (Phi up to a few percent)."""
    for scene, expect in ((F.b1_scene, F.b1_expect), (F.b2_scene, F.b2_expect)):
        s, m, c, em = scene(40, 24)
        e4, e8 = expect(s, m, c, 40, 24), expect(s, m, c, 40, 24, nq=8)
        assert np.abs(e4 - e8).max() < 1e-12
    # B3's lobe quadrature at the roughest setting (a singular corner where refl + r u can vanish) and B4's chain
    s, m, c, em = F.b3_scene(40, 24, 1.0)
    e32, e48 = F.b3_expect(s, m, c, 40, 24)[0], F.b3_expect(s, m, c, 40, 24, n=48)[0]
    assert np.abs(e32 - e48).max() < 2e-5 * e32.mean()
    s, m, c, em = F.b4_scene(40, 24)
    assert np.abs(F.b4_expect(s, m, c, 40, 24)[0] - F.b4_expect(s, m, c, 40, 24, nq=8)[0]).max() < 1e-9
    s, m, c, em = F.b1_scene(40, 24)
    e = F.b1_expect(s, m, c, 40, 24)
    flat = m["albedo"][0] * F.MITSUBA_SKY
    assert (e / flat).min() > 1.3 and np.ptp(e[..., 0]) > 0.05 * e[..., 0].mean()


def batch_means(render, w, h, batches, frames):
    """[batches, h, w, 3] independent per-pixel means: batch b = frames [b*frames, (b+1)*frames) drawn progressively
    into a zero buffer, divided by their combined weight."""
    out = []
    for b in range(batches):
        buf = np.zeros((h, w, 4), np.float32)
        render(buf, b * frames, frames)
        W, _ = F.frame_weights(b * frames, frames, 2)
        out.append(buf[..., :3].astype(np.float64) / (1.0 - W))
    return np.array(out)


B_PAIRS = ([(sc, wh) for sc in F.B_SCENES if sc != "b1_nols" for wh in ("orc", "rgo")]
           + [("b1_nols", "orc_nolight"), ("b1_nols", "rgo_nolight")])


@pytest.mark.parametrize("scene,which", B_PAIRS)
def test_b_expectations_match_restatements(oracles, which, scene):
    """16 batches of 16 frames x 16 spp (4096 spp), every bin of >= 1 000 pixels within max(5 se, 1e-4 E) of the analytic
    expectation. B1: light sampling on and off converge to the same E (the restatements built without it run "b1_nols";
    the scenes without lights run once per estimator). B4 takes the CPU path's rules for "orc" and the GPU shader's
    saturating Schlick and shorter depth limit for "rgo"; the two expectations differ by up to 4.5e-3 relative."""
    fn, _ls = oracles[which]
    s, m, c, em, w, h, e, bins, mitsuba, _ = F.b_case(scene, "gpu" if which.startswith("rgo") else "cpu")
    B = batch_means(lambda buf, f0, n: fn(s, m, c, w, h, f0, n, flags=2, spp=16, mitsuba=mitsuba, buf=buf),
                    w, h, 16, 16)
    assert min((bins == b).sum() for b in range(bins.max() + 1)) >= 1000
    F.check_bins(B, e, bins)
