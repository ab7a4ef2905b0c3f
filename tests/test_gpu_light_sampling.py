"""The runtime DO_LIGHT_SAMPLING switch (option "light_sampling" = 0) on the GPU: exact and reference-GPU strict modes
bitwise against the restatements with the switch off and the reference compiled with it off; fast mode statistically
against exact mode with the switch off; the option's scene semantics."""
import numpy as np
import pytest

from conftest import bits_differ, rel_l2
from test_gpu_configs import CLASS_NAMES, ExactPair, first_hit_classes, rl2
from test_light_sampling import assert_matches_nolight_render, oracle_nl  # noqa: F401  (oracle_nl: fixture)
from test_oracle import golden_scene

pytestmark = pytest.mark.gpu

LANES = (0, 1, 2, 8, 9, 32, 64, 65, 66, 67, 70, 71)


@pytest.fixture
def nolight(gpu_ctx):
    gpu_ctx.set_option("light_sampling", 0)
    yield gpu_ctx
    for k, v in (("light_sampling", 1), ("exact_lanes", 0), ("exact_lookahead", 0), ("fast_variant", 3), ("fast_kform", 2)):
        gpu_ctx.set_option(k, v)


def test_exact_mode_without_light_sampling_bitwise(nolight, libs, oracle, oracle_nl):
    ctx = nolight
    w, h = 200, 120
    sph, mats, cam, em = libs.reference_scene(w, h)
    ctx.set_scene(sph, mats, cam, em)
    for flags in (0, 2, 3):
        obuf, orays, pads = oracle_nl.orc_render(sph, mats, cam, w, h, 0, 3, flags=flags)
        if flags != 3:
            assert_matches_nolight_render(f"nolight_{w}x{h}_f0_n3_flags{flags}", obuf, orays)
        live = oracle.have_ref_variant("nolight") and flags != 3
        if live:
            rbuf, rrays = oracle.ref_render(w, h, 0, 3, flags=flags, variant="nolight")
        for lanes in LANES:
            ctx.set_option("exact_lanes", lanes)
            buf = np.zeros((h, w, 4), np.float32)
            total, pf = ctx.draw(0, 3, w, h, buf, flags=flags, mode=0, per_frame=True)
            assert pf == orays, (flags, lanes)
            assert not bits_differ(buf, obuf, pads).any(), (flags, lanes)
            if live:
                assert pf == rrays and not bits_differ(buf, rbuf, pads).any(), (flags, lanes)
        # a strided row shard
        ctx.set_option("exact_lanes", 0)
        band = np.zeros((h, w, 4), np.float32)
        ctx.draw(0, 3, w, h, band, flags=flags, mode=0, rows=(1, h // 4, 4, 0))
        assert not bits_differ(band[1::4], obuf[1::4], [(x, (y - 1) // 4) for (x, y, _f) in pads if y % 4 == 1]).any()


def test_exact_mode_without_light_sampling_720p(nolight, libs):
    w, h = 1280, 720
    sph, mats, cam, em = libs.reference_scene(w, h)
    nolight.set_scene(sph, mats, cam, em)
    buf = np.zeros((h, w, 4), np.float32)
    total, pf = nolight.draw(0, 3, w, h, buf, flags=0, mode=0, per_frame=True)
    assert_matches_nolight_render("nolight_1280x720_f0_n3_flags0", buf, pf)


@pytest.mark.parametrize("lookahead", [4, -1])
def test_lookahead_cache_does_not_serve_frames_of_the_other_setting(gpu_ctx, libs, oracle, oracle_nl, lookahead):
    w, h = 200, 120
    sph, mats, cam, em = libs.reference_scene(w, h)
    ref_mix = np.zeros((h, w, 4), np.float32)
    _, r1, p1 = oracle.orc_render(sph, mats, cam, w, h, 0, 3, flags=2, buf=ref_mix)
    _, r2, p2 = oracle_nl.orc_render(sph, mats, cam, w, h, 3, 3, flags=2, buf=ref_mix)
    gpu_ctx.set_option("exact_lookahead", lookahead)
    try:
        buf = np.zeros((h, w, 4), np.float32)
        rays = []
        for f in range(6):
            if f == 3:
                gpu_ctx.set_option("light_sampling", 0)
            gpu_ctx.set_scene(sph, mats, cam, em)          # a shell's UpdateTest: every frame
            rays.append(gpu_ctx.draw(f, 1, w, h, buf, flags=2, mode=0))
        assert rays == r1 + r2
        assert not bits_differ(buf, ref_mix, p1 + p2).any()
    finally:
        gpu_ctx.set_option("exact_lookahead", 0)
        gpu_ctx.set_option("light_sampling", 1)


def test_dropin_shim_without_light_sampling(libs):
    w, h = 320, 180
    libs.set_light_sampling(False)
    try:
        libs.InitializeTest()
        libs.set_mode(libs.MODE_EXACT)
        buf = np.zeros((h, w, 4), np.float32)
        rays = []
        for f in range(3):
            libs.UpdateTest(0.0, f, w, h, 2)
            rays.append(libs.DrawTest(0.0, f, w, h, buf, 2))
        assert_matches_nolight_render(f"nolight_{w}x{h}_f0_n3_flags2", buf, rays)
        libs.ShutdownTest()
    finally:
        libs.set_light_sampling(True)


def test_refgpu_strict_without_light_sampling(nolight, libs, oracle_nl):
    """The cases of test_gpu_modes.test_refgpu_strict_equals_cpu_restatement with the switch off."""
    ctx = nolight
    sph, mats, cam, em = golden_scene()
    s9 = libs.reference_scene(320, 180, big_scene=False, mitsuba_compare=True)
    s203 = libs.stress_scene(160, 90, count=203)
    cam_odd = libs.make_camera((0, 2, 3), (0, 0, 0), (0, 1, 0), 60, 97 / 53, 0.02, 3)
    cases = [(sph, mats, cam, 320, 180, False), (s9[0], s9[1], s9[2], 320, 180, True),
             (s203[0], s203[1], s203[2], 160, 90, False), (sph, mats, cam_odd, 97, 53, False)]
    try:
        for (s, m, c, w, h, mitsuba) in cases:
            ctx.set_option("mitsuba_compare", 1 if mitsuba else 0)
            ctx.set_scene(s, m, c, None)
            for flags, f0 in ((0, 5), (2, 0), (3, 2)):
                init = np.full((h, w, 4), 0.25, np.float32)
                obuf, orays = oracle_nl.rgo_render(s, m, c, w, h, f0, 3, flags=flags, mitsuba=mitsuba, buf=init.copy())
                buf = init.copy()
                total, pf = ctx.draw(f0, 3, w, h, buf, flags=flags, mode=libs.MODE_REFGPU, per_frame=True)
                assert total == sum(orays), (len(s), flags)
                assert not bits_differ(buf, obuf).any(), (len(s), flags)
    finally:
        ctx.set_option("mitsuba_compare", 0)


def check_fast_against_exact_nolight(ctx, ex, sph, mats, cam, w, h, frames, label, rl2_bar=1.10, class_rl2=True):
    """The bars of test_gpu_configs.check_fast_against_exact without its noise model (that one is the light-sampled
    estimator's): relL2 <= 1.10 x the exact-vs-exact floor, <= 1.15 x per first-hit class, region means within
    max(6 sigma, 2e-4), rays per sample within 3e-3 of exact mode's."""
    F = np.zeros((h, w, 4), np.float32)
    frays = ctx.draw(0, frames, w, h, F, flags=2, mode=1)
    assert np.isfinite(F).all(), label
    F = F.astype(np.float64)[..., :3]
    floor, r = rl2(ex.B, ex.A), rl2(F, ex.A)
    assert r <= rl2_bar * floor, (label, r, floor)
    assert abs(frays / frames / ex.rays_per_frame - 1) < 3e-3, (label, frays / frames, ex.rays_per_frame)
    cls = first_hit_classes(sph, mats, cam, w, h)
    for k, name in enumerate(CLASS_NAMES):
        m = cls == k
        n = int(m.sum())
        if n < 200:
            continue
        fm, fl = rl2(F, ex.A, m), rl2(ex.B, ex.A, m)
        assert not class_rl2 or fm <= 1.15 * fl + 2e-5, (label, name, fm, fl)
        mean_f, mean_c = F[m].mean(axis=0), ex.C[m].mean(axis=0)
        se = np.sqrt(ex.var_px[m].sum(axis=0) * 1.5) / n
        assert (np.abs(mean_f - mean_c) <= np.maximum(6 * se, 2e-4 * mean_c)).all(), (label, name, mean_f, mean_c, se)


def exact_pair(ctx, w, h, frames):
    ex = ExactPair(ctx, w, h, frames)
    n = min(frames, 64)
    ex.rays_per_frame = ctx.draw(0, n, w, h, np.zeros((h, w, 4), np.float32), flags=2, mode=0) / n
    return ex


@pytest.fixture(scope="module")
def exact_16k_nolight(gpu_ctx, libs):
    w, h = 640, 360
    sph, mats, cam, em = libs.reference_scene(w, h)
    gpu_ctx.set_option("light_sampling", 0)
    try:
        gpu_ctx.set_scene(sph, mats, cam, em)
        return exact_pair(gpu_ctx, w, h, 4096), (sph, mats, cam, em)
    finally:
        gpu_ctx.set_option("light_sampling", 1)


@pytest.mark.parametrize("variant,kform", [(3, 2), (3, 1), (3, 0), (8, 2), (8, 0), (5, 2), (7, 2)])
def test_fast_without_light_sampling_converges_to_exact(nolight, exact_16k_nolight, variant, kform):
    ex, (sph, mats, cam, em) = exact_16k_nolight
    nolight.set_scene(sph, mats, cam, em)
    nolight.set_option("fast_variant", variant)
    nolight.set_option("fast_kform", kform)
    check_fast_against_exact_nolight(nolight, ex, sph, mats, cam, 640, 360, 4096, f"nolight v{variant} kform{kform}")


def test_fast_without_light_sampling_conservative_instance(nolight, libs):
    """The 4096-sphere stress scene fails the expanded-form gate: variant 3 runs the 768-thread KFORM 3 instance. 160x90
    at 4096 spp. Without light sampling the per-pixel distribution is heavy-tailed (rare direct hits of the small lights)
    and 14 400 pixels do not average the outliers out: relL2 ratios then depend on the sample realisation. Measured on
    an H100 at this size: fast/exact relL2 over the exact-vs-exact floor 1.19 for variants 1, 3, 5 and 8 (which share
    their per-path streams), 1.00 for variant 0 (other streams), with every region mean within 1e-3 relative. So this
    size asserts the bias bars and rays per sample as in the 640x360 test, and relL2 <= 1.25 x floor overall."""
    w, h = 160, 90
    sph, mats, cam, em = libs.stress_scene(w, h, count=4096)
    nolight.set_scene(sph, mats, cam, em)
    ex = exact_pair(nolight, w, h, 1024)
    nolight.set_option("fast_variant", 3)
    check_fast_against_exact_nolight(nolight, ex, sph, mats, cam, w, h, 1024, "nolight stress4096 v3", rl2_bar=1.25, class_rl2=False)


@pytest.mark.parametrize("variant", [0, 1, 2, 4, 6, 9])
def test_fast_variants_without_light_sampling(nolight, libs, oracle_nl, variant):
    """The cheaper check of test_gpu_modes: 256 spp against the restatement with the switch off."""
    w, h = 320, 180
    sph, mats, cam, em = libs.reference_scene(w, h)
    nolight.set_scene(sph, mats, cam, em)
    obuf, orays, _ = oracle_nl.orc_render(sph, mats, cam, w, h, 0, 64, flags=2)
    o2 = obuf.copy()
    oracle_nl.orc_render(sph, mats, cam, w, h, 64, 64, flags=2, buf=o2)
    floor = rel_l2(2.0 * o2.astype(np.float64) - obuf, obuf)
    nolight.set_option("fast_variant", variant)
    fb = np.zeros((h, w, 4), np.float32)
    frays = nolight.draw(0, 64, w, h, fb, flags=2, mode=1)
    assert rel_l2(fb, obuf) < 1.15 * floor, variant
    assert abs(frays / sum(orays) - 1) < 3e-3, variant


def test_option_is_a_scene_flag(gpu_ctx, libs):
    """Applied by the next set_scene only; toggling re-uploads the same bytes; light-sampled draws after toggling back
    are bit-identical to draws that never toggled."""
    w, h = 160, 90
    sph, mats, cam, em = libs.reference_scene(w, h)
    gpu_ctx.set_scene(sph, mats, cam, em)
    a = np.zeros((h, w, 4), np.float32)
    ra = gpu_ctx.draw(0, 2, w, h, a, flags=2, mode=0)
    try:
        gpu_ctx.set_option("light_sampling", 0)
        b = np.zeros((h, w, 4), np.float32)
        assert gpu_ctx.draw(0, 2, w, h, b, flags=2, mode=0) == ra and not bits_differ(a, b).any()   # not applied yet
        gpu_ctx.set_scene(sph, mats, cam, em)
        size = gpu_ctx.last_scene_upload_bytes()
        assert size > 0
        c = np.zeros((h, w, 4), np.float32)
        rc = gpu_ctx.draw(0, 2, w, h, c, flags=2, mode=0)
        assert rc < ra and bits_differ(a, c).any()
        gpu_ctx.set_option("light_sampling", 1)
        gpu_ctx.set_scene(sph, mats, cam, em)
        assert gpu_ctx.last_scene_upload_bytes() == size
        d = np.zeros((h, w, 4), np.float32)
        assert gpu_ctx.draw(0, 2, w, h, d, flags=2, mode=0) == ra and not bits_differ(a, d).any()
    finally:
        gpu_ctx.set_option("light_sampling", 1)
