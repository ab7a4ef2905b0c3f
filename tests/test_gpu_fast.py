"""Fast (throughput) mode: per-path RNG streams, so parity with the reference is statistical. The bar is the
measured Monte-Carlo noise floor of the reference itself (SURVEY §9.3: two independent N-spp reference renders
differ by relL2 ~= 0.194/sqrt(N)); a biased estimator would sit far above it and would not shrink with N."""
import numpy as np
import pytest

from conftest import rel_l2
from test_oracle import golden_scene

pytestmark = pytest.mark.gpu

W, H = 640, 360
VARIANTS = (0, 1, 3, 4, 5, 6, 8, 9)


@pytest.fixture(scope="module")
def ref64(oracle):
    """64 spp of the restatement (== reference, tests/test_oracle.py) + an independent 64 spp (frames 16..31)."""
    sph, mats, cam, em = golden_scene()
    a, ra, _ = oracle.orc_render(sph, mats, cam, W, H, 0, 16, flags=2)
    b, rb, _ = oracle.orc_render(sph, mats, cam, W, H, 16, 16, flags=2)
    return a, sum(ra), b, sum(rb)


@pytest.mark.parametrize("variant", VARIANTS)
def test_statistical_parity(gpu_ctx, ref64, variant):
    a, ra, b, rb = ref64
    floor = rel_l2(b, a)                       # reference vs itself with other seeds: the noise floor at 64 spp
    sph, mats, cam, em = golden_scene()
    gpu_ctx.set_scene(sph, mats, cam, em)
    gpu_ctx.set_option("fast_variant", variant)
    img = np.zeros((H, W, 4), np.float32)
    rays = gpu_ctx.draw(0, 16, W, H, img, flags=2, mode=1)
    assert np.isfinite(img).all()
    r = rel_l2(img, a)
    assert r < 1.25 * floor, f"relL2 {r:.4e} vs noise floor {floor:.4e}"
    # rays per primary sample: reference 4.5616 (SURVEY §9.8); independent reference runs agree to ~3e-4
    rps, rps_ref = rays / (W * H * 64), ra / (W * H * 64)
    assert abs(rps / rps_ref - 1) < 2e-3
    # no colour bias: channel means agree within 3 sigma of the reference's own run-to-run difference + 0.2 %
    ma, mb, mi = (x[..., :3].reshape(-1, 3).astype(np.float64).mean(0) for x in (a, b, img))
    tol = 3 * np.abs(ma - mb) + 2e-3 * ma
    assert (np.abs(mi - ma) < tol).all(), (mi, ma, tol)


@pytest.mark.parametrize("variant", VARIANTS)
def test_error_shrinks_like_monte_carlo(gpu_ctx, ref64, variant):
    """relL2 against a 1024-spp fast render must fall ~ 1/sqrt(N): bias would flatten it."""
    sph, mats, cam, em = golden_scene()
    gpu_ctx.set_scene(sph, mats, cam, em)
    gpu_ctx.set_option("fast_variant", variant)
    hi = np.zeros((H, W, 4), np.float32)
    gpu_ctx.draw(0, 256, W, H, hi, flags=2, mode=1)     # progressive mean of frames 0..255 = 1024 spp
    a = ref64[0]
    r_ref = rel_l2(a, hi)                                   # reference@64 vs fast@1024
    assert r_ref < 1.2 * 0.194 / 8 * np.sqrt(1 + 64 / 1024)
    lo = np.zeros((H, W, 4), np.float32)
    gpu_ctx.draw(0, 4, W, H, lo, flags=2, mode=1)           # 16 spp (a subset of hi's samples: factor sqrt(1-16/1024))
    r16 = rel_l2(lo, hi)
    assert 0.7 < r16 / (0.194 / 4) < 1.3


def same_sample_draws(ctx, light_sampling):
    """{variant: (image, rays)} of variants 0-9: golden scene, 640x360, spp 1, fast_kform 0, 64 progressive frames in one
    draw. At spp 1 variant 0's stream per pixel and frame is every other variant's stream per sample, and with fast_kform 0
    every variant sweeps in the reference form."""
    sph, mats, cam, em = golden_scene()
    out = {}
    try:
        ctx.set_option("light_sampling", light_sampling)
        ctx.set_option("fast_kform", 0)
        ctx.set_spp(1)
        ctx.set_scene(sph, mats, cam, em)
        for v in range(10):
            ctx.set_option("fast_variant", v)
            img = np.zeros((H, W, 4), np.float32)
            out[v] = (img, ctx.draw(0, 64, W, H, img, flags=2, mode=1))
    finally:
        ctx.set_spp(4)
        for k, val in (("light_sampling", 1), ("fast_kform", 2), ("fast_variant", 3)):
            ctx.set_option(k, val)
    return out


@pytest.mark.parametrize("light_sampling", (1, 0))
def test_variants_trace_the_same_samples(gpu_ctx, light_sampling):
    """Every variant shades with path_step, so on the same streams and sweep form they trace the same paths: only FMA
    contraction, which differs between kernel instances, can flip a decision now and then. Measured against variant 3 on
    an H100 80GB HBM3 (700 W): relL2 <= 1.4e-7 and equal ray counts for every variant, light sampling on and off. The
    bars, 2e-6 and 1e-7, are ~14x the image figure and about 5 rays in the 5e7 of a draw. Copies of the estimator that
    draw or weigh samples differently land above the image bar: measured 8.3e-6 (and 5.3e-8 more rays without light
    sampling) for a wavefront with its own copy of the shading, 8.8e-4 for one with its own light-cone basis, 2e-2 and
    4e-5 fewer rays for variants 0-2 with their own light and roughness sampling."""
    out = same_sample_draws(gpu_ctx, light_sampling)
    ref, ref_rays = out[3]
    for v, (img, rays) in out.items():
        assert rel_l2(img, ref) <= 2e-6, (v, rel_l2(img, ref))
        assert abs(rays / ref_rays - 1) <= 1e-7, (v, rays, ref_rays)


def test_variants_and_sharding_consistent(gpu_ctx):
    """Packed interleaved bands (multi-GPU layout) give the same image as a full draw: the RNG stream depends on
    the pixel, not on which rank/launch renders it (variant 1)."""
    sph, mats, cam, em = golden_scene()
    gpu_ctx.set_scene(sph, mats, cam, em)
    gpu_ctx.set_option("fast_variant", 3)
    full = np.zeros((H, W, 4), np.float32)
    total = gpu_ctx.draw(0, 2, W, H, full, flags=2, mode=1)
    img = np.zeros((H, W, 4), np.float32)
    r = 0
    for rank in range(2):
        band = np.zeros((H // 2, W, 4), np.float32)
        r += gpu_ctx.draw(0, 2, W, H, band, flags=2, mode=1, rows=(rank, H // 2, 2, 1))
        img[rank::2] = band
    assert r == total
    assert rel_l2(img, full) < 1e-5      # same streams; only the smem accumulation order may differ


def test_progressive_accumulation_matches_single_call(gpu_ctx):
    sph, mats, cam, em = golden_scene()
    gpu_ctx.set_scene(sph, mats, cam, em)
    gpu_ctx.set_option("fast_variant", 3)
    one = np.zeros((H, W, 4), np.float32)
    gpu_ctx.draw(0, 8, W, H, one, flags=2, mode=1)
    seq = np.zeros((H, W, 4), np.float32)
    for f in range(8):
        gpu_ctx.draw(f, 1, W, H, seq, flags=2, mode=1)
    assert rel_l2(seq, one) < 1e-5


def test_tonemap(gpu_ctx):
    img = np.zeros((4, 8, 4), np.float32)
    img[0, :, 0] = np.linspace(0, 1, 8); img[3, :, 1] = 2.0
    out = gpu_ctx.tonemap_srgb8(img, 8, 4)
    ref = np.clip(np.maximum(1.055 * np.power(np.maximum(img[::-1, :, :3], 0), 0.416666667) - 0.055, 0), 0, 1) * 255 + 0.5
    assert np.abs(out[..., :3].astype(np.int32) - ref.astype(np.int32)).max() <= 1
    assert (out[..., 3] == 255).all()


def test_tonemap_other_shells_conversions(gpu_ctx):
    """The WebAssembly shell's sqrt gamma with Y flip (Emscripten/main.cpp:67-79) and the C# TGA writer's BGR
    LinearToSRGB with its 255.9 truncation (Cs/Program.cs:34-68), against numpy restatements of those lines."""
    rng = np.random.default_rng(5)
    img = (rng.random((9, 16, 4), dtype=np.float32) * 1.6).astype(np.float32)
    img[0, 0, :3] = (0.0, 1.0, 4.0)
    out = gpu_ctx.tonemap_rgba8(img, 16, 9, transfer=1, bgr=False, flip_y=True)
    ref = np.minimum(np.sqrt(img[::-1, :, :3]) * np.float32(255), np.float32(255.0)).astype(np.uint8)
    assert (out[..., :3] == ref).all() and (out[..., 3] == 255).all()
    out = gpu_ctx.tonemap_rgba8(img, 16, 9, transfer=2, bgr=True, flip_y=False)
    x = np.maximum(img[..., :3], 0)
    x = np.maximum(np.float32(1.055) * np.power(x, np.float32(0.416666667)) - np.float32(0.055), 0).astype(np.float32)
    ref = np.minimum((x * np.float32(255.9)).astype(np.uint32), 255).astype(np.int32)[..., ::-1]
    assert np.abs(out[..., :3].astype(np.int32) - ref).max() <= 1          # __powf vs powf: at most one code at a truncation edge
    assert (np.abs(out[..., :3].astype(np.int32) - ref) != 0).mean() < 0.02


def test_host_band_pipelining_equals_single_launch(gpu_ctx):
    """Host-buffer draws overlap the D2H with tracing, either (a) with ONE kernel that publishes per-band completion
    counters the copy stream waits on (cuStreamWaitValue32, `host_progress`), or (b) with one launch per row band on its
    own stream (`host_bands`). Both must give the image of the plain draw (same per-pixel streams; only the order of the
    L2 reductions differs) — and the progress path must never copy a band before its last path has landed."""
    sph, mats, cam, em = golden_scene()
    gpu_ctx.set_scene(sph, mats, cam, em)
    gpu_ctx.set_option("fast_variant", 3)
    outs = []
    for (progress, pbands, bands) in [(0, 8, 1), (0, 8, 4), (0, 8, 7), (1, 1, 3), (1, 8, 3), (1, 16, 3)]:
        gpu_ctx.set_option("host_progress", progress)
        gpu_ctx.set_option("progress_bands", pbands)
        gpu_ctx.set_option("host_bands", bands)
        for rep in range(3):                       # repeat: a too-early copy would be a race, not a constant error
            img = np.full((H, W, 4), 0.25, np.float32)
            rays = gpu_ctx.draw(5, 2, W, H, img, flags=2, mode=1)
            outs.append((img, rays))
    gpu_ctx.set_option("host_progress", 1); gpu_ctx.set_option("progress_bands", 4); gpu_ctx.set_option("host_bands", 3)
    for img, rays in outs[1:]:
        assert rays == outs[0][1]
        assert rel_l2(img, outs[0][0]) < 1e-5
        assert (img[..., 3] == np.float32(0.25)).all()      # progressive: alpha preserved


def test_expanded_form_sweep_matches_reference_form(gpu_ctx):
    """The fast kernels' 8-slot expanded-form discriminant (FastHitterK) against the reference-form sweep on the SAME
    per-path RNG streams: paths only differ where a rounding flips a hit decision, so the two images must agree far
    below the Monte-Carlo noise (which would be ~2.4e-2 at 64 spp) and the ray counts within 1e-4."""
    sph, mats, cam, em = golden_scene()
    gpu_ctx.set_scene(sph, mats, cam, em)
    gpu_ctx.set_option("fast_variant", 3)
    out = []
    for k in (2, 1, 0):
        gpu_ctx.set_option("fast_kform", k)
        img = np.zeros((H, W, 4), np.float32)
        rays = gpu_ctx.draw(0, 16, W, H, img, flags=2, mode=1)
        out.append((img, rays))
    gpu_ctx.set_option("fast_kform", 2)
    # the pair array's two chains evaluate the scalar expanded form's products — the sweeps are bit-identical ray by ray (test
    # below); the kernels still differ in a handful of decisions per 10^7 rays (measured: 10 of 67 M) because the shading
    # code around the sweep is contracted differently (-fmad) in each template instance
    assert abs(out[0][1] / out[1][1] - 1) < 5e-6 and rel_l2(out[0][0], out[1][0]) < 1e-3
    assert abs(out[1][1] / out[2][1] - 1) < 1e-4
    assert rel_l2(out[1][0], out[2][0]) < 3e-3


def surface_rays(spheres, n, seed):
    """Rays a path tracer produces, the hard ones over-represented: origins on sphere surfaces (a third on the ground
    sphere, sphere 0), a fifth at the camera position; directions mostly leaving the surface, some entering it
    (refraction), a fifth grazing. Returns float32 [n, 6] = {o.xyz, d.xyz}."""
    rng = np.random.default_rng(seed)
    raw = np.asarray(spheres).view(np.float32).reshape(-1, 5).astype(np.float64)     # {centre.xyz, radius, invRadius}
    c, r = raw[:, :3], raw[:, 3]
    pick = rng.integers(0, len(r), n)
    pick[: n // 3] = 0
    nrm = rng.normal(size=(n, 3)); nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    g = pick == 0
    xz = rng.uniform(-40, 40, (n, 2))
    top = np.stack([xz[:, 0], np.sqrt(r[0] ** 2 - xz[:, 0] ** 2 - xz[:, 1] ** 2), xz[:, 1]], 1) / r[0]
    nrm[g] = top[g]
    o = c[pick] + nrm * r[pick, None]
    d = rng.normal(size=(n, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
    flip = ((d * nrm).sum(1) < 0) & (rng.random(n) < 0.8)
    d[flip] = -d[flip]
    graze = rng.random(n) < 0.2
    d[graze] = d[graze] - 0.98 * (d[graze] * nrm[graze]).sum(1, keepdims=True) * nrm[graze]
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    cam = rng.random(n) < 0.2
    o[cam] = np.array([0, 6, 14.0]) + rng.normal(size=(int(cam.sum()), 3)) * 0.02
    return np.concatenate([o, d], 1).astype(np.float32)


def same_hits(a, b):
    return (a[0] == b[0]).all() and (a[1].view(np.uint32) == b[1].view(np.uint32)).all()


def test_sweep_forms_ray_by_ray(gpu_ctx, libs):
    """tpt_debug_hit: the nearest-hit query of each sweep form on 2 M rays. The pair-array form must return the
    scalar expanded form's ids and distance BITS; the conservative form (packed pass 1 with the error bound folded in +
    reference-form pass 2) must return the reference-form sweep's, on the reference scene and on the 4096-sphere scene
    that fails the expanded form's accuracy gate."""
    sph, mats, cam, em = golden_scene()
    gpu_ctx.set_scene(sph, mats, cam, em)
    rays = surface_rays(sph, 2_000_000, 11)
    res = {k: gpu_ctx.debug_hit(k, rays) for k in (0, 1, 2, 3)}
    assert 0.2 < (res[0][0] >= 0).mean() < 0.8
    assert same_hits(res[1], res[2])
    assert same_hits(res[0], res[3])
    assert (res[0][0] != res[1][0]).mean() < 2e-2          # the expanded form itself: other rounding, mostly at grazing self-hits
    s2 = libs.stress_scene(1920, 1080, count=4096)
    gpu_ctx.set_scene(s2[0], s2[1], s2[2], None)
    rays = surface_rays(s2[0], 2_000_000, 12)
    ref = gpu_ctx.debug_hit(0, rays)
    assert 0.2 < (ref[0] >= 0).mean() < 0.8
    assert same_hits(ref, gpu_ctx.debug_hit(3, rays))
    assert same_hits(gpu_ctx.debug_hit(1, rays), gpu_ctx.debug_hit(2, rays))


def test_fast_odd_sizes_all_variants(gpu_ctx):
    """Ragged shapes in the throughput kernels (tile / slab tails): finite image, sane rays per sample, every pixel hit."""
    import toypathtracer_b200 as tpt
    sph, mats, cam0, em = golden_scene()
    for (w, h) in [(97, 53), (257, 3), (1, 130)]:
        cam = tpt.make_camera((0, 2, 3), (0, 0, 0), (0, 1, 0), 60, w / h, 0.02, 3)
        gpu_ctx.set_scene(sph, mats, cam, em)
        for variant in VARIANTS:
            gpu_ctx.set_option("fast_variant", variant)
            img = np.full((h, w, 4), -1.0, np.float32)
            rays = gpu_ctx.draw(0, 2, w, h, img, flags=0, mode=1)
            assert np.isfinite(img).all() and (img[..., :3] >= 0).all(), (w, h, variant)
            assert (img[..., :3].sum(axis=2) > 0).all(), (w, h, variant)      # sky/ground everywhere: no pixel skipped
            assert 1.0 <= rays / (w * h * 4) < 12.0
    gpu_ctx.set_option("fast_variant", 3)


def test_more_than_256_frames_in_one_call(gpu_ctx):
    """Fast mode fuses at most 256 frames per launch; longer accumulations are chained launches with the same result as
    two explicit calls."""
    sph, mats, cam, em = golden_scene()
    gpu_ctx.set_scene(sph, mats, cam, em)
    gpu_ctx.set_option("fast_variant", 3)
    w, h = 96, 54
    one = np.zeros((h, w, 4), np.float32)
    r1 = gpu_ctx.draw(0, 300, w, h, one, flags=2, mode=1)
    two = np.zeros((h, w, 4), np.float32)
    r2 = gpu_ctx.draw(0, 256, w, h, two, flags=2, mode=1) + gpu_ctx.draw(256, 44, w, h, two, flags=2, mode=1)
    assert r1 == r2 and rel_l2(one, two) < 1e-5


def test_zero_copy_host_write_out(gpu_ctx):
    """Variant 8 stores finished pixels straight into a page-locked host buffer (coalesced 128-bit stores over PCIe, no
    staging image, no D2H copy); pageable buffers and progressive draws take the staged path. All must agree."""
    import torch
    sph, mats, cam, em = golden_scene()
    gpu_ctx.set_scene(sph, mats, cam, em)
    gpu_ctx.set_option("fast_variant", 8)
    try:
        ref = np.zeros((H, W, 4), np.float32)                                   # pageable: staged path
        rays_ref = gpu_ctx.draw(7, 1, W, H, ref, flags=0, mode=1)
        pinned = torch.full((H, W, 4), 3.0, dtype=torch.float32).pin_memory().numpy()
        for rep in range(3):
            pinned[...] = 3.0
            rays = gpu_ctx.draw(7, 1, W, H, pinned, flags=0, mode=1)             # zero-copy
            assert rays == rays_ref
            assert rel_l2(pinned, ref) < 1e-5 and (pinned[..., 3] == 0).all()
        gpu_ctx.set_option("host_zero_copy", 0)
        pinned[...] = 3.0
        assert gpu_ctx.draw(7, 1, W, H, pinned, flags=0, mode=1) == rays_ref
        assert rel_l2(pinned, ref) < 1e-5
        gpu_ctx.set_option("host_zero_copy", 1)
        # a row shard of a pinned full-size buffer: only those rows are written
        pinned[...] = 3.0
        gpu_ctx.draw(7, 1, W, H, pinned, flags=0, mode=1, rows=(2, 50, 3, 0))
        mine = np.zeros(H, bool); mine[2:152:3] = True
        assert (pinned[~mine] == 3.0).all() and rel_l2(pinned[mine], ref[mine]) < 1e-5
        # progressive (prev has weight): staged path, alpha preserved
        pinned[...] = 0.0; pinned[..., 3] = 0.5
        seq = np.zeros((H, W, 4), np.float32); seq[..., 3] = 0.5
        for f in range(1, 4):                                   # frame 0 has lerpFac 0: prev would have no weight
            gpu_ctx.draw(f, 1, W, H, pinned, flags=2, mode=1)
            gpu_ctx.draw(f, 1, W, H, seq, flags=2, mode=1)
        assert rel_l2(pinned, seq) < 1e-5 and (pinned[..., 3] == 0.5).all()
        # default options ("fast_variant" -1 = auto): a pinned host buffer takes the zero-copy kernel (1 trace launch + the
        # ray-count fold), a device buffer the slab queue (prepare + trace + fold)
        import toypathtracer_b200 as tpt
        ctx2 = tpt.Context(0)
        ctx2.set_scene(sph, mats, cam, em)
        pinned[...] = 3.0
        assert ctx2.draw(7, 1, W, H, pinned, flags=0, mode=1) == rays_ref and ctx2.last_launch_count() == 2
        assert rel_l2(pinned, ref) < 1e-5
        dev = torch.zeros((H, W, 4), dtype=torch.float32, device="cuda")
        # the slab queue is a different kernel: same per-path RNG streams, but its shading code is compiled (FMA-contracted)
        # on its own, so a handful of paths in millions may take a different branch
        rays_dev = ctx2.draw(7, 1, W, H, dev, flags=0, mode=1)
        assert abs(rays_dev - rays_ref) <= 2e-5 * rays_ref and ctx2.last_launch_count() == 3
        ctx2.close()
    finally:
        gpu_ctx.set_option("fast_variant", 3)
