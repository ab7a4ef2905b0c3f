"""Sweep form 5 on the GPU: the half-precision pass 1 (FastHitterKH) that the slab queue's form-4 kernels run for scenes build_half_pairs accepts (fast_kform 2; fast_kform 4 keeps the FP32 pass 1). Through tpt_debug_hit, form 5
returns the ids and distance bits of forms 2 and 4 at every padded count from 4 to 64 on the sweep oracle's ray sets and
on rays outside the bound (the warp's FP32 fallback); scenes outside the half range are refused the form; draws and
caller rays trace the same paths with either pass 1, with light sampling on and off, in the same kernel instance."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

COUNTS = [p - (i % 4) for i, p in enumerate(range(4, 65, 4))] + [64]


def _rays(sph, count, n=2500):
    from test_gpu_fast import surface_rays
    from test_sweep_oracle import aimed_rays, degenerate_rays, near_tangent_rays, pad_aimed_rays, tmin_rays
    seed = 700 + count
    surf = surface_rays(sph, 4 * n, seed)
    rng = np.random.default_rng(seed)
    far = np.concatenate([rng.uniform(-40, 40, (n, 3)), rng.normal(size=(n, 3))], 1)
    far[:, 3:] /= np.linalg.norm(far[:, 3:], axis=1, keepdims=True)
    mixed = surf[:n].copy()
    mixed[::7, :3] *= 5.0                  # one lane in seven outside |o| <= 16: whole warps fall back to FP32
    return {"surface": surf[np.isfinite(surf).all(1)], "tangent": near_tangent_rays(sph, n, seed + 1)[0],
            "tmin": tmin_rays(sph, n, seed + 2)[0], "degenerate": degenerate_rays(sph, seed + 3),
            "pad": pad_aimed_rays(max(16, n // 4), seed + 4), "aimed": aimed_rays(sph, seed + 5)[0],
            "far": far.astype(np.float32), "mixed": mixed[np.isfinite(mixed).all(1)]}


@pytest.mark.parametrize("count", COUNTS)
def test_half_pass_matches_fp32_forms(gpu_ctx, count):
    from test_sweep_oracle import make_scene
    sph, mats, cam, dup = make_scene(count, "compact")
    gpu_ctx.set_scene(sph, mats, cam, None)
    for name, rays in _rays(sph, count).items():
        i2, t2 = gpu_ctx.debug_hit(2, rays)
        i4, t4 = gpu_ctx.debug_hit(4, rays)
        i5, t5 = gpu_ctx.debug_hit(5, rays)
        assert (i4 == i2).all() and (i5 == i2).all(), (count, name, int((i5 != i2).sum()))
        assert (t5.view(np.uint32) == t2.view(np.uint32)).all(), (count, name)
        assert (t4.view(np.uint32) == t2.view(np.uint32)).all(), (count, name)
        if dup >= 0 and name == "aimed":
            assert not (i5 == dup + 1).any()          # the lower id of the exact duplicate pair wins


def test_half_pass_on_the_reference_scene(gpu_ctx):
    import toypathtracer_b200 as tpt
    from toypathtracer_b200 import scenes
    sp, mats, cam, em = tpt.reference_scene(1280, 720)
    gpu_ctx.set_scene(sp, mats, cam, em)
    rays = scenes.camera_rays(cam, 1280, 720, 1, seed=11)[::7]
    sets = {"camera": rays}
    i2, t2 = gpu_ctx.debug_hit(2, rays)
    hit = i2 >= 0
    # secondary rays from the first hits in random directions
    rng = np.random.default_rng(12)
    p = rays[hit, :3] + t2[hit, None] * rays[hit, 3:]
    d = rng.normal(size=p.shape)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    sets["bounce"] = np.concatenate([p, d], 1).astype(np.float32)
    for name, r in sets.items():
        a2, b2 = gpu_ctx.debug_hit(2, r)
        a5, b5 = gpu_ctx.debug_hit(5, r)
        assert (a5 == a2).all() and (b5.view(np.uint32) == b2.view(np.uint32)).all(), name


def test_scenes_outside_the_half_range_are_refused(gpu_ctx):
    import toypathtracer_b200 as tpt
    from test_sweep_oracle import make_scene
    for count, layout in ((40, "spread"), (65, "compact")):
        sph, mats, cam, dup = make_scene(count, layout)
        gpu_ctx.set_scene(sph, mats, cam, None)
        with pytest.raises(tpt.TptError):
            gpu_ctx.debug_hit(5, np.array([[0, 6, 14, 0, 0, -1]], np.float32))


@pytest.mark.parametrize("ls", [1, 0])
def test_draws_and_caller_rays_trace_the_same_paths(gpu_ctx, ls):
    """The reference scene with the half pass 1 (fast_kform 2) and without it (fast_kform 4): the same kernel instance
    (Context.last_kernels), the same hits, so the same paths and ray counts."""
    import toypathtracer_b200 as tpt
    from toypathtracer_b200 import scenes
    from conftest import rel_l2
    w, h = 320, 180
    sp, mats, cam, em = tpt.reference_scene(w, h)
    gpu_ctx.set_option("light_sampling", ls)
    gpu_ctx.set_scene(sp, mats, cam, em)
    rays = scenes.camera_rays(cam, w, h, 1, seed=5)
    out = {}
    try:
        for k in (2, 4):
            gpu_ctx.set_option("fast_kform", k)
            img = np.zeros((h, w, 4), np.float32)
            n = gpu_ctx.draw(0, 4, w, h, img, flags=tpt.kFlagProgressive, mode=tpt.MODE_FAST)
            kd = gpu_ctx.last_kernels()
            res, nr = gpu_ctx.trace_rays(rays, spp=4)
            kr = gpu_ctx.last_kernels()
            out[k] = (n, img, kd, nr, res, kr)
    finally:
        gpu_ctx.set_option("fast_kform", 2)
        gpu_ctx.set_option("light_sampling", 1)
    suffix = "" if ls else "_nolight"
    assert out[2][2] == out[4][2] == [f"k_fast_queue{suffix}<128, 6, 4>"], (out[2][2], out[4][2])
    assert out[2][5] == out[4][5] == [f"k_fast_rays{suffix}<128, 6, 4>"], (out[2][5], out[4][5])
    assert out[2][0] == out[4][0] and out[2][3] == out[4][3]
    assert rel_l2(out[2][1][..., :3], out[4][1][..., :3]) < 1e-6
    assert rel_l2(out[2][4][:, :3], out[4][4][:, :3]) < 1e-6
