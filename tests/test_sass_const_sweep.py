"""Sweep form 4 of the fast slab queue: the pair array of a scene of at most 64 padded spheres passed in a
__grid_constant__ kernel parameter, so that pass 1 reads the sphere values from the constant bank instead of shared memory.
The SASS claims are read off the shipped binary (no GPU); the GPU tests check that form 4 returns exactly what form 2
returns, ray by ray, at every padded count up to 64, and that the slab queue gives the same ray counts with either."""
import os, re, shutil, subprocess, sys
import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import sass_counts
LIB = os.path.join(ROOT, "toypathtracer_b200", "libtpt_b200.so")
have_sass = shutil.which("cuobjdump") is not None and shutil.which("cu++filt") is not None and os.path.exists(LIB)


def _sass_by_kernel():
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
    out, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = sass_counts.demangle(m.group(1))
            out[cur] = []
        elif cur and re.match(r"\s+/\*[0-9a-f]{4,}\*/", line):
            out[cur].append(line.split("*/", 1)[1].split(";")[0].strip())
    return out


@pytest.fixture(scope="module")
def sass():
    return _sass_by_kernel()


@pytest.mark.skipif(not have_sass, reason="needs cuobjdump and the built library")
@pytest.mark.parametrize("name", ["k_fast_queue<128, 6, 4>", "k_fast_queue<128, 8, 4>", "k_fast_queue_nolight<128, 6, 4>",
                                  "k_fast_rays<128, 6, 4>", "k_fast_rays_nolight<128, 8, 4>"])
def test_param_pair_sweep_reads_no_pair_array_from_shared_memory(sass, name):
    ins = sass[name]
    form2 = sass[name.replace(", 4", ", 2")]
    lds = lambda k: sum(1 for i in k if i.startswith("LDS.128"))
    # form 2's pass 1 is two LDS.128 per pair of spheres; form 4 keeps only pass 2's and the ray buffer's
    assert lds(form2) >= 128 and lds(ins) <= 16, (lds(form2), lds(ins))
    # ptxas (CUDA 12.9, sm_90a) moves the parameter's values into uniform registers (ULDC.64) and the FFMAs read them from
    # there: no vector register and no shared-memory load per value, but one uniform load per two values
    uniform_ffma = sum(1 for i in ins if re.match(r"FFMA\b", i) and re.search(r"\bUR\d+", i))
    assert uniform_ffma >= 384, uniform_ffma


# ---- GPU -------------------------------------------------------------------------------------------------------------
COUNTS = [1, 2, 3] + [p - (i % 4) for i, p in enumerate(range(4, 65, 4))] + [64]


@pytest.mark.gpu
@pytest.mark.parametrize("count", COUNTS)
def test_param_pair_form_matches_shared_pair_form(gpu_ctx, count):
    from test_gpu_fast import surface_rays
    from test_sweep_oracle import aimed_rays, degenerate_rays, make_scene, near_tangent_rays, pad_aimed_rays, tmin_rays
    sph, mats, cam, dup = make_scene(count, "compact")
    gpu_ctx.set_scene(sph, mats, cam, None)
    seed = 300 + count
    n = 3000
    surf = surface_rays(sph, 4 * n, seed)
    sets = {"surface": surf[np.isfinite(surf).all(1)], "tangent": near_tangent_rays(sph, n, seed + 1)[0],
            "tmin": tmin_rays(sph, n, seed + 2)[0], "degenerate": degenerate_rays(sph, seed + 3),
            "pad": pad_aimed_rays(max(16, n // 4), seed + 4), "aimed": aimed_rays(sph, seed + 5)[0]}
    for name, rays in sets.items():
        i2, t2 = gpu_ctx.debug_hit(2, rays)
        i4, t4 = gpu_ctx.debug_hit(4, rays)
        assert (i4 == i2).all(), (count, name, int((i4 != i2).sum()))
        assert (t4.view(np.uint32) == t2.view(np.uint32)).all(), (count, name)


@pytest.mark.gpu
def test_param_pair_form_refuses_larger_scenes(gpu_ctx):
    import toypathtracer_b200 as tpt
    from test_sweep_oracle import make_scene
    sph, mats, cam, dup = make_scene(65, "compact")
    gpu_ctx.set_scene(sph, mats, cam, None)
    with pytest.raises(tpt.TptError):
        gpu_ctx.debug_hit(4, np.array([[0, 6, 14, 0, 0, -1]], np.float32))


@pytest.mark.gpu
@pytest.mark.parametrize("variant", [3, 9])
def test_slab_queue_same_rays_with_either_pair_array(gpu_ctx, variant):
    """The reference scene (46 spheres) through the slab queue with the pair array in the kernel parameter (fast_kform 2)
    and in shared memory (fast_kform 3): the same hits, so the same paths; ray counts may differ only by the FMA
    contraction that differs between kernel instances."""
    import toypathtracer_b200 as tpt
    w, h = 320, 180
    gpu_ctx.set_scene(*tpt.reference_scene(w, h))
    gpu_ctx.set_option("fast_variant", variant)
    out = {}
    try:
        for k in (2, 3):
            gpu_ctx.set_option("fast_kform", k)
            img = np.zeros((h, w, 4), np.float32)
            rays = gpu_ctx.draw(0, 4, w, h, img, flags=tpt.kFlagProgressive, mode=tpt.MODE_FAST)
            out[k] = (rays, img)
    finally:
        gpu_ctx.set_option("fast_kform", 2)
        gpu_ctx.set_option("fast_variant", -1)
    assert abs(out[2][0] - out[3][0]) <= 1e-5 * out[3][0], (out[2][0], out[3][0])
    from conftest import rel_l2
    assert rel_l2(out[2][1][..., :3], out[3][1][..., :3]) < 1e-3
