"""tpt_draw's host-side branches that no image test tells apart: which kernels a banded host-buffer draw launches, a
buffer page-locked by "register_host", the automatic variant on the 4096-sphere scene, and the reference-GPU modes'
launch counts. Expected trace kernels come from test_gpu_mirror_chains.image_instances, the restatement of the
launchers' pick rules."""
import numpy as np
import pytest
import torch

from conftest import bits_differ, rel_l2
from test_gpu_mirror_chains import image_instances
from test_oracle import golden_scene

pytestmark = pytest.mark.gpu

W, H = 640, 360


def _instance(mode, a, sph, em, kopt=2, ls=True):
    s = np.ascontiguousarray(sph).view(np.float32).reshape(-1, 5).astype(np.float64)    # {center, radius, invRadius}
    gate = bool(((s[:, :3] ** 2).sum(axis=1) <= 128.0 + 2.0 * s[:, 3] ** 2).all())     # tpt_set_scene's kformOk
    return image_instances(mode, a, len(sph), len(em) if ls else 0, kopt, gate, ls)


@pytest.fixture
def dctx(libs):
    """A context of its own: "register_host" keeps a buffer page-locked until the context is destroyed."""
    ctx = libs.Context(0)
    yield ctx
    ctx.close()


# (fast_variant, host_progress): a variant with progress counters draws ONE kernel whose bands the copy stream follows;
# with host_progress 0, or a variant without counters, every one of the 3 row bands gets its own launch sequence
# (variants 3/4/6/7/9: prepare + trace, 5: trace). Variants 0/1/2/8 are not banded.
BANDED = [(3, 1, 1, 2), (9, 1, 1, 2), (3, 0, 3, 6), (4, 0, 3, 6), (5, 1, 3, 3), (6, 1, 3, 6), (7, 0, 3, 6), (8, 1, 1, 1),
          (0, 1, 1, 1), (2, 1, 1, 1)]


@pytest.mark.parametrize("variant,progress,kernels,launches", BANDED, ids=[f"v{v}-p{p}" for v, p, _, _ in BANDED])
def test_banded_host_draw_kernels(dctx, variant, progress, kernels, launches):
    sph, mats, cam, em = golden_scene()
    dctx.set_scene(sph, mats, cam, em)
    dctx.set_option("fast_variant", variant)
    dctx.set_option("host_progress", progress)
    dctx.set_option("host_bands", 3)
    img = np.full((H, W, 4), 0.25, np.float32)
    rays = dctx.draw(5, 2, W, H, img, flags=2, mode=1)
    assert dctx.last_kernels() == [_instance("fast", variant, sph, em)] * kernels
    assert dctx.last_launch_count() == launches + 1           # + the ray-count fold
    dev = torch.full((H, W, 4), 0.25, dtype=torch.float32, device="cuda")
    assert dctx.draw(5, 2, W, H, dev, flags=2, mode=1) == rays
    assert rel_l2(img, dev.cpu().numpy()) < 1e-5 and (img[..., 3] == np.float32(0.25)).all()


def test_register_host(dctx):
    """A pageable buffer page-locked and mapped by "register_host": the automatic variant then stores straight into it
    (variant 8, one trace launch), only the drawn rows change, and an exact-mode draw through it keeps its bits."""
    sph, mats, cam, em = golden_scene()
    dctx.set_scene(sph, mats, cam, em)
    ref, buf = np.zeros((H, W, 4), np.float32), np.full((H, W, 4), 3.0, np.float32)
    plain = np.full((90, 160, 4), 0.5, np.float32)
    other = plain.copy()
    try:
        _register_host(dctx, sph, em, ref, buf, plain, other)
    finally:
        dctx.close()                                              # unregisters: the buffers must outlive it


def _register_host(dctx, sph, em, ref, buf, plain, other):
    dctx.set_option("fast_variant", 8)
    rays_ref = dctx.draw(7, 1, W, H, ref, flags=0, mode=1)       # pageable: staged
    dctx.set_option("fast_variant", -1)
    dctx.set_option("register_host", 1)
    for rep in range(2):
        buf[...] = 3.0
        assert dctx.draw(7, 1, W, H, buf, flags=0, mode=1) == rays_ref
        assert dctx.last_kernels() == [_instance("fast", 8, sph, em)] and dctx.last_launch_count() == 2
        assert rel_l2(buf, ref) < 1e-5 and (buf[..., 3] == 0).all()
    buf[...] = 3.0
    dctx.draw(7, 1, W, H, buf, flags=0, mode=1, rows=(2, 50, 3, 0))
    mine = np.zeros(H, bool); mine[2:152:3] = True
    assert (buf[~mine] == 3.0).all() and rel_l2(buf[mine], ref[mine]) < 1e-5
    dctx.set_option("register_host", 0)
    dctx.draw(3, 2, 160, 90, plain, flags=2, mode=0)
    dctx.set_option("register_host", 1)                           # a second buffer: registration moves to it
    dctx.draw(3, 2, 160, 90, other, flags=2, mode=0)
    assert not bits_differ(other, plain).any()


@pytest.mark.parametrize("kform", [1, 2])
def test_auto_variant_on_4096_spheres(gpu_ctx, libs, kform):
    """From 1024 spheres the automatic variant is the block wavefront (7) where the slab queue cannot run a packed-pair
    sweep ("fast_kform" 1 here), else the slab queue (3)."""
    w, h = 320, 180
    sph, mats, cam, em = libs.stress_scene(w, h, count=4096)
    gpu_ctx.set_scene(sph, mats, cam, em)
    gpu_ctx.set_option("fast_variant", -1)
    gpu_ctx.set_option("fast_kform", kform)
    try:
        dev = torch.zeros((h, w, 4), dtype=torch.float32, device="cuda")
        assert gpu_ctx.draw(0, 1, w, h, dev, flags=0, mode=1) > 0
        assert gpu_ctx.last_kernels() == [_instance("fast", 7 if kform == 1 else 3, sph, em, kopt=kform)]
        assert gpu_ctx.last_launch_count() == 3
    finally:
        gpu_ctx.set_option("fast_kform", 2)


@pytest.mark.parametrize("mode,name", [(2, "refgpu"), (3, "refgpu_native")])
@pytest.mark.parametrize("frames", [1, 3])
def test_refgpu_launch_counts(gpu_ctx, mode, name, frames):
    """The reference-GPU modes trace all frames of a draw in one launch, then fold the ray counts."""
    sph, mats, cam, em = golden_scene()
    gpu_ctx.set_scene(sph, mats, cam, em)
    for buf in (np.zeros((90, 160, 4), np.float32), torch.zeros((90, 160, 4), dtype=torch.float32, device="cuda")):
        assert gpu_ctx.draw(0, frames, 160, 90, buf, flags=2, mode=mode) > 0
        assert gpu_ctx.last_kernels() == [_instance(name, 0, sph, em)]
        assert gpu_ctx.last_launch_count() == 2
