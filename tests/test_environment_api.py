"""tpt_set_environment without a GPU: the library exports it, the Python binding declares the header's signature,
Context.set_environment refuses wrong shapes, dtypes and values before it reaches the library, and
scenes.sky_environment samples the reference sky at texel centres."""
import ctypes
import os
import re

import numpy as np
import pytest

from test_irradiance_api import _NoLib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_set_environment(libs):
    L = ctypes.CDLL(libs.LIB_PATH)
    assert hasattr(L, "tpt_set_environment")


def test_binding_matches_header_signature(libs):
    hdr = open(os.path.join(ROOT, "include", "tpt_b200.h")).read()
    m = re.search(r"int\s+tpt_set_environment\s*\(([^)]*)\)\s*;", hdr)
    assert m, "tpt_set_environment is not declared in include/tpt_b200.h"
    params = [" ".join(p.split()[:-1]) + ("*" if "*" in p.split()[-1] else "") for p in m.group(1).split(",")]
    assert params == ["tpt_context*", "const float*", "int", "int", "int"], params
    ctype = {"tpt_context*": ctypes.c_void_p, "const float*": ctypes.c_void_p, "int": ctypes.c_int}
    fn = libs._load_lib().tpt_set_environment
    assert [ctype[p] for p in params] == list(fn.argtypes)
    assert fn.restype is ctypes.c_int


@pytest.fixture
def fake_ctx(libs):
    ctx = libs.Context.__new__(libs.Context)
    ctx._L, ctx._h, ctx.device, ctx.spp = _NoLib(), ctypes.c_void_p(), 0, 4
    return ctx


def test_set_environment_refuses_before_the_library(libs, fake_ctx):
    good = np.ones((4, 8, 3), np.float32)
    nan, inf, neg = good.copy(), good.copy(), good.copy()
    nan[1, 2, 0] = np.nan
    inf[3, 7, 2] = np.inf
    neg[0, 0, 1] = -1e-30
    negzero = good.copy()
    negzero[2, 5, 2] = -0.0
    bad = [
        (np.ones((4, 8), np.float32), r"shape \(H, W, 3\) or \(H, W, 4\)"),
        (np.ones((4, 8, 2), np.float32), r"shape \(H, W, 3\) or \(H, W, 4\)"),
        (np.ones((2, 4, 8, 3), np.float32), r"shape \(H, W, 3\) or \(H, W, 4\)"),
        (good.astype(np.float64), "float32"),
        (good.astype(np.float16), "float32"),
        (nan, "finite and not negative"),
        (inf, "finite and not negative"),
        (neg, "finite and not negative"),
        (negzero, "finite and not negative"),
        ([[[1.0, 1.0, 1.0]]], "numpy array or a torch tensor"),
    ]
    for img, text in bad:
        with pytest.raises(libs.TptError, match=text):
            fake_ctx.set_environment(img)


def test_set_environment_refuses_torch_inputs_before_the_library(libs, fake_ctx):
    import torch
    good = torch.ones((4, 8, 4))
    with pytest.raises(libs.TptError, match="float32"):
        fake_ctx.set_environment(good.double())
    with pytest.raises(libs.TptError, match="shape"):
        fake_ctx.set_environment(torch.ones((4, 8, 5)))
    for v in (float("nan"), float("inf"), -2.0):
        t = good.clone()
        t[2, 3, 1] = v
        with pytest.raises(libs.TptError, match="finite and not negative"):
            fake_ctx.set_environment(t)


def test_alpha_is_not_checked(libs):
    """Alpha is ignored: a NaN there reaches the library (here a recording stand-in) with RGB padded to RGBA."""
    seen = {}

    class Rec:
        def tpt_set_environment(self, h, ptr, w, hgt, on_dev):
            seen.update(w=w, h=hgt, on_dev=on_dev,
                        data=np.ctypeslib.as_array(ctypes.cast(ptr, ctypes.POINTER(ctypes.c_float)), (hgt * w * 4,)).copy())
            return 0

    ctx = libs.Context.__new__(libs.Context)
    ctx._L, ctx._h, ctx.device, ctx.spp = Rec(), ctypes.c_void_p(), 0, 4
    img = np.arange(2 * 3 * 4, dtype=np.float32).reshape(2, 3, 4)
    img[..., 3] = np.nan
    ctx.set_environment(img)
    assert (seen["w"], seen["h"], seen["on_dev"]) == (3, 2, 0)
    assert np.array_equal(seen["data"].reshape(2, 3, 4)[..., :3], img[..., :3])
    rgb = np.arange(2 * 3 * 3, dtype=np.float32).reshape(2, 3, 3)
    ctx.set_environment(rgb)
    assert np.array_equal(seen["data"].reshape(2, 3, 4)[..., :3], rgb)


def test_sky_environment_samples_the_gradient_at_texel_centres(libs):
    from toypathtracer_b200 import scenes
    w, h = 16, 9
    env = scenes.sky_environment(w, h)
    assert env.shape == (h, w, 3) and env.dtype == np.float32 and env.flags["C_CONTIGUOUS"]
    for j in range(h):
        theta = (j + 0.5) / h * np.pi
        y = np.cos(theta)
        t = 0.5 * (y + 1.0)
        want = ((1.0 - t) * np.ones(3) + t * np.array([0.5, 0.7, 1.0])) * 0.3
        for i in range(w):
            np.testing.assert_allclose(env[j, i], want, rtol=1e-7, atol=0)
    # row 0 is the zenith (bluer, t near 1), the last row the nadir (whiter)
    assert env[0, 0, 2] > env[0, 0, 0] and env[-1, 0, 0] > env[0, 0, 0]
    np.testing.assert_allclose(env[0, 0], np.float32([0.15, 0.21, 0.3]), rtol=1e-2)


def test_environment_oracle_is_exact_on_constant_maps_and_continuous_across_the_seam():
    """The float64 oracle of the GPU tests: a constant map returns its constant, columns wrap across phi = +-pi, rows
    clamp at the poles, and the centre column lies along -z."""
    from test_gpu_environment import env_lookup, lat_long_dir
    c = np.float32([0.15, 0.21, 0.3])
    rng = np.random.default_rng(1)
    d = rng.normal(size=(200, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    const = np.broadcast_to(c, (5, 7, 3))
    assert np.array_equal(env_lookup(const, d), np.broadcast_to(c.astype(np.float64), (200, 3)))
    m = rng.random((6, 10, 3))
    eps = 1e-9
    a = env_lookup(m, np.array([[np.sin(np.pi - eps), 0.3, -np.cos(np.pi - eps)]]))
    b = env_lookup(m, np.array([[np.sin(-np.pi + eps), 0.3, -np.cos(-np.pi + eps)]]))
    np.testing.assert_allclose(a, b, atol=1e-7)
    # at a texel centre the oracle returns that texel
    for (i, j) in [(0, 0), (9, 5), (4, 2), (5, 3)]:
        np.testing.assert_allclose(env_lookup(m, lat_long_dir(i + 0.5, j + 0.5, 10, 6)[None])[0], m[j, i], atol=1e-12)
    np.testing.assert_allclose(lat_long_dir(5.0, 3.0, 10, 6), [0, 0, -1], atol=1e-12)
    # both poles: the whole first / last row at once, blended across its columns only
    np.testing.assert_allclose(env_lookup(m, np.array([[0.0, 1.0, 0.0]]))[0], 0.5 * (m[0, 0] + m[0, 9]), atol=1e-12)
