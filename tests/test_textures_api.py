"""tpt_set_textures without a GPU: the library exports it, the Python binding declares the header's signature, and
Context.set_textures refuses wrong shapes, dtypes, texel values and sphere layers before it reaches the library."""
import ctypes
import os
import re

import numpy as np
import pytest

from test_irradiance_api import _NoLib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_set_textures(libs):
    L = ctypes.CDLL(libs.LIB_PATH)
    assert hasattr(L, "tpt_set_textures")


def test_binding_matches_header_signature(libs):
    hdr = open(os.path.join(ROOT, "include", "tpt_b200.h")).read()
    m = re.search(r"int\s+tpt_set_textures\s*\(([^)]*)\)\s*;", hdr)
    assert m, "tpt_set_textures is not declared in include/tpt_b200.h"
    params = [" ".join(p.split()[:-1]) + ("*" if "*" in p.split()[-1] else "") for p in m.group(1).split(",")]
    assert params == ["tpt_context*", "const float*", "int", "int", "int", "const int*", "int", "int"], params
    ctype = {"tpt_context*": ctypes.c_void_p, "const float*": ctypes.c_void_p, "const int*": ctypes.c_void_p,
             "int": ctypes.c_int}
    fn = libs._load_lib().tpt_set_textures
    assert [ctype[p] for p in params] == list(fn.argtypes)
    assert fn.restype is ctypes.c_int


@pytest.fixture
def fake_ctx(libs):
    ctx = libs.Context.__new__(libs.Context)
    ctx._L, ctx._h, ctx.device, ctx.spp = _NoLib(), ctypes.c_void_p(), 0, 4
    return ctx


def test_set_textures_refuses_bad_textures_before_the_library(libs, fake_ctx):
    good = np.ones((2, 4, 8, 3), np.float32)
    layers = np.array([0, 1, -1], np.int32)
    nan, inf, neg, negzero = good.copy(), good.copy(), good.copy(), good.copy()
    nan[1, 1, 2, 0] = np.nan
    inf[0, 3, 7, 2] = np.inf
    neg[1, 0, 0, 1] = -1e-30
    negzero[0, 2, 5, 2] = -0.0
    shape_text = r"shape \(L, H, W, 3\) or \(L, H, W, 4\)"
    bad = [
        (np.ones((4, 8, 3), np.float32), shape_text),
        (np.ones((2, 4, 8, 2), np.float32), shape_text),
        (np.ones((2, 4, 8, 5), np.float32), shape_text),
        (np.ones((1, 2, 4, 8, 3), np.float32), shape_text),
        (np.ones((0, 4, 8, 3), np.float32), shape_text),
        (np.ones((2, 0, 8, 3), np.float32), shape_text),
        (good.astype(np.float64), "float32"),
        (good.astype(np.float16), "float32"),
        (nan, "finite and not negative"),
        (inf, "finite and not negative"),
        (neg, "finite and not negative"),
        (negzero, "finite and not negative"),
        ([[[[1.0, 1.0, 1.0]]]], "numpy array or a torch tensor"),
    ]
    for tex, text in bad:
        with pytest.raises(libs.TptError, match=text):
            fake_ctx.set_textures(tex, layers)


def test_set_textures_refuses_bad_sphere_layers_before_the_library(libs, fake_ctx):
    good = np.ones((2, 4, 8, 4), np.float32)
    for layers, text in (([0, 2], r"sphere_layers\[1\] = 2 is outside \[-1, 2\)"),
                         ([-2, 0], r"sphere_layers\[0\] = -2 is outside \[-1, 2\)"),
                         ([0, 1, 1 << 40], r"sphere_layers\[2\] = 1099511627776 is outside"),
                         (np.zeros((2, 2), np.int32), "1-D integer array"),
                         (np.zeros(3, np.float32), "1-D integer array"),
                         (np.zeros(3, bool), "1-D integer array"),
                         (None, "sphere_layers is required")):
        with pytest.raises(libs.TptError, match=text):
            fake_ctx.set_textures(good, layers)


def test_set_textures_refuses_torch_inputs_before_the_library(libs, fake_ctx):
    import torch
    good = torch.ones((2, 4, 8, 4))
    layers = torch.tensor([0, 1])
    with pytest.raises(libs.TptError, match="float32"):
        fake_ctx.set_textures(good.double(), layers)
    with pytest.raises(libs.TptError, match="shape"):
        fake_ctx.set_textures(torch.ones((2, 4, 8, 5)), layers)
    with pytest.raises(libs.TptError, match="outside"):
        fake_ctx.set_textures(good, torch.tensor([0, 3]))
    for v in (float("nan"), float("inf"), -2.0, -0.0):
        t = good.clone()
        t[1, 2, 3, 1] = v
        with pytest.raises(libs.TptError, match="finite and not negative"):
            fake_ctx.set_textures(t, layers)


def test_textures_reach_the_library_as_rgba_with_alpha_unchecked(libs):
    """Alpha is ignored: a NaN there reaches the library (here a recording stand-in) with RGB padded to RGBA, the layers
    as int32 and the sizes as (width, height, layers)."""
    seen = {}

    class Rec:
        def tpt_set_textures(self, h, ptr, w, hgt, nl, layers, ns, on_dev):
            seen.update(w=w, h=hgt, nl=nl, ns=ns, on_dev=on_dev,
                        data=np.ctypeslib.as_array(ctypes.cast(ptr, ctypes.POINTER(ctypes.c_float)), (nl * hgt * w * 4,)).copy(),
                        layers=None if layers is None else
                        np.ctypeslib.as_array(ctypes.cast(layers, ctypes.POINTER(ctypes.c_int32)), (ns,)).copy())
            return 0

    ctx = libs.Context.__new__(libs.Context)
    ctx._L, ctx._h, ctx.device, ctx.spp = Rec(), ctypes.c_void_p(), 0, 4
    tex = np.arange(2 * 3 * 5 * 4, dtype=np.float32).reshape(2, 3, 5, 4)
    tex[..., 3] = np.nan
    ctx.set_textures(tex, np.array([1, -1, 0], np.int64))
    assert (seen["w"], seen["h"], seen["nl"], seen["ns"], seen["on_dev"]) == (5, 3, 2, 3, 0)
    assert np.array_equal(seen["data"].reshape(2, 3, 5, 4)[..., :3], tex[..., :3])
    assert seen["layers"].tolist() == [1, -1, 0]
    rgb = np.arange(1 * 2 * 2 * 3, dtype=np.float32).reshape(1, 2, 2, 3)
    ctx.set_textures(rgb, np.zeros(0, np.int32))
    assert np.array_equal(seen["data"].reshape(1, 2, 2, 4)[..., :3], rgb) and seen["ns"] == 0 and seen["layers"] is None
