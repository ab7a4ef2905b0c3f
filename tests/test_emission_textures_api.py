"""tpt_set_emission_textures without a GPU: the library exports it, the Python binding declares the header's signature,
Context.set_emission_textures refuses wrong shapes, dtypes, texel values and sphere layers before it reaches the
library and hands RGB over as RGBA, and every instance that carries the texture lookups has neither stack nor spills."""
import ctypes
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

from test_irradiance_api import _NoLib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "toypathtracer_b200", "libtpt_b200.so")

# the slab queue's reference-form 6-CTA and 768-thread instances and their light-sampling-off twins (tex_mode)
TEX_INSTANCES = [f"{k}{tw}<{shape}, 0{tail}" for k in ("k_fast_queue", "k_fast_rays", "k_fast_samples")
                 for tw in ("", "_nolight") for shape in ("128, 6", "768, 1")
                 for tail in ((", 0>", ", 1>") if k == "k_fast_samples" else (">",))]


def test_library_exports_set_emission_textures(libs):
    L = ctypes.CDLL(libs.LIB_PATH)
    assert hasattr(L, "tpt_set_emission_textures")


def test_binding_matches_header_signature(libs):
    hdr = open(os.path.join(ROOT, "include", "tpt_b200.h")).read()
    m = re.search(r"int\s+tpt_set_emission_textures\s*\(([^)]*)\)\s*;", hdr)
    assert m, "tpt_set_emission_textures is not declared in include/tpt_b200.h"
    params = [" ".join(p.split()[:-1]) + ("*" if "*" in p.split()[-1] else "") for p in m.group(1).split(",")]
    assert params == ["tpt_context*", "const float*", "int", "int", "int", "const int*", "int", "int"], params
    ctype = {"tpt_context*": ctypes.c_void_p, "const float*": ctypes.c_void_p, "const int*": ctypes.c_void_p,
             "int": ctypes.c_int}
    fn = libs._load_lib().tpt_set_emission_textures
    assert [ctype[p] for p in params] == list(fn.argtypes)
    assert fn.restype is ctypes.c_int


@pytest.fixture
def fake_ctx(libs):
    ctx = libs.Context.__new__(libs.Context)
    ctx._L, ctx._h, ctx.device, ctx.spp = _NoLib(), ctypes.c_void_p(), 0, 4
    return ctx


def test_refuses_bad_textures_before_the_library(libs, fake_ctx):
    good = np.ones((2, 4, 8, 3), np.float32)
    layers = np.array([0, 1, -1], np.int32)
    nan, inf, neg, negzero = good.copy(), good.copy(), good.copy(), good.copy()
    nan[1, 1, 2, 0] = np.nan
    inf[0, 3, 7, 2] = np.inf
    neg[1, 0, 0, 1] = -1e-30
    negzero[0, 2, 5, 2] = -0.0
    shape_text = r"set_emission_textures: textures must have shape \(L, H, W, 3\) or \(L, H, W, 4\)"
    bad = [
        (np.ones((4, 8, 3), np.float32), shape_text),
        (np.ones((2, 4, 8, 2), np.float32), shape_text),
        (np.ones((2, 4, 8, 5), np.float32), shape_text),
        (np.ones((0, 4, 8, 3), np.float32), shape_text),
        (np.ones((2, 4, 0, 3), np.float32), shape_text),
        (good.astype(np.float64), "set_emission_textures: textures must be float32"),
        (nan, "finite and not negative"),
        (inf, "finite and not negative"),
        (neg, "finite and not negative"),
        (negzero, "finite and not negative"),
        ([[[[1.0, 1.0, 1.0]]]], "numpy array or a torch tensor"),
    ]
    for tex, text in bad:
        with pytest.raises(libs.TptError, match=text):
            fake_ctx.set_emission_textures(tex, layers)


def test_refuses_bad_sphere_layers_before_the_library(libs, fake_ctx):
    good = np.ones((2, 4, 8, 4), np.float32)
    for layers, text in (([0, 2], r"set_emission_textures: sphere_layers\[1\] = 2 is outside \[-1, 2\)"),
                         ([-2, 0], r"sphere_layers\[0\] = -2 is outside \[-1, 2\)"),
                         (np.zeros((2, 2), np.int32), "1-D integer array"),
                         (np.zeros(3, np.float32), "1-D integer array"),
                         (None, "sphere_layers is required")):
        with pytest.raises(libs.TptError, match=text):
            fake_ctx.set_emission_textures(good, layers)


def test_refuses_torch_inputs_before_the_library(libs, fake_ctx):
    import torch
    good = torch.ones((2, 4, 8, 4))
    layers = torch.tensor([0, 1])
    with pytest.raises(libs.TptError, match="float32"):
        fake_ctx.set_emission_textures(good.double(), layers)
    with pytest.raises(libs.TptError, match="shape"):
        fake_ctx.set_emission_textures(torch.ones((2, 4, 8, 5)), layers)
    with pytest.raises(libs.TptError, match="outside"):
        fake_ctx.set_emission_textures(good, torch.tensor([0, 3]))
    for v in (float("nan"), float("inf"), -2.0, -0.0):
        t = good.clone()
        t[1, 2, 3, 1] = v
        with pytest.raises(libs.TptError, match="finite and not negative"):
            fake_ctx.set_emission_textures(t, layers)


def test_emission_textures_reach_the_library_as_rgba(libs):
    """RGB is padded to RGBA (alpha, even NaN, is not checked), the layers arrive as int32 and the sizes as (width,
    height, layers); clearing passes NULL. The albedo call is not touched."""
    seen = {}

    class Rec:
        def tpt_set_emission_textures(self, h, ptr, w, hgt, nl, layers, ns, on_dev):
            seen.update(w=w, h=hgt, nl=nl, ns=ns, on_dev=on_dev, ptr=ptr,
                        data=None if ptr is None else
                        np.ctypeslib.as_array(ctypes.cast(ptr, ctypes.POINTER(ctypes.c_float)), (nl * hgt * w * 4,)).copy(),
                        layers=None if layers is None else
                        np.ctypeslib.as_array(ctypes.cast(layers, ctypes.POINTER(ctypes.c_int32)), (ns,)).copy())
            return 0

        def tpt_set_textures(self, *args):
            raise AssertionError("tpt_set_textures was called")

    ctx = libs.Context.__new__(libs.Context)
    ctx._L, ctx._h, ctx.device, ctx.spp = Rec(), ctypes.c_void_p(), 0, 4
    tex = np.arange(2 * 3 * 5 * 4, dtype=np.float32).reshape(2, 3, 5, 4)
    tex[..., 3] = np.nan
    ctx.set_emission_textures(tex, np.array([1, -1, 0], np.int64))
    assert (seen["w"], seen["h"], seen["nl"], seen["ns"], seen["on_dev"]) == (5, 3, 2, 3, 0)
    assert np.array_equal(seen["data"].reshape(2, 3, 5, 4)[..., :3], tex[..., :3])
    assert seen["layers"].tolist() == [1, -1, 0]
    rgb = np.arange(1 * 2 * 2 * 3, dtype=np.float32).reshape(1, 2, 2, 3)
    ctx.set_emission_textures(rgb, np.zeros(0, np.int32))
    got = seen["data"].reshape(1, 2, 2, 4)
    assert np.array_equal(got[..., :3], rgb) and (got[..., 3] == 0).all() and seen["ns"] == 0 and seen["layers"] is None
    ctx.set_emission_textures(None)
    assert seen["ptr"] is None and (seen["w"], seen["h"], seen["nl"], seen["ns"]) == (0, 0, 0, 0)


def _res_usage(lib, demangle):
    """{demangled kernel name: (registers, stack bytes, local bytes)} from cuobjdump -res-usage."""
    out = subprocess.run(["cuobjdump", "-res-usage", lib], capture_output=True, text=True, check=True).stdout
    res, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            cur = demangle(m.group(1))
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", line)
        if m and cur:
            res[cur] = tuple(int(g) for g in m.groups())
    return res


@pytest.mark.skipif(shutil.which("cuobjdump") is None or shutil.which("cu++filt") is None or not os.path.exists(LIB),
                    reason="needs cuobjdump and the built library")
def test_texture_instances_have_no_stack_and_no_spills():
    """Both lookups (albedo and emission, at hits and at a light's shadow ray) live in these instances only; at their
    register caps they must still keep everything in registers."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import sass_counts
    res = _res_usage(LIB, sass_counts.demangle)
    for inst in TEX_INSTANCES:
        found = [k for k in res if k.startswith(inst)]
        assert found, (inst, sorted(k for k in res if k.startswith("k_fast_samples"))[:8])
        for k in found:
            reg, stack, local = res[k]
            assert stack == 0 and local == 0, (k, reg, stack, local)
