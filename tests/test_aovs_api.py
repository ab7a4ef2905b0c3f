"""The caller-buffer calls (tpt_trace_rays, tpt_draw_aovs, tpt_trace_aovs, tpt_draw_samples) without a GPU: the Python
binding declares the header's signatures, and the wrappers refuse wrong shapes, dtypes, sizes, buffer kinds and n before
they reach the library. Also: the library exports the AOV calls."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FUNCS = ("tpt_draw_aovs", "tpt_trace_aovs")
CALLER_BUFFER_FUNCS = ("tpt_trace_rays",) + FUNCS + ("tpt_draw_samples",)


@pytest.mark.parametrize("name", FUNCS)
def test_library_exports(libs, name):
    L = ctypes.CDLL(libs.LIB_PATH)
    assert hasattr(L, name)


@pytest.mark.parametrize("name", CALLER_BUFFER_FUNCS)
def test_binding_matches_header_signature(libs, name):
    hdr = open(os.path.join(ROOT, "include", "tpt_b200.h")).read()
    m = re.search(r"int\s+" + name + r"\s*\(([^)]*)\)\s*;", hdr)
    assert m, f"{name} is not declared in include/tpt_b200.h"
    params = [" ".join(p.split()[:-1]) + ("*" if "*" in p.split()[-1] else "") for p in m.group(1).split(",")]
    ctype = {"tpt_context*": ctypes.c_void_p, "const float*": ctypes.c_void_p, "float*": ctypes.c_void_p,
             "const int*": ctypes.c_void_p, "int*": ctypes.c_void_p, "void*": ctypes.c_void_p, "int": ctypes.c_int,
             "unsigned": ctypes.c_uint, "long long": ctypes.c_longlong, "long long*": ctypes.POINTER(ctypes.c_longlong)}
    L = libs._load_lib()
    fn = getattr(L, name)
    assert [ctype[p.replace(" *", "*")] for p in params] == list(fn.argtypes), params
    assert fn.restype is ctypes.c_int


class _NoLib:
    """Stands in for the library: any call reaching it fails the test."""

    def __getattr__(self, name):
        raise AssertionError(f"{name} was called")


@pytest.fixture
def fake_ctx(libs):
    ctx = libs.Context.__new__(libs.Context)
    ctx._L, ctx._h, ctx.device, ctx.spp = _NoLib(), ctypes.c_void_p(), 0, 4
    return ctx


def test_trace_rays_refuses_before_the_library(libs, fake_ctx):
    """`out` must hold N float4, like the AOV outputs: the library writes N x 16 bytes into it."""
    rays = np.zeros((8, 6), np.float32)
    f4 = np.zeros((8, 4), np.float32)
    bad = [
        (dict(rays=rays, out=np.zeros((3, 4), np.float32)), "trace_rays: out must hold 8 x 4 float32"),
        (dict(rays=rays, out=np.zeros((9, 4), np.float32)), "trace_rays: out must hold 8 x 4 float32"),
        (dict(rays=rays, out=f4.astype(np.float64)), "float32"),
        (dict(rays=rays, out=np.zeros((4, 8), np.float32).T), "C-contiguous"),
        (dict(rays=np.zeros((8, 5), np.float32), out=f4), "shape"),
        (dict(rays=np.zeros(48, np.float32), out=f4), "shape"),
        (dict(rays=libs.DevicePtr(256), out=f4), "needs n"),
        (dict(rays=rays, out=f4, n=7), "n does not match"),
    ]
    for kw, text in bad:
        with pytest.raises(libs.TptError, match=text):
            fake_ctx.trace_rays(**kw)


def test_trace_aovs_refuses_before_the_library(libs, fake_ctx):
    rays = np.zeros((8, 6), np.float32)
    f4 = np.zeros((8, 4), np.float32)
    bad = [
        (dict(rays=np.zeros((8, 5), np.float32), albedo=f4), "shape"),
        (dict(rays=np.zeros(48, np.float32), albedo=f4), "shape"),
        (dict(rays=rays.astype(np.float64), albedo=f4), "float32"),
        (dict(rays=rays, albedo=f4, n=7), "n does not match"),
        (dict(rays=libs.DevicePtr(256)), "needs n"),
        (dict(rays=rays, albedo=np.zeros((7, 4), np.float32)), "albedo must hold"),
        (dict(rays=rays, normal=np.zeros((8, 3), np.float32)), "normal must hold"),
        (dict(rays=rays, albedo=f4.astype(np.float64)), "float32"),
        (dict(rays=rays, ids=np.zeros(8, np.int64)), "int32"),
        (dict(rays=rays, ids=np.zeros(8, np.float32)), "int32"),
        (dict(rays=rays, ids=np.zeros(9, np.int32)), "ids must hold"),
        (dict(rays=rays, albedo=np.zeros((4, 8), np.float32).T), "C-contiguous"),
        (dict(rays=rays, albedo=f4, ids=libs.DevicePtr(256)), "all host or all device"),
    ]
    for kw, text in bad:
        with pytest.raises(libs.TptError, match=text):
            fake_ctx.trace_aovs(**kw)


def test_draw_aovs_refuses_before_the_library(libs, fake_ctx):
    w, h = 16, 8
    f4, i1 = np.zeros((h, w, 4), np.float32), np.zeros((h, w), np.int32)
    with pytest.raises(libs.TptError, match="no output buffer"):
        fake_ctx.draw_aovs(0, 1, w, h)
    with pytest.raises(libs.TptError, match="albedo must hold"):
        fake_ctx.draw_aovs(0, 1, w, h, albedo=np.zeros((h - 1, w, 4), np.float32))
    with pytest.raises(libs.TptError, match="ids must hold"):
        fake_ctx.draw_aovs(0, 1, w, h, ids=np.zeros((h, w, 4), np.int32))
    with pytest.raises(libs.TptError, match="int32"):
        fake_ctx.draw_aovs(0, 1, w, h, ids=i1.astype(np.uint32))
    with pytest.raises(libs.TptError, match="float32"):
        fake_ctx.draw_aovs(0, 1, w, h, normal=f4.astype(np.float16))
    # a packed band holds numRows rows: a full-size buffer is the wrong size for it
    with pytest.raises(libs.TptError, match="normal must hold"):
        fake_ctx.draw_aovs(0, 1, w, h, normal=f4, rows=(2, 3, 1, 1))
    with pytest.raises(libs.TptError, match="all host or all device"):
        fake_ctx.draw_aovs(0, 1, w, h, albedo=f4, normal=libs.DevicePtr(256))


def test_draw_samples_refuses_before_the_library(libs, fake_ctx):
    w, h = 16, 8
    px = np.arange(10, dtype=np.int32)
    f4 = np.zeros((10, 4), np.float32)
    bad = [
        (dict(pixels=px.reshape(2, 5), sum4=f4), "shape"),
        (dict(pixels=px.astype(np.int64), sum4=f4), "int32"),
        (dict(pixels=px.astype(np.float32), sum4=f4), "int32"),
        (dict(pixels=px[::2], sum4=f4[:5]), "C-contiguous"),
        (dict(pixels=px, sum4=f4, n=9), "n does not match"),
        (dict(pixels=libs.DevicePtr(256)), "needs n"),
        (dict(pixels=px, sum4=np.zeros((9, 4), np.float32)), "sum4 must hold"),
        (dict(pixels=px, sum4=f4, sq4=np.zeros((10, 3), np.float32)), "sq4 must hold"),
        (dict(pixels=px, sum4=f4.astype(np.float64)), "float32"),
        (dict(pixels=px, sq4=f4), "sq4 needs sum4"),
        (dict(pixels=px, sum4=f4, sq4=libs.DevicePtr(256)), "all host or all device"),
        (dict(pixels=libs.DevicePtr(256), n=10, sum4=f4), "all host or all device"),
        (dict(pixels=libs.DevicePtr(256), n=-1, sum4=libs.DevicePtr(512)), "n < 0"),
        (dict(sum4=np.zeros((w * h, 4), np.float32), n=w * h - 1), "n must be width"),
        (dict(sum4=np.zeros((w * h - 1, 4), np.float32)), "sum4 must hold"),
    ]
    for kw, text in bad:
        with pytest.raises(libs.TptError, match=text):
            fake_ctx.draw_samples(0, w, h, **kw)


def test_as_ptr_keeps_its_float32_behaviour(libs):
    a = np.zeros(4, np.float32)
    assert libs._as_ptr(a)[:2] == (a.ctypes.data, False)
    with pytest.raises(libs.TptError, match="backbuffer must be a C-contiguous float32 array"):
        libs._as_ptr(np.zeros(4, np.int32))
    i = np.zeros(4, np.int32)
    assert libs._as_ptr(i, "int32")[:2] == (i.ctypes.data, False)
    import torch
    with pytest.raises(libs.TptError, match="backbuffer tensor must be contiguous float32"):
        libs._as_ptr(torch.zeros(4, dtype=torch.int32))
    with pytest.raises(libs.TptError, match="backbuffer tensor must be contiguous int32"):
        libs._as_ptr(torch.zeros(4), "int32")
