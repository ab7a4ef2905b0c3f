"""tpt_trace_irradiance without a GPU: the library exports it, the Python binding declares the header's signature, and
Context.trace_irradiance refuses wrong shapes, dtypes, sizes, buffer kinds and n before it reaches the library."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_trace_irradiance(libs):
    L = ctypes.CDLL(libs.LIB_PATH)
    assert hasattr(L, "tpt_trace_irradiance")


def test_binding_matches_header_signature(libs):
    hdr = open(os.path.join(ROOT, "include", "tpt_b200.h")).read()
    m = re.search(r"int\s+tpt_trace_irradiance\s*\(([^)]*)\)\s*;", hdr)
    assert m, "tpt_trace_irradiance is not declared in include/tpt_b200.h"
    params = [" ".join(p.split()[:-1]) + ("*" if "*" in p.split()[-1] else "") for p in m.group(1).split(",")]
    assert params == ["tpt_context*", "const float*", "const int*", "int", "long long", "int", "int", "float*", "int",
                      "long long*", "void*"], params
    ctype = {"tpt_context*": ctypes.c_void_p, "const float*": ctypes.c_void_p, "float*": ctypes.c_void_p,
             "const int*": ctypes.c_void_p, "void*": ctypes.c_void_p, "int": ctypes.c_int,
             "long long": ctypes.c_longlong, "long long*": ctypes.POINTER(ctypes.c_longlong)}
    fn = libs._load_lib().tpt_trace_irradiance
    assert [ctype[p] for p in params] == list(fn.argtypes)
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


def test_trace_irradiance_refuses_before_the_library(libs, fake_ctx):
    pts = np.zeros((8, 6), np.float32)
    ids = np.zeros(8, np.int32)
    f4 = np.zeros((8, 4), np.float32)
    bad = [
        (dict(points=np.zeros((8, 5), np.float32)), "points must have shape"),
        (dict(points=np.zeros(48, np.float32)), "points must have shape"),
        (dict(points=pts.astype(np.float64)), "float32"),
        (dict(points=np.zeros((6, 8), np.float32).T), "C-contiguous"),
        (dict(points=libs.DevicePtr(256)), "needs n"),
        (dict(points=pts, n=7), "n does not match points"),
        (dict(points=pts, ids=np.zeros(7, np.int32)), "n does not match ids"),
        (dict(points=pts, ids=np.zeros((8, 1), np.int32)), "ids must have shape"),
        (dict(points=pts, ids=ids.astype(np.int64)), "int32"),
        (dict(points=pts, ids=ids.astype(np.float32)), "int32"),
        (dict(points=pts, ids=np.zeros(16, np.int32)[::2]), "C-contiguous"),
        (dict(points=pts, ids=libs.DevicePtr(256)), "points and ids must be all host or all device"),
        (dict(points=libs.DevicePtr(256), n=8, ids=ids, out=libs.DevicePtr(512)),
         "points and ids must be all host or all device"),
        (dict(points=pts, out=np.zeros((7, 4), np.float32)), "out must hold 8 x 4 float32"),
        (dict(points=pts, out=np.zeros((8, 3), np.float32)), "out must hold 8 x 4 float32"),
        (dict(points=pts, out=f4.astype(np.float64)), "float32"),
        (dict(points=pts, out=np.zeros((4, 8), np.float32).T), "C-contiguous"),
    ]
    for kw, text in bad:
        with pytest.raises(libs.TptError, match=text):
            fake_ctx.trace_irradiance(**kw)


def test_trace_irradiance_refuses_torch_buffers_before_the_library(libs, fake_ctx):
    import torch
    pts = torch.zeros((8, 6))
    with pytest.raises(libs.TptError, match="contiguous float32"):
        fake_ctx.trace_irradiance(pts.double())
    with pytest.raises(libs.TptError, match="contiguous int32"):
        fake_ctx.trace_irradiance(pts, ids=torch.zeros(8, dtype=torch.int64))
    with pytest.raises(libs.TptError, match="contiguous float32"):
        fake_ctx.trace_irradiance(torch.zeros((6, 8)).t())
    with pytest.raises(libs.TptError, match="out must hold 8 x 4 float32"):
        fake_ctx.trace_irradiance(pts, out=torch.zeros((8, 3)))
