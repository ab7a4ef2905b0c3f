"""tpt_trace_samples without a GPU: the library exports it, the Python binding declares the header's signature, and
Context.trace_samples / trace_adaptive refuse wrong shapes, dtypes, sizes, buffer kinds and counts before they reach the
library."""
import ctypes
import os
import re

import numpy as np
import pytest

from test_irradiance_api import _NoLib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_trace_samples(libs):
    L = ctypes.CDLL(libs.LIB_PATH)
    assert hasattr(L, "tpt_trace_samples")


def test_binding_matches_header_signature(libs):
    hdr = open(os.path.join(ROOT, "include", "tpt_b200.h")).read()
    m = re.search(r"int\s+tpt_trace_samples\s*\(([^)]*)\)\s*;", hdr)
    assert m, "tpt_trace_samples is not declared in include/tpt_b200.h"
    params = [" ".join(p.split()[:-1]) + ("*" if "*" in p.split()[-1] else "") for p in m.group(1).split(",")]
    assert params == ["tpt_context*", "const float*", "const int*", "int", "long long", "const int*", "long long", "int",
                      "int", "float*", "float*", "int", "long long*", "void*"], params
    ctype = {"tpt_context*": ctypes.c_void_p, "const float*": ctypes.c_void_p, "float*": ctypes.c_void_p,
             "const int*": ctypes.c_void_p, "void*": ctypes.c_void_p, "int": ctypes.c_int,
             "long long": ctypes.c_longlong, "long long*": ctypes.POINTER(ctypes.c_longlong)}
    fn = libs._load_lib().tpt_trace_samples
    assert [ctype[p] for p in params] == list(fn.argtypes)
    assert fn.restype is ctypes.c_int


@pytest.fixture
def fake_ctx(libs):
    ctx = libs.Context.__new__(libs.Context)
    ctx._L, ctx._h, ctx.device, ctx.spp = _NoLib(), ctypes.c_void_p(), 0, 4
    return ctx


def test_trace_samples_refuses_before_the_library(libs, fake_ctx):
    inp = np.zeros((8, 6), np.float32)
    ids = np.zeros(8, np.int32)
    lst = np.zeros(5, np.int32)
    f4 = np.zeros((5, 4), np.float32)
    bad = [
        (dict(inputs=np.zeros((8, 5), np.float32)), "inputs must have shape"),
        (dict(inputs=inp.astype(np.float64)), "float32"),
        (dict(inputs=np.zeros((6, 8), np.float32).T), "C-contiguous"),
        (dict(inputs=libs.DevicePtr(256)), "DevicePtr inputs need num_in"),
        (dict(inputs=inp, num_in=7), "n does not match inputs"),
        (dict(inputs=inp, ids=ids), "ids are only taken with points"),
        (dict(inputs=inp, ids=np.zeros(7, np.int32), points=True), "n does not match ids"),
        (dict(inputs=inp, ids=ids.astype(np.int64), points=True), "int32"),
        (dict(inputs=inp, n=7), "without entries n must be num_in"),
        (dict(inputs=inp, entries=lst, n=4), "n does not match entries"),
        (dict(inputs=inp, entries=lst.astype(np.int64)), "int32"),
        (dict(inputs=inp, entries=np.zeros((5, 1), np.int32)), "entries must have shape"),
        (dict(inputs=inp, entries=libs.DevicePtr(256)), "needs n"),
        (dict(inputs=inp, entries=lst, sq4=f4), "sq4 needs sum4"),
        (dict(inputs=inp, entries=lst, sum4=np.zeros((8, 4), np.float32)), "sum4 must hold 5 x 4 float32"),
        (dict(inputs=inp, entries=lst, sum4=f4, sq4=np.zeros((5, 3), np.float32)), "sq4 must hold 5 x 4 float32"),
        (dict(inputs=inp, entries=lst, sum4=f4.astype(np.float64)), "float32"),
        (dict(inputs=inp, entries=libs.DevicePtr(256), n=5, sum4=f4), "entries, sum4 and sq4 must be all host or all device"),
        (dict(inputs=inp, entries=lst, sum4=libs.DevicePtr(256)), "must be all host or all device"),
        (dict(inputs=libs.DevicePtr(256), num_in=8, entries=lst, sum4=f4), "must be all host or all device"),
        (dict(inputs=inp, ids=libs.DevicePtr(256), points=True), "inputs and ids must be all host or all device"),
    ]
    for kw, text in bad:
        with pytest.raises(libs.TptError, match=text):
            fake_ctx.trace_samples(**kw)


def test_trace_samples_refuses_torch_buffers_before_the_library(libs, fake_ctx):
    import torch
    inp = torch.zeros((8, 6))
    with pytest.raises(libs.TptError, match="contiguous float32"):
        fake_ctx.trace_samples(inp.double())
    with pytest.raises(libs.TptError, match="contiguous int32"):
        fake_ctx.trace_samples(inp, entries=torch.zeros(3, dtype=torch.int64))
    with pytest.raises(libs.TptError, match="sum4 must hold 3 x 4 float32"):
        fake_ctx.trace_samples(inp, entries=torch.zeros(3, dtype=torch.int32), sum4=torch.zeros((3, 3)))


def test_trace_adaptive_refuses_before_the_library(libs, fake_ctx):
    with pytest.raises(libs.TptError, match="need 1 <= base_spp <= max_spp"):
        fake_ctx.trace_adaptive(np.zeros((8, 6), np.float32), base_spp=8, max_spp=4)
    with pytest.raises(libs.TptError, match="need 1 <= base_spp <= max_spp"):
        fake_ctx.trace_adaptive(np.zeros((8, 6), np.float32), base_spp=0)
