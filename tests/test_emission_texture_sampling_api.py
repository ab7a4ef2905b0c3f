"""The "emission_texture_sampling" option without a GPU: the header documents it; the per-layer table build
(toypathtracer_b200/csrc/tpt_env_tables.h, built with g++ into a small library by a fixture here) gives each layer the
environment builder's tables for that layer alone, and a layer without weight its sentinel; the slot size is the
documented formula; and the layout the trace kernels take has not grown."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

from test_environment_sampling_api import build_tables, tables_lib  # noqa: F401

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emit_lib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("emit_tables") / "emit_tables_check.so")
    src = os.path.join(ROOT, "tests", "host_sim", "emit_tables_check.cpp")
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", out, src], check=True)
    L = ctypes.CDLL(out)
    L.emit_tables_check.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    L.emit_tables_check.restype = ctypes.c_int
    for f in (L.emit_slot_size, L.emit_tables_at):
        f.argtypes = [ctypes.c_int] * 4
        f.restype = ctypes.c_longlong
    L.scene_layout_size.restype = ctypes.c_longlong
    return L


def build_layer_tables(L, layers):
    """(ok, texels with alpha, [(rows bytes, cols bytes)] per layer) of tpt_set_emission_textures' build."""
    n, H, W = layers.shape[:3]
    tex = np.zeros((n, H, W, 4), np.float32)
    tex[..., :3] = layers[..., :3]
    tex[..., 3] = -7.0
    block = H + W * H
    tabs = bytearray(8 * block * n)
    tb = (ctypes.c_char * len(tabs)).from_buffer(tabs)
    ok = L.emit_tables_check(tex.ctypes.data, W, H, n, ctypes.addressof(tb))
    raw = bytes(tabs)
    out = [(raw[8 * block * k: 8 * (block * k + H)], raw[8 * (block * k + H): 8 * block * (k + 1)]) for k in range(n)]
    return ok, tex, out


def _layer_sets():
    rng = np.random.default_rng(4)
    H, W = 12, 20
    rand = rng.exponential(1.0, (H, W, 3)).astype(np.float32)
    rand[rng.random((H, W)) < 0.3] = 0.0
    one_hot = np.zeros((H, W, 3), np.float32)
    one_hot[7, 19] = (2.0, 0.5, 0.0)
    hot = np.full((H, W, 3), 1e-3, np.float32)
    hot[3:5, 8:10] = 400.0
    zero = np.zeros((H, W, 3), np.float32)
    return {
        "mixed": np.stack([rand, zero, one_hot, hot]),
        "zero_first": np.stack([zero, hot]),
        "all_zero": np.stack([zero, zero]),
        "1x1": np.array([[[[0.5, 1.0, 2.0]]], [[[0.0, 0.0, 0.0]]], [[[3.0, 0.0, 0.0]]]], np.float32),
        "single_row": np.stack([rng.random((1, 29, 3)).astype(np.float32), np.zeros((1, 29, 3), np.float32)]),
    }


SETS = _layer_sets()


@pytest.mark.parametrize("name", sorted(SETS))
def test_each_layer_gets_the_environment_builders_tables(emit_lib, tables_lib, name):
    layers = SETS[name]
    ok, tex, tabs = build_layer_tables(emit_lib, layers)
    any_weight = False
    for k in range(len(layers)):
        eok, etex, erows, ecols, _w = build_tables(tables_lib, layers[k])
        rows, cols = tabs[k]
        if eok:
            any_weight = True
            assert rows == erows and cols == ecols, (name, k)
            assert np.array_equal(tex[k, ..., 3], etex[..., 3]), (name, k)
        else:
            # no weight: the sentinel in every entry of its block, zero probability in its alpha
            r = np.frombuffer(rows + cols, dtype=[("p", "<f4"), ("a", "<i4")])
            assert (r["a"] == emit_lib.emit_no_tables()).all() and (r["p"] == 0).all(), (name, k)
            assert (tex[k, ..., 3] == 0).all(), (name, k)
        assert np.array_equal(tex[k, ..., :3], layers[k]), (name, k)     # RGB untouched
    assert ok == int(any_weight)


def test_sentinel_is_what_the_kernels_test():
    """The kernels test the first row entry's alias for a negative value (emit_tables)."""
    src = open(os.path.join(ROOT, "toypathtracer_b200", "csrc", "tpt_env_tables.h")).read()
    assert re.search(r"constexpr int32_t kEmitNoTables = -1;", src)
    fast = open(os.path.join(ROOT, "toypathtracer_b200", "csrc", "tpt_fast.cu")).read()
    assert re.search(r"__float_as_int\(__ldg\(t\)\.y\) < 0", fast)


def test_slot_bytes_match_the_documented_formula(emit_lib):
    for W, H, L, S in [(1, 1, 1, 0), (20, 12, 4, 3), (512, 256, 8, 46), (7, 3, 2, 1), (4096, 2048, 1, 4096)]:
        pad = 4 * (S % 2)
        assert emit_lib.emit_slot_size(W, H, L, S) == 16 * W * H * L + 4 * S + pad + 8 * W * H * L + 8 * H * L
        off = emit_lib.emit_tables_at(W, H, L, S)
        assert off == 16 * W * H * L + 4 * S + pad and off % 8 == 0


def test_scene_layout_did_not_grow(emit_lib):
    # the probe's static_asserts pin TexSet at 32 and SceneBlobLayout at 116 bytes; the library agrees
    assert emit_lib.scene_layout_size() == 116


def test_header_documents_the_option():
    hdr = open(os.path.join(ROOT, "include", "tpt_b200.h")).read()
    m = re.search(r'"emission_texture_sampling" \(default 0[^;]*;', hdr)
    assert m, "include/tpt_b200.h does not document \"emission_texture_sampling\""
    opt = hdr[hdr.index('"emission_texture_sampling" (default 0'):hdr.index("int tpt_set_option")]
    for needle in ("six draws", "pt(x)", "cos_x", "power heuristic", "kSceneEmitSampling", "rays", "8 * width * height"):
        assert needle in opt, needle
    emit = hdr[hdr.index("Emission textures for the fast mode"):hdr.index("int tpt_set_emission_textures")]
    assert "emission_texture_sampling" in emit and "8 * height * layers" in emit
