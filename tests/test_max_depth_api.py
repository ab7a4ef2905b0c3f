"""The "max_depth" option without a GPU: the header documents it (range, default, refusal text, the roll rule and the
calls it covers), and a host build of the per-call encoding (toypathtracer_b200/csrc/tpt_types.h, built with g++ into a
small library by a fixture here) round-trips every value, sets no bit for the default and routes every other value to
the reference-form instances."""
import ctypes
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K_SCENE_DEPTH = 256
K_SCENE_FLAGS_BELOW = 0x1ff          # kSceneMitsuba .. kSceneDepth


def _header():
    return open(os.path.join(ROOT, "include", "tpt_b200.h")).read()


def _option_text(hdr, key):
    """The header's paragraph for option `key` of tpt_set_option, whitespace and comment stars folded."""
    i = hdr.index(f'"{key}" (')
    j = hdr.index("int tpt_set_option", i)
    return re.sub(r"\s*\*\s*", " ", hdr[i:j])


def test_header_documents_max_depth():
    text = " ".join(_option_text(_header(), "max_depth").split())
    for phrase in ('"max_depth" (1..256, default 10', '"max_depth: 1..256"', "keeps its value",
                   "uploads nothing", "calls already issued keep the value they were issued with",
                   "Depth counts Lambert bounces, Metal and glass continuations and medium scatter events",
                   "only when max_depth > 10", "at depth >= 10", "draws u from its own stream",
                   "q = min(1, max(thr.r, thr.g, thr.b))", "u >= q ends it with nothing added",
                   "the throughput becomes thr / q", "Shadow rays and misses take no roll",
                   "tpt_trace_rays", "tpt_trace_irradiance", "tpt_draw_samples", "tpt_trace_samples",
                   "tpt_draw_aovs and tpt_trace_aovs", "an explicit \"fast_variant\" 0, 1, 2, 4, 5, 6, 7 or 8 is refused",
                   "TPT_MODE_EXACT, TPT_MODE_REFGPU and TPT_MODE_REFGPU_FAST is refused"):
        assert phrase in text, phrase


def test_media_block_points_at_the_option():
    hdr = " ".join(re.sub(r"\s*\*\s*", " ", _header()).split())
    assert "dense media lose energy to it at the default cap of 10: the option \"max_depth\" (tpt_set_option) raises it" \
        in hdr


@pytest.fixture(scope="module")
def enc(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("max_depth") / "max_depth_check.so")
    src = os.path.join(ROOT, "tests", "host_sim", "max_depth_check.cpp")
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", out, src], check=True)
    L = ctypes.CDLL(out)
    for fn, args, res in (("depth_flags_of", [ctypes.c_int], ctypes.c_uint),
                          ("max_depth_of", [ctypes.c_uint], ctypes.c_int),
                          ("scene_depth_flag", [], ctypes.c_uint),
                          ("ref_form_mask", [], ctypes.c_uint),
                          ("ref_max_depth", [], ctypes.c_int),
                          ("max_path_depth", [], ctypes.c_int),
                          ("view_max_depth", [ctypes.c_uint], ctypes.c_int)):
        getattr(L, fn).argtypes = args
        getattr(L, fn).restype = res
    return L


def test_constants(enc):
    assert enc.scene_depth_flag() == K_SCENE_DEPTH
    assert enc.ref_max_depth() == 10 and enc.max_path_depth() == 256
    assert enc.ref_form_mask() & K_SCENE_DEPTH


def test_default_sets_no_bit(enc):
    assert enc.depth_flags_of(10) == 0
    assert enc.max_depth_of(0) == 10 and enc.view_max_depth(0) == 10


def test_every_value_round_trips(enc):
    seen = set()
    for n in range(1, 257):
        f = enc.depth_flags_of(n)
        if n == 10:
            continue
        # the flag, and bits above every kScene* flag: the scene's own flags are untouched
        assert f & K_SCENE_DEPTH and f & ~K_SCENE_DEPTH & K_SCENE_FLAGS_BELOW == 0, (n, hex(f))
        assert enc.max_depth_of(f) == n and enc.view_max_depth(f) == n, n
        # with every other flag set as well
        assert enc.max_depth_of(f | (K_SCENE_FLAGS_BELOW & ~K_SCENE_DEPTH)) == n
        seen.add(f)
    assert len(seen) == 255
    # other flags alone never decode to anything but the default
    for bits in (1, 2, 4, 8, 16, 32, 64, 128, 255):
        assert enc.max_depth_of(bits) == 10


def test_option_is_not_a_scene_flag():
    """begin_call writes the value into the call's copy of the layout; tpt_set_option never touches the scene's flags for
    it, so the upload dedupe (which compares the scene's own flags) never sees it."""
    src = open(os.path.join(ROOT, "toypathtracer_b200", "csrc", "tpt_api.cu")).read()
    line = next(ln for ln in src.splitlines() if '"max_depth"' in ln and "strcmp" in ln)
    assert "sceneFlags" not in line and "scene.layout" not in line and "maxDepth = value" in line
    assert "scene->layout.flags |= depth_flags(ctx->maxDepth);" in src
