"""tpt_set_media without a GPU: the library exports it, the Python binding declares the header's signature,
Context.set_media refuses what the library refuses with the same field names before it reaches the library, the scene
pack (toypathtracer_b200/csrc/tpt_scene_pack.h, built with g++ into a small library by a fixture here) keeps the bytes
of a scene without media and lays the media section out as documented, and every instance that carries the medium step
has neither stack nor spills."""
import ctypes
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

from test_emission_textures_api import LIB, TEX_INSTANCES, _res_usage
from test_irradiance_api import _NoLib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K_SCENE_MEDIA = 128


def test_library_exports_set_media(libs):
    L = ctypes.CDLL(libs.LIB_PATH)
    assert hasattr(L, "tpt_set_media")


def test_binding_matches_header_signature(libs):
    hdr = open(os.path.join(ROOT, "include", "tpt_b200.h")).read()
    m = re.search(r"int\s+tpt_set_media\s*\(([^)]*)\)\s*;", hdr)
    assert m, "tpt_set_media is not declared in include/tpt_b200.h"
    params = [" ".join(p.split()[:-1]) + ("*" if "*" in p.split()[-1] else "") for p in m.group(1).split(",")]
    assert params == ["tpt_context*", "const float*", "int"], params
    ctype = {"tpt_context*": ctypes.c_void_p, "const float*": ctypes.c_void_p, "int": ctypes.c_int}
    fn = libs._load_lib().tpt_set_media
    assert [ctype[p] for p in params] == list(fn.argtypes)
    assert fn.restype is ctypes.c_int
    # the block sits right after tpt_set_emission_textures
    assert hdr.index("int tpt_set_emission_textures") < hdr.index("int tpt_set_media") < hdr.index("int tpt_set_camera")


@pytest.fixture
def fake_ctx(libs):
    ctx = libs.Context.__new__(libs.Context)
    ctx._L, ctx._h, ctx.device, ctx.spp = _NoLib(), ctypes.c_void_p(), 0, 4
    return ctx


def test_refuses_bad_media_before_the_library(libs, fake_ctx):
    good = np.array([[0.1, 0.2, 0.3, 1.0, 0.5], [0, 0, 0, 0, 0], [0, 0, 0, 2.0, -0.9]], np.float32)
    cases = []
    for row, field, value, text in ((1, 0, np.nan, "sphere 1 has sigma_a.r = nan"),
                                    (2, 1, np.inf, "sphere 2 has sigma_a.g = inf"),
                                    (0, 2, -1e-30, "sphere 0 has sigma_a.b = -1e-30"),
                                    (2, 3, -1.0, "sphere 2 has sigma_s = -1"),
                                    (0, 3, -0.0, "sphere 0 has sigma_s = -0"),
                                    (1, 4, 1.0, "sphere 1 has g = 1"),
                                    (1, 4, -1.0, "sphere 1 has g = -1"),
                                    (0, 4, np.nan, "sphere 0 has g = nan")):
        m = good.copy()
        m[row, field] = value
        cases.append((m, "set_media: " + re.escape(text) + "$"))
    cases += [(good.astype(np.float64), "set_media: media must be float32"),
              (good[:, :4], r"set_media: media must have shape \(N, 5\)"),
              (good.reshape(-1), r"set_media: media must have shape \(N, 5\)"),
              ([[0.0, 0.0, 0.0, 1.0, 0.0]], "numpy array or a CPU torch tensor")]
    for media, text in cases:
        with pytest.raises(libs.TptError, match=text):
            fake_ctx.set_media(media)


def test_refuses_torch_inputs_before_the_library(libs, fake_ctx):
    import torch
    good = torch.tensor([[0.1, 0.2, 0.3, 1.0, 0.5]])
    with pytest.raises(libs.TptError, match="float32"):
        fake_ctx.set_media(good.double())
    bad = good.clone()
    bad[0, 3] = -2.0
    with pytest.raises(libs.TptError, match="sphere 0 has sigma_s = -2"):
        fake_ctx.set_media(bad)


def test_media_reach_the_library_as_given(libs):
    """Numpy and CPU torch records arrive as N x 5 float32 in host memory; None and an empty array pass NULL, 0."""
    seen = {}

    class Rec:
        def tpt_set_media(self, h, ptr, n):
            seen.update(n=n, ptr=ptr, data=None if ptr is None else
                        np.ctypeslib.as_array(ctypes.cast(ptr, ctypes.POINTER(ctypes.c_float)), (n * 5,)).copy())
            return 0

    import torch
    ctx = libs.Context.__new__(libs.Context)
    ctx._L, ctx._h, ctx.device, ctx.spp = Rec(), ctypes.c_void_p(), 0, 4
    m = np.array([[0.5, 0.25, 0.0, 3.0, 0.8], [0, 0, 0, 0, 0.99]], np.float32)
    ctx.set_media(m)
    assert seen["n"] == 2 and np.array_equal(seen["data"], m.reshape(-1))
    ctx.set_media(torch.from_numpy(m[::-1].copy()))
    assert seen["n"] == 2 and np.array_equal(seen["data"], m[::-1].reshape(-1))
    ctx.set_media(np.zeros((0, 5), np.float32))
    assert seen["ptr"] is None and seen["n"] == 0
    ctx.set_media(None)
    assert seen["ptr"] is None and seen["n"] == 0


# ---- the pack, through a host build of tpt_scene_pack.h

@pytest.fixture(scope="module")
def pack_lib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("media_pack") / "media_pack_check.so")
    src = os.path.join(ROOT, "tests", "host_sim", "media_pack_check.cpp")
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", out, src], check=True)
    L = ctypes.CDLL(out)
    L.pack_blob.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_uint,
                            ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_void_p]
    L.pack_blob.restype = ctypes.c_longlong
    L.media_offset_of.argtypes = [ctypes.c_uint, ctypes.c_int]
    L.media_offset_of.restype = ctypes.c_longlong
    L.media_bytes_of.argtypes = [ctypes.c_int]
    L.media_bytes_of.restype = ctypes.c_longlong
    return L


# SceneBlobLayout: offSph, offMatA, offMatB, offLights, offInvRadius, offMatRi, totalBytes, geomBytes, flags, ...
LAYOUT = ["offSph", "offMatA", "offMatB", "offLights", "offInvRadius", "offMatRi", "totalBytes", "geomBytes", "flags"]


def pack(L, scene, media=None, flags=0):
    """(blob bytes, layout dict) of the scene (spheres, materials, camera, emissives) packed with `media`."""
    s, m = np.ascontiguousarray(scene[0]), np.ascontiguousarray(scene[1])
    n = s.nbytes // 20
    buf = np.zeros(1 << 20, np.uint8)
    lay = np.zeros(29, np.uint32)
    med = None if media is None else np.ascontiguousarray(media, np.float32)
    size = L.pack_blob(s.ctypes.data, m.ctypes.data, n, None, 0, flags, None if med is None else med.ctypes.data,
                       0 if med is None else med.shape[0], buf.ctypes.data, buf.size, lay.ctypes.data)
    assert size <= buf.size
    return buf[:size].tobytes(), dict(zip(LAYOUT, (int(v) for v in lay[:9])))


def section_bytes(count):
    a16 = lambda x: (x + 15) // 16 * 16  # noqa: E731
    return a16((count + 1) * 16) + a16((count + 1) * 4)


@pytest.fixture(scope="module")
def scene46():
    from toypathtracer_b200 import scenes
    return scenes.reference_scene(1280, 720)


@pytest.fixture(scope="module")
def scene4096():
    from toypathtracer_b200 import scenes
    return scenes.stress_scene(64, 36)


def test_blob_without_media_keeps_the_parents_bytes(pack_lib, scene46):
    """tests/golden/scene46_blob.bin: the 46-sphere scene's blob as the pack made it before media existed (2720 B,
    what bench.py's end-to-end leg copies every step)."""
    golden = open(os.path.join(ROOT, "tests", "golden", "scene46_blob.bin"), "rb").read()
    assert len(golden) == 2720
    blob, lay = pack(pack_lib, scene46)
    assert blob == golden and lay["totalBytes"] == 2720 and lay["flags"] == 0
    # media that reach no sphere: all-zero records, ids past the count (or both) leave the blob plain
    n = 46
    zero = np.zeros((n, 5), np.float32)
    zero[:, 4] = 0.7                                   # g alone is no medium
    past = np.zeros((n + 3, 5), np.float32)
    past[n:, :4] = 1.0
    for media in (zero, past, np.zeros((0, 5), np.float32)):
        b, l2 = pack(pack_lib, scene46, media)
        assert b == golden and l2 == lay
    # the caller's flags cannot ask for the section
    b, l2 = pack(pack_lib, scene46, None, flags=K_SCENE_MEDIA)
    assert b == golden and l2["flags"] == 0


@pytest.mark.parametrize("which", ["scene46", "scene4096"])
def test_media_section_layout(pack_lib, which, request):
    scene = request.getfixturevalue(which)
    n = scene[0].nbytes // 20
    plain, lay0 = pack(pack_lib, scene)
    rng = np.random.default_rng(7)
    media = np.zeros((n + 5, 5), np.float32)                  # records past the count are dropped
    ids = rng.choice(n, size=min(n, 9), replace=False)
    media[ids, :4] = rng.exponential(1.0, (ids.size, 4)).astype(np.float32)
    media[ids[0], :3] = 0.0                                   # scattering only
    media[ids[1], 3] = 0.0                                    # absorbing only
    media[ids, 4] = rng.uniform(-0.95, 0.95, ids.size).astype(np.float32)
    media[n:, :4] = 5.0
    blob, lay = pack(pack_lib, scene, media)
    off = int(pack_lib.media_offset_of(lay["offMatRi"], n))
    assert off == lay0["totalBytes"] == lay["offMatRi"] + (n + 1 + 3) // 4 * 16
    assert int(pack_lib.media_bytes_of(n)) == section_bytes(n)
    assert lay["totalBytes"] == lay0["totalBytes"] + section_bytes(n) == len(blob)
    assert lay["geomBytes"] == lay0["geomBytes"] and lay["flags"] == K_SCENE_MEDIA
    assert {k: v for k, v in lay.items() if k not in ("totalBytes", "flags")} == \
           {k: v for k, v in lay0.items() if k not in ("totalBytes", "flags")}
    assert blob[:off] == plain                                # everything before the section is unchanged
    q4 = np.frombuffer(blob, np.float32, (n + 1) * 4, off).reshape(n + 1, 4)
    g = np.frombuffer(blob, np.float32, n + 1, off + (n + 1) * 16)
    assert np.array_equal(q4[:n], media[:n, :4]) and np.array_equal(g[:n], media[:n, 4])
    assert not q4[n].any() and g[n] == 0                      # entry [count]: no medium
    assert not any(blob[off + (n + 1) * 16 + (n + 1) * 4:])   # padding


def test_scene_layout_did_not_grow(pack_lib):
    # the probe's static_assert pins SceneBlobLayout at 116 bytes
    src = open(os.path.join(ROOT, "tests", "host_sim", "media_pack_check.cpp")).read()
    assert "sizeof(tpt::SceneBlobLayout) == 116" in src


@pytest.mark.skipif(shutil.which("cuobjdump") is None or shutil.which("cu++filt") is None or not os.path.exists(LIB),
                    reason="needs cuobjdump and the built library")
def test_medium_instances_have_no_stack_and_no_local_memory():
    """The medium step lives in the texture instances only; at their register caps it must not spill."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import sass_counts
    res = _res_usage(LIB, sass_counts.demangle)
    for inst in TEX_INSTANCES:
        found = [k for k in res if k.startswith(inst)]
        assert found, inst
        for k in found:
            reg, stack, local = res[k]
            assert stack == 0 and local == 0, (k, reg, stack, local)
            assert reg <= 80, (k, reg)
