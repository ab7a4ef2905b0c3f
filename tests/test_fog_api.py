"""tpt_set_fog without a GPU: the library exports it, the Python binding declares the header's signature, Context.set_fog
refuses what the library refuses with the same field names before it reaches the library, the header documents the
estimator, a host build of the pack, the chord helper and the phase function (tests/host_sim/fog_check.cpp) keeps the
plain scene's bytes, lays the fog section out as documented, measures chords as float64 does and integrates the phase
function to 1, and every instance that carries the fog step has neither stack nor spills."""
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
K_SCENE_FOG = 512
TPT_MAX_T = 1.0e7


def test_library_exports_set_fog(libs):
    L = ctypes.CDLL(libs.LIB_PATH)
    assert hasattr(L, "tpt_set_fog")


def test_binding_matches_header_signature(libs):
    hdr = open(os.path.join(ROOT, "include", "tpt_b200.h")).read()
    m = re.search(r"int\s+tpt_set_fog\s*\(([^)]*)\)\s*;", hdr)
    assert m, "tpt_set_fog is not declared in include/tpt_b200.h"
    params = [" ".join(p.split()[:-1]) + ("*" if "*" in p.split()[-1] else "") for p in m.group(1).split(",")]
    assert params == ["tpt_context*", "const float*"], params
    fn = libs._load_lib().tpt_set_fog
    assert list(fn.argtypes) == [ctypes.c_void_p, ctypes.c_void_p]
    assert fn.restype is ctypes.c_int
    # the block sits right after tpt_set_media
    assert hdr.index("int tpt_set_media") < hdr.index("int tpt_set_fog") < hdr.index("int tpt_set_camera")


def test_header_documents_the_estimator():
    hdr = open(os.path.join(ROOT, "include", "tpt_b200.h")).read()
    block = hdr[hdr.index("int tpt_set_media"):hdr.index("int tpt_set_fog")]
    for text in ("{c.x, c.y, c.z, R, sigma_a.r, sigma_a.g, sigma_a.b, sigma_s, g}",
                 "dot(d, normal) <= 0", "L = |[0, t] ∩ [t_in, t_out]|", "o + d (max(t_in, 0) + t_s)",
                 "t_s = -ln(1 - u) / sigma_s", "exp(-sigma_a L)", "exp(-sigma_a t_s)",
                 "p(cos) = (1 - g^2) / (4 pi (1 + g^2 - 2 g cos)^(3/2))", "exactly 1 / (4 pi) for |g| < 1e-3",
                 "none is excluded", "T_shadow = exp(-(sigma_a + sigma_s) L)",
                 "counts as air", "\"tpt_set_fog: radius = -1\"", "-1, 3 or 9", "do not change"):
        assert text in block, text


@pytest.fixture
def fake_ctx(libs):
    ctx = libs.Context.__new__(libs.Context)
    ctx._L, ctx._h, ctx.device, ctx.spp = _NoLib(), ctypes.c_void_p(), 0, 4
    return ctx


GOOD = dict(centre=(0.0, 1.0, -1.5), radius=6.0, sigma_a=(0.01, 0.02, 0.03), sigma_s=0.1, g=0.3)


def test_refuses_bad_fog_before_the_library(libs, fake_ctx):
    cases = [(dict(centre=(np.nan, 0, 0)), "centre.x = nan"), (dict(centre=(0, np.inf, 0)), "centre.y = inf"),
             (dict(centre=(0, 0, -np.inf)), "centre.z = -inf"), (dict(centre=(0, 0, 1e39)), "centre.z = inf"),
             (dict(radius=-1.0), "radius = -1"), (dict(radius=0.0), "radius = 0"), (dict(radius=-0.0), "radius = -0"),
             (dict(radius=np.inf), "radius = inf"), (dict(radius=np.nan), "radius = nan"),
             (dict(sigma_a=(0.1, -0.0, 0.1)), "sigma_a.g = -0"), (dict(sigma_a=(0.1, 0.1, np.nan)), "sigma_a.b = nan"),
             (dict(sigma_a=-1e-30), "sigma_a.r = -1e-30"), (dict(sigma_s=-2.0), "sigma_s = -2"),
             (dict(sigma_s=np.inf), "sigma_s = inf"), (dict(g=1.0), "g = 1"), (dict(g=-1.0), "g = -1"),
             (dict(g=np.nan), "g = nan")]
    for change, text in cases:
        with pytest.raises(libs.TptError, match="^set_fog: " + re.escape(text) + "$"):
            fake_ctx.set_fog(**{**GOOD, **change})
    for change, text in ((dict(centre=(0, 0)), "centre must be 3 numbers"),
                         (dict(sigma_a=(0.1, 0.2)), "sigma_a must be a number or 3 numbers"),
                         (dict(radius="x"), "radius, sigma_a, sigma_s and g numbers")):
        with pytest.raises(libs.TptError, match=text):
            fake_ctx.set_fog(**{**GOOD, **change})


def test_fog_reaches_the_library_as_given(libs):
    """A fog arrives as 9 float32 in host memory, in the documented order; a grey sigma_a is repeated; None passes NULL."""
    seen = {}

    class Rec:
        def tpt_set_fog(self, h, ptr):
            seen.update(ptr=ptr, data=None if ptr is None else
                        np.ctypeslib.as_array(ctypes.cast(ptr, ctypes.POINTER(ctypes.c_float)), (9,)).copy())
            return 0

    ctx = libs.Context.__new__(libs.Context)
    ctx._L, ctx._h, ctx.device, ctx.spp = Rec(), ctypes.c_void_p(), 0, 4
    ctx.set_fog(**GOOD)
    assert np.array_equal(seen["data"], np.float32([0, 1, -1.5, 6, 0.01, 0.02, 0.03, 0.1, 0.3]))
    ctx.set_fog((1, 2, 3), 0.5, 0.25, 0.0)
    assert np.array_equal(seen["data"], np.float32([1, 2, 3, 0.5, 0.25, 0.25, 0.25, 0, 0]))
    ctx.set_fog(None)
    assert seen["ptr"] is None


# ---- the pack, the chord and the phase function, through a host build ------------------------------------------------

@pytest.fixture(scope="module")
def fog_lib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("fog_check") / "fog_check.so")
    src = os.path.join(ROOT, "tests", "host_sim", "fog_check.cpp")
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", out, src], check=True)
    L = ctypes.CDLL(out)
    vp = ctypes.c_void_p
    L.pack_blob_fog.argtypes = [vp, vp, ctypes.c_int, vp, ctypes.c_int, ctypes.c_uint, vp, ctypes.c_int, vp, vp,
                                ctypes.c_longlong, vp]
    L.pack_blob_fog.restype = ctypes.c_longlong
    L.fog_offset_of.argtypes = [ctypes.c_uint, ctypes.c_int, ctypes.c_uint]
    L.fog_offset_of.restype = ctypes.c_longlong
    L.fog_chords.argtypes = [vp, vp, ctypes.c_int, vp, vp]
    L.hg_phases.argtypes = [vp, ctypes.c_int, ctypes.c_float, vp]
    return L


LAYOUT = ["offSph", "offMatA", "offMatB", "offLights", "offInvRadius", "offMatRi", "totalBytes", "geomBytes", "flags"]


def pack(L, scene, media=None, fog=None, flags=0):
    s, m = np.ascontiguousarray(scene[0]), np.ascontiguousarray(scene[1])
    n = s.nbytes // 20
    buf = np.zeros(1 << 20, np.uint8)
    lay = np.zeros(29, np.uint32)
    med = None if media is None else np.ascontiguousarray(media, np.float32)
    f9 = None if fog is None else np.ascontiguousarray(fog, np.float32)
    size = L.pack_blob_fog(s.ctypes.data, m.ctypes.data, n, None, 0, flags, None if med is None else med.ctypes.data,
                           0 if med is None else med.shape[0], None if f9 is None else f9.ctypes.data, buf.ctypes.data,
                           buf.size, lay.ctypes.data)
    assert size <= buf.size
    return buf[:size].tobytes(), dict(zip(LAYOUT, (int(v) for v in lay[:9])))


@pytest.fixture(scope="module")
def scene46():
    from toypathtracer_b200 import scenes
    return scenes.reference_scene(1280, 720)


FOG = np.float32([0.0, 1.0, -1.5, 6.0, 0.02, 0.03, 0.05, 0.15, 0.4])


def test_blob_without_fog_keeps_the_parents_bytes(fog_lib, scene46):
    golden = open(os.path.join(ROOT, "tests", "golden", "scene46_blob.bin"), "rb").read()
    blob, lay = pack(fog_lib, scene46)
    assert blob == golden and lay["totalBytes"] == 2720 and lay["flags"] == 0
    # all-zero sigmas are no fog, whatever the ball and g; the caller's flags cannot ask for the section
    zero = FOG.copy()
    zero[4:8] = 0.0
    for fog, flags in ((zero, 0), (None, K_SCENE_FOG)):
        b, l2 = pack(fog_lib, scene46, fog=fog, flags=flags)
        assert b == golden and l2 == lay


@pytest.mark.parametrize("with_media", [False, True])
def test_fog_section_layout(fog_lib, scene46, with_media):
    n = 46
    media = None
    if with_media:
        media = np.zeros((n, 5), np.float32)
        media[7] = (0.3, 0.2, 0.1, 2.0, 0.5)
    plain, lay0 = pack(fog_lib, scene46, media)
    for rec in (FOG, np.float32([1, 2, 3, 0.5, 0, 0, 0, 0.7, -0.2]), np.float32([1, 2, 3, 0.5, 0, 0.1, 0, 0, 0])):
        blob, lay = pack(fog_lib, scene46, media, rec)
        off = int(fog_lib.fog_offset_of(lay["offMatRi"], n, lay["flags"]))
        assert off == lay0["totalBytes"] and len(blob) == off + 48 == lay["totalBytes"]
        assert lay["flags"] == (K_SCENE_MEDIA if with_media else 0) | K_SCENE_FOG
        assert {k: v for k, v in lay.items() if k not in ("totalBytes", "flags")} == \
               {k: v for k, v in lay0.items() if k not in ("totalBytes", "flags")}
        assert blob[:off] == plain
        sec = np.frombuffer(blob, np.float32, 12, off)
        assert np.array_equal(sec[:9], rec) and not sec[9:].any()


def test_scene_layout_did_not_grow():
    src = open(os.path.join(ROOT, "tests", "host_sim", "fog_check.cpp")).read()
    assert "sizeof(tpt::SceneBlobLayout) == 116" in src


def chord64(o, d, t, c, R):
    """Float64 fog length and start of segments o + s d, s in [0, t] (rows), in balls {c, R}."""
    o, d, c = (np.asarray(a, np.float64) for a in (o, d, c))
    dn = d / np.linalg.norm(d, axis=1, keepdims=True)
    p = o - c
    b = (p * dn).sum(1)
    h = p - b[:, None] * dn
    disc = R.astype(np.float64) ** 2 - (h * h).sum(1)
    q = np.sqrt(np.maximum(disc, 0))
    a = np.maximum(-b - q, 0)
    L = np.where(disc > 0, np.maximum(np.minimum(q - b, t) - a, 0), 0.0)
    return L, np.where(L > 0, a, 0.0)


def run_chords(lib, o, d, t, c, R):
    n = len(o)
    seg = np.concatenate([o, d, t[:, None], c], 1).astype(np.float32)
    R = np.ascontiguousarray(R, np.float32)
    L = np.zeros(n, np.float32)
    tin = np.zeros(n, np.float32)
    lib.fog_chords(seg.ctypes.data, R.ctypes.data, n, L.ctypes.data, tin.ctypes.data)
    return L.astype(np.float64), tin.astype(np.float64), seg


def test_chord_matches_float64(fog_lib):
    """Random segments of every kind: origins inside and outside the ball, misses, near-tangent lines, segments that end
    before the ball, inside it or leave the scene (t = TPT_MAX_T), with R from 1e-2 to 1e3. The float32 helper is within
    a few ulp of the segment's scale S = |o - c| + R + |t| in the start and the length, plus the sqrt(u) S that a
    near-tangent line's half-chord q = sqrt(R^2 - |h|^2) can lose to the rounding of |h|^2."""
    rng = np.random.default_rng(3)
    n = 200_000
    R = 10.0 ** rng.uniform(-2, 3, n)
    c = rng.normal(scale=3.0, size=(n, 3)) * R[:, None]
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    kind = rng.integers(0, 4, n)
    # inside, outside towards the ball, outside anywhere, near-tangent
    off = rng.normal(size=(n, 3))
    off /= np.linalg.norm(off, axis=1, keepdims=True)
    o = np.where((kind == 0)[:, None], c + off * (R * rng.uniform(0, 0.999, n))[:, None], 0.0)
    far = R * rng.uniform(1.01, 20, n)
    aim = c - d * far[:, None]                                   # d points at c
    o = np.where((kind == 1)[:, None], aim + np.cross(d, off) * (R * rng.uniform(0, 0.99, n))[:, None], o)
    o = np.where((kind == 2)[:, None], c + off * far[:, None], o)
    perp = np.cross(d, off)
    perp /= np.linalg.norm(perp, axis=1, keepdims=True)
    o = np.where((kind == 3)[:, None], aim + perp * (R * (1 + rng.uniform(-1e-3, 1e-3, n)))[:, None], o)
    t = np.where(rng.random(n) < 0.2, TPT_MAX_T, rng.uniform(0, 1, n) * (far + 2 * R))
    t[rng.random(n) < 0.05] = 1e-3
    L, tin, seg = run_chords(fog_lib, o, d, t, c, R)
    # the reference from the float32 inputs the helper saw
    o32, d32, t32, c32 = (seg[:, 0:3], seg[:, 3:6], seg[:, 6].astype(np.float64), seg[:, 7:10])
    L64, tin64 = chord64(o32, d32, t32, c32, R.astype(np.float32))
    S = np.linalg.norm(o32.astype(np.float64) - c32, axis=1) + R + np.where(t32 < TPT_MAX_T, t32, 0)
    u = 2.0 ** -24
    tol = 16 * u * S + np.sqrt(16 * u) * S
    bad = (np.abs(L - L64) > tol) | ((L > 0) & (np.abs(tin - tin64) > tol))
    assert not bad.any(), [(int(i), kind[i], L[i], L64[i], tin[i], tin64[i], tol[i]) for i in np.nonzero(bad)[0][:5]]
    # away from tangency the sqrt term is not needed
    q2 = (R.astype(np.float64) ** 2 - ((o32 - c32 - ((o32 - c32) * d32).sum(1)[:, None] * d32) ** 2).sum(1))
    clear = q2 > 1e-2 * R ** 2
    assert (np.abs(L - L64)[clear] <= 64 * u * S[clear]).all()
    # every kind happened, with hits and misses
    for k in range(4):
        assert (L[kind == k] > 0).any() and (kind == k).sum() > 1000
    assert (L[kind == 2] == 0).any() and (L[kind == 3] == 0).any()


def test_chord_edge_cases(fog_lib):
    o = np.float32([[0, 0, 0], [0, 0, 0], [0, 0, 5], [0, 0, 5], [0, 0, 5], [0, 2, 5], [0, 0, -5]])
    d = np.float32([[0, 0, 1], [0, 0, 1], [0, 0, -1], [0, 0, -1], [0, 0, 1], [0, 0, -1], [0, 0, -1]])
    t = np.float32([0.5, TPT_MAX_T, 2.0, 5.0, TPT_MAX_T, TPT_MAX_T, TPT_MAX_T])
    c = np.zeros((7, 3), np.float32)
    R = np.full(7, 1.0, np.float32)
    L, tin, _ = run_chords(fog_lib, o, d, t, c, R)
    # inside, ends inside | inside, leaves | ends before the ball | ends at its centre | points away | misses | behind
    assert L.tolist() == [0.5, 1.0, 0.0, 1.0, 0.0, 0.0, 0.0]
    assert tin.tolist() == [0.0, 0.0, 0.0, 4.0, 0.0, 0.0, 0.0]


def phases(lib, cos, g):
    cos = np.ascontiguousarray(cos, np.float32)
    out = np.zeros(cos.size, np.float32)
    lib.hg_phases(cos.ctypes.data, cos.size, g, out.ctypes.data)
    return out.astype(np.float64)


@pytest.mark.parametrize("g", [-0.9, -0.5, -1e-3, -5e-4, 0.0, 3e-4, 0.2, 0.7, 0.95])
def test_phase_integrates_to_one(fog_lib, g):
    """2 pi times the integral of p over cos in [-1, 1] is 1 (Gauss-Legendre on a graded mesh), and p is the closed form
    in float64; below |g| = 1e-3 it is exactly float32(1 / (4 pi))."""
    g32 = float(np.float32(g))
    g_ = np.geomspace(1e-9, 1, 300)                                   # graded towards both poles, where lobes peak
    edges = np.unique(np.concatenate([[-1.0], -1 + g_, 1 - g_, [1.0]]))
    x, w = np.polynomial.legendre.leggauss(12)
    a, b = edges[:-1, None], edges[1:, None]
    cs = (a + (b - a) * (x + 1) / 2).reshape(-1)
    ws = ((b - a) / 2 * w).reshape(-1)
    p = phases(fog_lib, cs, g32)
    if abs(g32) < 1e-3:
        assert (p == np.float64(np.float32(1 / (4 * np.pi)))).all()
    else:
        c32 = cs.astype(np.float32).astype(np.float64)
        den = 1 + g32 * g32 - 2 * g32 * c32
        want = (1 - g32 * g32) / (4 * np.pi * den ** 1.5)
        # float32 cancellation in 1 + g^2 - 2 g cos where the lobe peaks: 1.5 x the rounding of its terms over den
        rel = 1e-6 + 1.5 * 8 * 2.0 ** -24 * (1 + g32 * g32 + 2 * abs(g32)) / den
        assert (np.abs(p - want) <= rel * want).all()
    assert abs(2 * np.pi * (p * ws).sum() - 1) < 2e-5


@pytest.mark.skipif(shutil.which("cuobjdump") is None or shutil.which("cu++filt") is None or not os.path.exists(LIB),
                    reason="needs cuobjdump and the built library")
def test_fog_instances_have_no_stack_and_no_local_memory():
    """The fog step lives in the texture instances only; at their register caps it must not spill."""
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
