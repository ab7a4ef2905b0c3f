"""Scene inputs: the reference's 46-sphere scene (through the drop-in's own GetSceneDesc) and the procedural
4096-sphere stress scene of BASELINE.json configs[4] (the reference has no such scene: its scene is a static
array, Cpp/Source/Test.cpp:13-64, and its GPU shaders cap at kCSMaxObjects = 64, Config.h:30)."""
from __future__ import annotations

import numpy as np

_F = np.float32


def make_camera(lookfrom, lookat, vup, vfov, aspect, aperture, focus_dist) -> np.ndarray:
    """The reference's Camera constructor (Cpp/Source/Maths.h:418-435) in float32. For runtime scenes the camera is
    plain input data shared by the oracle and the kernels, so only self-consistency matters here; for the
    reference scene use UpdateTest()/GetSceneDesc(), which is bit-identical to the reference."""
    from . import CAMERA_DTYPE
    f = lambda v: np.asarray(v, _F)
    lookfrom, lookat, vup = f(lookfrom), f(lookat), f(vup)
    norm = lambda v: (v * (_F(1) / np.sqrt(np.dot(v, v), dtype=_F))).astype(_F)
    theta = _F(vfov) * _F(3.1415926) / _F(180)
    half_h = _F(np.tan(theta / _F(2)))
    half_w = _F(aspect) * half_h
    w = norm(lookfrom - lookat)
    u = norm(np.cross(vup, w).astype(_F))
    v = np.cross(w, u).astype(_F)
    fd = _F(focus_dist)
    cam = np.zeros(1, CAMERA_DTYPE)
    cam["origin"] = lookfrom
    cam["lowerLeftCorner"] = lookfrom - half_w * fd * u - half_h * fd * v - fd * w
    cam["horizontal"] = _F(2) * half_w * fd * u
    cam["vertical"] = _F(2) * half_h * fd * v
    cam["uu"], cam["vv"], cam["ww"] = u, v, w
    cam["lensRadius"] = _F(aperture) / _F(2)
    return cam


def camera_rays(camera, width: int, height: int, per_pixel: int = 1, seed: int = 0) -> np.ndarray:
    """Rays of the thin-lens camera (Camera::GetRay, Cpp/Source/Maths.h:437-442) for Context.trace_rays: an
    (width * height * per_pixel, 6) float32 array {o.xyz, d.xyz}, `per_pixel` rays per pixel, each with a uniform jitter
    inside its pixel and a uniform sample of the lens disk. Pixel-major: the rays of pixel (x, y) are rows
    (y * width + x) * per_pixel + k, with row y = 0 at the bottom like the backbuffer. Computed in float64 from the float32
    camera, unit directions, deterministic in `seed`."""
    cam = {k: np.asarray(camera[k], np.float64).reshape(-1)
           for k in ("origin", "lowerLeftCorner", "horizontal", "vertical", "uu", "vv", "lensRadius")}
    rng = np.random.default_rng(seed)
    n = width * height * per_pixel
    pix = np.arange(n) // per_pixel
    s = (pix % width + rng.random(n)) / width
    t = (pix // width + rng.random(n)) / height
    r = cam["lensRadius"][0] * np.sqrt(rng.random(n))
    phi = 2.0 * np.pi * rng.random(n)
    offset = (r * np.cos(phi))[:, None] * cam["uu"] + (r * np.sin(phi))[:, None] * cam["vv"]
    d = cam["lowerLeftCorner"] + s[:, None] * cam["horizontal"] + t[:, None] * cam["vertical"] - cam["origin"] - offset
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return np.concatenate([cam["origin"] + offset, d], axis=1).astype(np.float32)


def sky_environment(width: int, height: int) -> np.ndarray:
    """The reference's gradient sky (Test.cpp:228-231: 0.3 * lerp(white, (0.5, 0.7, 1.0), (d.y + 1) / 2)) as a lat-long
    map for Context.set_environment: an (height, width, 3) float32 array, texel (i, j) holding the sky at its centre,
    theta = (j + 1/2) / height * pi from the zenith (d.y = cos theta; the sky does not depend on phi). Computed in
    float64. With it the fast mode reproduces the default look up to the map's bilinear error."""
    theta = (np.arange(height, dtype=np.float64) + 0.5) / height * np.pi
    t = 0.5 * (np.cos(theta) + 1.0)
    col = ((1.0 - t)[:, None] * np.ones(3) + t[:, None] * np.array([0.5, 0.7, 1.0])) * 0.3
    return np.ascontiguousarray(np.broadcast_to(col[:, None, :], (height, width, 3)), dtype=np.float32)


def reference_scene(width: int, height: int, time: float = 0.0, flags: int = 0, big_scene: bool = True,
                    mitsuba_compare: bool = False):
    """(spheres, materials, camera, emissives) of the reference scene at this aspect ratio, produced by the
    drop-in's UpdateTest + GetSceneDesc (host code only; works without a GPU). big_scene / mitsuba_compare select the
    reference's DO_BIG_SCENE (Test.cpp:10-11) and DO_MITSUBA_COMPARE (Config.h:25) variants; the latter only changes
    the camera here (zero aperture) — pass Context.set_option("mitsuba_compare", 1) for its integrator effects."""
    from . import UpdateTest, GetSceneDesc, reset_scene, set_variant
    set_variant(big_scene, mitsuba_compare)
    UpdateTest(time, 0, width, height, flags)
    out = GetSceneDesc()
    set_variant(True, False)
    return out


class _XorShift:
    def __init__(self, seed):
        self.s = seed & 0xFFFFFFFF

    def f01(self) -> float:
        x = self.s
        x ^= (x << 13) & 0xFFFFFFFF
        x ^= x >> 17
        x ^= (x << 15) & 0xFFFFFFFF
        self.s = x
        return (x & 0xFFFFFF) / 16777216.0


def stress_scene(width: int, height: int, count: int = 4096, seed: int = 0x9E3779B9):
    """Procedural stress scene (BASELINE.json configs[4], constants after SURVEY.md §8d): sphere 0 = ground
    (0,-1000,0) r=1000; the rest on a jittered 1.0-pitch grid centred on the origin, radius 0.2-0.35 resting on the
    ground; material by draw (<0.6 Lambert, <0.9 Metal with roughness = draw*0.5, else Dielectric ri 1.5); 6
    emissive Lambert spheres r=0.5 raised to y=3 (emission 10-30). Deterministic: XorShift32 (Maths.cpp:5-13)."""
    from . import SPHERE_DTYPE, MATERIAL_DTYPE
    rng = _XorShift(seed | 1)
    spheres = np.zeros(count, SPHERE_DTYPE)
    mats = np.zeros(count, MATERIAL_DTYPE)
    spheres[0] = ((0, -1000, 0), 1000, 0)
    mats[0] = (0, (0.5, 0.5, 0.5), (0, 0, 0), 0, 0)
    side = int(np.ceil(np.sqrt(count - 1)))
    n_lights = 6
    light_every = max(1, (count - 1) // n_lights)
    for i in range(1, count):
        gx, gz = (i - 1) % side, (i - 1) // side
        jx, jz = rng.f01(), rng.f01()
        r = 0.2 + 0.15 * rng.f01()
        x = (gx - side / 2 + 0.15 + 0.7 * jx) * 1.0
        z = (gz - side / 2 + 0.15 + 0.7 * jz) * 1.0 - side / 4
        t = rng.f01()
        col = (0.1 + 0.8 * rng.f01(), 0.1 + 0.8 * rng.f01(), 0.1 + 0.8 * rng.f01())
        if (i - 1) % light_every == light_every // 2 and (i - 1) // light_every < n_lights:
            e = 10 + 20 * rng.f01()
            spheres[i] = ((x, 3.0, z), 0.5, 0)
            mats[i] = (0, col, (e, e * 0.9, e * 0.7), 0, 0)
        elif t < 0.6:
            spheres[i] = ((x, r, z), r, 0)
            mats[i] = (0, col, (0, 0, 0), 0, 0)
        elif t < 0.9:
            spheres[i] = ((x, r, z), r, 0)
            mats[i] = (1, col, (0, 0, 0), 0.5 * rng.f01(), 0)
        else:
            spheres[i] = ((x, r, z), r, 0)
            mats[i] = (2, (1, 1, 1), (0, 0, 0), 0, 1.5)
    spheres["invRadius"] = (_F(1) / spheres["radius"]).astype(_F)
    cam = make_camera((0, 6, 14), (0, 0, -side / 4), (0, 1, 0), 50, width / height, 0.02, 16)
    em = np.nonzero((mats["emissive"] > 0).any(axis=1))[0].astype(np.int32)
    return spheres, mats, cam, em
