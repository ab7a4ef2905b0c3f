"""tpt_trace_rays without a GPU: the library exports it, and scenes.camera_rays builds the thin-lens rays of the
reference's Camera::GetRay (Maths.h:437-442). The binding's signature and the wrapper's refusals are checked with the
other caller-buffer calls in test_aovs_api.py."""
import ctypes

import numpy as np


def test_library_exports_trace_rays(libs):
    L = ctypes.CDLL(libs.LIB_PATH)
    assert hasattr(L, "tpt_trace_rays")


def _cam(libs, aperture):
    return libs.make_camera((0.5, 2.0, 6.0), (0.0, 0.5, -1.0), (0, 1, 0), 40.0, 16 / 9, aperture, 5.0)


def _screen_coords(cam, rays):
    """(s, t, lens offset) of pinhole rays: where each direction meets the focus plane, in the camera's screen coordinates."""
    c = {k: cam[k][0].astype(np.float64) for k in ("origin", "lowerLeftCorner", "horizontal", "vertical", "ww")}
    o, d = rays[:, :3].astype(np.float64), rays[:, 3:].astype(np.float64)
    ww = c["ww"] / np.linalg.norm(c["ww"])
    dist = ((c["origin"] - c["lowerLeftCorner"]) @ ww)           # focus distance along -w
    q = o + d * (dist / -(d @ ww))[:, None] - c["lowerLeftCorner"]
    s = q @ c["horizontal"] / (c["horizontal"] @ c["horizontal"])
    t = q @ c["vertical"] / (c["vertical"] @ c["vertical"])
    return s, t, o - c["origin"]


def test_camera_rays_reproduce_the_corner_rays(libs):
    """Zero aperture: every ray starts at the camera origin and points into its own pixel's footprint; the extreme
    rays of the corner pixels come within a small fraction of a pixel of make_camera's four corner rays."""
    w, h, k = 8, 5, 4000
    cam = _cam(libs, 0.0)
    rays = libs.camera_rays(cam, w, h, per_pixel=k, seed=3)
    assert rays.shape == (w * h * k, 6) and rays.dtype == np.float32
    assert np.abs(np.linalg.norm(rays[:, 3:].astype(np.float64), axis=1) - 1).max() < 1e-6
    s, t, off = _screen_coords(cam, rays)
    assert np.abs(off).max() < 1e-6
    pix = np.arange(len(rays)) // k
    x, y = pix % w, pix // w
    eps = 1e-5
    assert ((s * w >= x - eps) & (s * w <= x + 1 + eps)).all() and ((t * h >= y - eps) & (t * h <= y + 1 + eps)).all()
    for (cx, cy), (su, tv) in {(0, 0): (0, 0), (w - 1, 0): (1, 0), (0, h - 1): (0, 1), (w - 1, h - 1): (1, 1)}.items():
        m = (x == cx) & (y == cy)
        d2 = (s[m] - su) ** 2 * w * w + (t[m] - tv) ** 2 * h * h           # squared distance in pixels
        assert d2.min() < 0.03 ** 2, (cx, cy, d2.min())
    # the rays' mean direction over the image is the ray through the screen centre
    centre = cam["lowerLeftCorner"][0] + 0.5 * cam["horizontal"][0] + 0.5 * cam["vertical"][0] - cam["origin"][0]
    sc, tc, _ = _screen_coords(cam, np.concatenate([cam["origin"][0], centre / np.linalg.norm(centre)])[None].astype(np.float32))
    assert abs(s.mean() - sc[0]) < 2e-3 and abs(t.mean() - tc[0]) < 2e-3


def test_camera_rays_sample_the_lens_disk(libs):
    """With an aperture the origins fill the lens disk uniformly (radius lensRadius in the camera's u, v plane) and every
    ray still passes through its pixel's footprint on the focus plane."""
    w, h, k = 4, 3, 20000
    cam = _cam(libs, 0.4)
    R = float(cam["lensRadius"][0])
    rays = libs.camera_rays(cam, w, h, per_pixel=k, seed=5)
    s, t, off = _screen_coords(cam, rays)
    uu, vv, ww = (cam[n][0].astype(np.float64) for n in ("uu", "vv", "ww"))
    r = np.linalg.norm(off, axis=1)
    assert r.max() <= R * (1 + 1e-6)
    assert np.abs(off @ ww).max() < 1e-6                                 # in the lens plane
    # uniform on the disk: P(r < a R) = a^2, and no preferred direction
    for a in (0.25, 0.5, 0.75):
        assert abs((r < a * R).mean() - a * a) < 0.01, a
    assert abs((off @ uu).mean()) < 0.01 * R and abs((off @ vv).mean()) < 0.01 * R
    pix = np.arange(len(rays)) // k
    eps = 1e-4
    assert ((s * w >= pix % w - eps) & (s * w <= pix % w + 1 + eps)).all()
    assert ((t * h >= pix // w - eps) & (t * h <= pix // w + 1 + eps)).all()
    again = libs.camera_rays(cam, w, h, per_pixel=k, seed=5)
    assert (again == rays).all() and not (libs.camera_rays(cam, w, h, per_pixel=k, seed=6) == rays).all()
