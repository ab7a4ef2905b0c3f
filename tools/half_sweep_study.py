"""Study of sweep form 5's half-precision pass 1 on the bench scene (46 spheres, 1280x720 camera): for each pass-1
formulation, the mean number of pass-2 trips with the warp maximum over groups of 32 rays, and the share of rays
outside the bound (FP32 fallback), next to each formulation's static pass-1 issue slots per pair of spheres (read off
the sm_90a SASS of the form-4 kernel, DESIGN §3.1c; the behind test's from a build that had it).

Rays: camera rays (scenes.camera_rays) and, from their first hits, the secondary rays of the fast mode's integrator
in its proportions: a Lambert hit casts one shadow ray per light plus a cosine bounce, a metal hit a reflection, a
glass hit a reflection or, standing in for the refraction, the unbent incoming direction (50/50): the glass row is a
rough proxy. Groups of 32 are consecutive rays of one kind, as a warp's
lanes start on neighbouring pixels. CPU only:  python tools/half_sweep_study.py [--pixels N]"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from toypathtracer_b200 import half_sweep as hs  # noqa: E402
from toypathtracer_b200 import scenes  # noqa: E402


def nearest(c, r2, o, d):
    acc = hs.exact_accepts(c, r2, o, d)
    x = c[None].astype(np.float64) - o[:, None]
    nb = (x * d[:, None]).sum(axis=2)
    sq = np.sqrt(np.maximum(nb * nb - (x * x).sum(axis=2) + r2[None], 0))
    t = np.where(nb - sq > 1e-3, nb - sq, nb + sq)
    t = np.where(acc, t, np.inf)
    i = t.argmin(axis=1)
    return np.where(np.isfinite(t.min(axis=1)), i, -1), t.min(axis=1)


def make_rays(npix, seed=1):
    sp, mats, cam, em = scenes.reference_scene(1280, 720)
    c = sp["center"].astype(np.float64)
    r2 = (sp["radius"] * sp["radius"]).astype(np.float32)
    rng = np.random.default_rng(seed)
    cr = scenes.camera_rays(cam, 1280, 720, 1, seed)
    pick = np.sort(rng.choice(len(cr), npix, replace=False))
    cr = cr[pick].astype(np.float64)
    o, d = cr[:, :3], cr[:, 3:]
    sets = {"camera": (o, d)}
    ids, t = nearest(c, r2.astype(np.float64), o, d)
    hit = ids >= 0
    p = o[hit] + t[hit, None] * d[hit]
    n = (p - c[ids[hit]]) / sp["radius"][ids[hit], None]
    typ = mats["type"][ids[hit]]
    # Lambert: cosine bounce and one shadow ray per light
    lam = typ == 0
    rnd = rng.normal(size=(lam.sum(), 3))
    b = n[lam] + rnd / np.linalg.norm(rnd, axis=1, keepdims=True)
    sets["bounce"] = (p[lam], b / np.linalg.norm(b, axis=1, keepdims=True))
    so, sd = [], []
    for li in em:
        lc = c[li] + rng.normal(size=(lam.sum(), 3)) * 0.2
        v = lc - p[lam]
        so.append(p[lam]); sd.append(v / np.linalg.norm(v, axis=1, keepdims=True))
    sets["shadow"] = (np.concatenate(so), np.concatenate(sd))
    met = typ == 1
    dm = d[hit][met]
    rf = dm - 2 * (dm * n[met]).sum(axis=1, keepdims=True) * n[met] + 0.1 * rng.normal(size=dm.shape)
    sets["metal"] = (p[met], rf / np.linalg.norm(rf, axis=1, keepdims=True))
    gl = typ == 2
    dg = d[hit][gl]
    sets["glass"] = (p[gl], np.where(rng.random((gl.sum(), 1)) < 0.5, dg,
                                     dg - 2 * (dg * n[gl]).sum(axis=1, keepdims=True) * n[gl]))
    return sp, sets


def trips(cand):
    k = cand.sum(axis=1)
    k = k[: len(k) // 32 * 32].reshape(-1, 32)
    return float(((k.max(axis=1) + 1) // 2).mean())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pixels", type=int, default=8192)
    a = ap.parse_args()
    sp, sets = make_rays(a.pixels)
    pad = (len(sp) + 3) // 4 * 4 - len(sp)
    c = np.concatenate([sp["center"], np.full((pad, 3), 10000, np.float32)])
    r2 = np.concatenate([(sp["radius"] * sp["radius"]).astype(np.float32), np.zeros(pad, np.float32)])
    real = np.arange(len(c)) < len(sp)
    print("| rays | count | fallback | form 4 trips | half, with behind test | half, no behind test | exact hits |")
    print("|---|---|---|---|---|---|---|")
    print("| pass-1 slots per pair | | | 24 | 17 | 12 | |")
    for name, (o, d) in sets.items():
        o = o.astype(np.float32); d = d.astype(np.float32)
        f4 = hs.fp32_candidates(c, r2, o, d) & real
        h5 = hs.half_pass(c, r2, o, d, True)[0] & real
        h5n = hs.half_pass(c, r2, o, d, False)[0] & real
        ex = hs.exact_accepts(c, r2, o, d) & real
        fb = 1.0 - hs.in_bound(o, d).mean()
        assert not (f4 & ~h5 & hs.in_bound(o, d)[:, None]).any(), "a form 4 candidate is missing from the half pass"
        print(f"| {name} | {len(o)} | {fb:.2%} | {trips(f4):.2f} | {trips(h5):.2f} | {trips(h5n):.2f} | {trips(ex):.2f} |")


if __name__ == "__main__":
    main()
