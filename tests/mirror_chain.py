"""All-mirror scenes whose every sample is deterministic at every depth, and their answer in float64, ray by ray.

Scene: a "mirror corridor" — a floor and a ceiling, Metal spheres of radius 100 whose facing surfaces are 3 apart
(y = -1.5 and y = +1.5 at x = z = 0), and small Metal spheres between them. Every material is Metal with roughness 0, so
a sample draws no random number that matters (path_step skips the lobe when roughness == 0; the exact mode and the
reference-GPU shader draw it and multiply it by 0) and its value is the chain's
    v = sum_k T_k E_k + T_end sky(d_end),      T_k = product of the albedos of hits 0 .. k-1,
with rays traced = segments. Albedos are on a grid of 1/64 and emissions on one of 1/8, so a wrong hit changes v by far
more than the tolerance. Two rules end a chain (the nearest hit of segment k is hit k, k = 0, 1, ...):
  cpu  fast and exact mode (Test.cpp:195-218, tpt_fast.cu path_step): segment 10 (depth 10 = TPT_MAX_DEPTH) adds its hit's
       emission and ends the chain: at most 11 segments, with a terminal emission.
  gpu  reference-GPU mode (ComputeShader.hlsl:300, tpt_refgpu.cuh): the loop runs 10 segments; the 10th hit adds its
       emission and the chain ends without a terminal sky or emission: at most 10 segments.
A miss at segment k adds T_k sky(d_k) and ends the chain under both rules (the gpu rule only for k <= 9).

The chain oracle traces every segment with test_sweep_oracle's pair_bounds / classify in float64. After the first segment
the kernel's origin and direction are no longer the exact float32 inputs: the bounds are widened by the propagated
uncertainties eps_o (origin) and eps_d (direction), carried through pos = o + t d (the root's rounding enclosure, and the
ray's displacement projected onto the surface along d), the normal (pos - s) * invRadius (the float32 invRadius the blob stores), reflect and the approximate normalize (rsqrt). A ray
is well conditioned when every segment is (one decided winner, no padded sphere that may be hit, a reflected direction
clearly above the surface)."""
from __future__ import annotations

import numpy as np

import furnace as F
import test_sweep_oracle as so
from toypathtracer_b200 import CAMERA_DTYPE, MATERIAL_DTYPE, SPHERE_DTYPE

U = 2.0 ** -24
CAP = {"cpu": 11, "gpu": 10}           # most segments a chain has under each rule
DIR_ERR = 2.0 ** -19                   # |normalize(d) - d / |d|| of a caller or camera ray on the GPU, generously
NORM_ERR = 2.0 ** -20                  # relative error of the kernel's normalize (rsqrt.approx 2^-22.9, dot, scaling)
SKY_SLOPE = 0.075                      # max |d sky / d d_y| of the gradient sky (furnace.sky_affine: 0.15 (c - 1))
FLOOR_Y, CEIL_Y, BIG_R = -1.5, 1.5, 100.0
METAL = 1


# ---- scenes --------------------------------------------------------------------------------------------------------
def corridor(count: int, layout: str, seed: int = 0):
    """`count` Metal spheres (roughness 0): sphere 0 the floor, sphere 1 the ceiling, the rest small spheres between them.
    compact: small spheres with |s| <= 8, so every sphere passes the expanded-form gate (|s|^2 <= 128 + 2 r^2);
    spread:  small spheres over x, z in [-40, 40] (one of them at |s| > 20), which fails it from 3 spheres on (the floor
             and the ceiling alone pass it).
    Albedos k/64 (floor and ceiling 48..63, small spheres 16..63); the floor, the ceiling and a quarter of the small
    spheres emissive (k/8), so that the cap's terminal emission is never zero. Returns (spheres, materials, emissive ids)."""
    rng = np.random.default_rng(seed * 7919 + count * 2 + (layout == "spread"))
    sph = np.zeros(count, SPHERE_DTYPE)
    mats = np.zeros(count, MATERIAL_DTYPE)
    sph[0] = ((0, FLOOR_Y - BIG_R, 0), BIG_R, 0)
    if count >= 2:
        sph[1] = ((0, CEIL_Y + BIG_R, 0), BIG_R, 0)
    k = max(count - 2, 0)
    if k:
        span = 8.0 if layout == "compact" else 40.0
        rmax = float(np.clip(2.5 / k ** (1 / 3), 0.06, 0.45)) if layout == "compact" else 0.45
        rad = rmax * (0.5 + 0.5 * rng.random(k))
        if layout == "compact":
            dirs = rng.normal(size=(k, 2)); dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
            xz = dirs * np.sqrt(rng.random(k))[:, None] * np.sqrt(span ** 2 - 1.5 ** 2)
        else:
            xz = rng.uniform(-span, span, (k, 2))
            xz[0] = (24.0, -18.0)
        y = rng.uniform(-1.0, 1.0, k) * (1.45 - rad)
        sph["center"][2:] = np.stack([xz[:, 0], y, xz[:, 1]], 1)
        sph["radius"][2:] = rad
    sph["invRadius"] = (np.float32(1) / sph["radius"]).astype(np.float32)
    mats["type"] = METAL
    mats["albedo"] = rng.integers(16, 64, (count, 3)) / 64.0
    mats["albedo"][:2] = rng.integers(48, 64, (min(count, 2), 3)) / 64.0
    em = np.zeros(count, bool)
    em[2:] = rng.random(k) < 0.25
    em[:2] = True                                      # a chain that reaches the cap ends on an emissive sphere
    mats["emissive"][em] = rng.integers(1, 17, (int(em.sum()), 3)) / 8.0
    mats["roughness"] = 0.0
    return sph, mats, np.nonzero(em)[0].astype(np.int32)


def point_camera(o, d):
    """A camera whose every sample of every pixel is the one ray {o, d}: horizontal = vertical = 0, lensRadius = 0,
    lowerLeftCorner = fl32(o + d). Returns (camera, the float32 ray {o, fl32(lowerLeftCorner - o)} the renderers trace)."""
    cam = np.zeros(1, CAMERA_DTYPE)
    o = np.asarray(o, np.float32)
    llc = (o.astype(np.float64) + np.asarray(d, np.float64)).astype(np.float32)
    cam["origin"] = o
    cam["lowerLeftCorner"] = llc
    cam["uu"] = (1, 0, 0); cam["vv"] = (0, 1, 0); cam["ww"] = (0, 0, 1)
    return cam, np.concatenate([o, llc - o]).astype(np.float32)


# ---- rays ----------------------------------------------------------------------------------------------------------
CAMERA_O = np.array([0.0, 0.3, 2.0])


def candidate_rays(sph, n: int, seed: int):
    """A third from (near) the camera position, the rest from sphere surfaces (float32-rounded points, directions
    leaving the surface); the vertical component of the direction log-uniform in [0.002, 0.1] for 30 % of them and
    uniform in [0.1, 0.99] for the rest, so that chains of every length come out: shallow rays run out of the corridor
    after a few bounces, steep ones bounce until the cap."""
    rng = np.random.default_rng(seed)
    raw = np.asarray(sph).view(np.float32).reshape(-1, 5).astype(np.float64)
    c, r = raw[:, :3], raw[:, 3]
    d = rng.normal(size=(n, 3))
    d[:, 1] = 0.0
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    dy = np.where(rng.random(n) < 0.3, 10.0 ** rng.uniform(-2.7, -1, n), rng.uniform(0.1, 0.99, n))
    dy = dy * np.where(rng.random(n) < 0.5, -1, 1)
    d = d * np.sqrt(np.maximum(1 - dy ** 2, 0))[:, None]
    d[:, 1] = dy
    o = np.empty((n, 3))
    cam = np.arange(n) < n // 3
    o[cam] = CAMERA_O + rng.normal(size=(int(cam.sum()), 3)) * 0.3
    m = int((~cam).sum())
    pick = rng.integers(0, len(r), m)
    nrm = rng.normal(size=(m, 3)); nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    big = r[pick] > 50
    if len(r) >= 1:                                    # floor / ceiling: a point of the corridor's surface
        xz = rng.uniform(-4, 4, (m, 2))
        sgn = np.where(c[pick, 1] < 0, 1.0, -1.0)
        top = np.stack([xz[:, 0], sgn * np.sqrt(np.maximum(r[pick] ** 2 - (xz ** 2).sum(1), 0)), xz[:, 1]], 1) / r[pick, None]
        nrm[big] = top[big]
    o[~cam] = c[pick] + nrm * r[pick, None]
    dd = d[~cam]
    flip = (dd * nrm).sum(1) < 0
    dd[flip, 1] = -dd[flip, 1]
    flip = (dd * nrm).sum(1) < 0
    dd[flip] = -dd[flip]
    d[~cam] = dd
    return np.concatenate([o, d], 1).astype(np.float32)


# ---- the chain oracle ------------------------------------------------------------------------------------------------
def _widened(o, d, eo, ed, s, r2, expanded):
    """pair_bounds for a kernel ray within eo of o and ed of d (per ray, [R,1]): |d nb| <= |d| eo + |s - o| ed + eo ed,
    |d c| <= 2 |s - o| eo + eo^2, plus the rounding of co = fl32(s - o') at a point that is not o (u per component)."""
    nb, c, enb, ec = so.pair_bounds(o, d, s, r2, expanded)
    co = s - o
    aco = np.abs(co)
    dist = np.sqrt((co * co).sum(-1))
    dn = np.sqrt((d * d).sum(-1))
    enb = enb * (1 + 1e-6) + dn * eo + dist * ed + eo * ed + 1.01 * U * (aco * np.abs(d)).sum(-1)
    ec = ec * (1 + 1e-6) + 2 * dist * eo + eo * eo + 2.01 * U * (aco * aco).sum(-1)
    return nb, c, enb, ec


def _nearest(o, d, eo, ed, S, R2, expanded, count, self_id=None, eo_self=None, chunk=1 << 21):
    """so.nearest_hit with per-ray uncertainties (no duplicate spheres in these scenes). Returns id, t, tlo, thi, well;
    [tlo, thi] encloses the root the kernel computes for its ray.
    Each pair is decided twice. (a) The float32 rounding alone at the ideal ray (eo = ed = 0): outcome and root
    enclosure. (b) The ray's displacement: a rejection must also hold with nb, c widened by eo, ed (_widened); an
    accepted root moves, to first order, by dt = -(r n.do + t (o - s).dd) / (r d.n) (differentiate |o + t d - s|^2 = R
    with the kernel's |d| = 1 assumption), and (o - s) = r n - t d, so |dt| <= (eo + t ed) / cos + t^2 |d.dd| / (r cos)
    with |d.dd| <= NORM_ERR + ed^2 (a direction error is a rotation to first order); 10 % is added for the second order,
    and the pair is ambiguous unless dt stays below half the gap sqrt(D) to the other root and the root above tMin.
    self_id / eo_self: per ray, the sphere whose surface the origin lies on and the origin's error along its normal
    (the origin's error within the tangent plane does not move the root near t = 0 that tMin must reject).
    The decomposition (b) alone would be far too loose for the floor and ceiling: their centres are 100 away, so
    |s - o| ed dwarfs the root's real sensitivity t ed."""
    n, ns = len(o), R2.shape[1]
    out = dict(id=np.full(n, -1), t=np.zeros(n), tlo=np.zeros(n), thi=np.zeros(n), well=np.zeros(n, bool),
               dtr=np.zeros(n))
    step = max(1, chunk // ns)
    pad = (count + 3) // 4 * 4 != count
    r_all = np.sqrt(R2)
    for a in range(0, n, step):
        sl = slice(a, a + step)
        oo, dd = o[sl, None, :], d[sl, None, :]
        e1, e2 = eo[sl, None], ed[sl, None]
        zero = np.zeros_like(e1)
        e1b = e1 if self_id is None else np.where(np.arange(ns)[None] == self_id[sl, None], eo_self[sl, None], e1)
        nb, c, enb, ec = _widened(oo, dd, zero, zero, S, R2, expanded)
        cls, t, tlo, thi = so.classify(nb, c, enb, ec)
        acc = cls > 0
        # a rejection holds for the displaced ray when the line passes the sphere by more than the displacement (miss),
        # or when the larger root, moved as above and with its rounding enclosure, stays below tMin (sphere behind)
        D = nb * nb - c
        with np.errstate(invalid="ignore", divide="ignore"):
            miss_gap = np.sqrt(np.maximum(c + R2 - nb * nb, 0.0)) - r_all
            ok_miss = (D <= 0) & (miss_gap > 1.1 * (e1 + np.abs(nb) * e2) + 1e-7)
            tp = nb + np.sqrt(np.maximum(D, 0.0))
            cos_p = np.abs(((oo + tp[..., None] * dd - S) * dd).sum(-1)) / r_all
            dtp = 1.1 * ((e1b + np.abs(tp) * e2) / cos_p + tp * tp * (NORM_ERR + e2 * e2) / (r_all * cos_p))
            nhi = np.abs(nb) + enb
            tphi = nb + enb + np.sqrt(np.maximum(nhi * nhi - (c - ec), 0.0)) * (1 + so.RHO) + U * (nhi + 1)
            ok_behind = (D > 0) & (tphi + dtp < so.T_MIN)
        cls = np.where((cls == 0) & ~(ok_miss | ok_behind), -1, cls)
        tt = np.where(acc, t, 0.0)
        p = oo + tt[..., None] * dd
        cos = np.abs(((p - S) * dd).sum(-1)) / r_all
        with np.errstate(divide="ignore", invalid="ignore"):
            dt = 1.1 * ((e1 + tt * e2) / cos + tt * tt * (NORM_ERR + e2 * e2) / (r_all * cos))
        gap = np.sqrt(np.maximum(nb * nb - c, 0.0))
        bad = acc & ~((dt < 0.5 * gap) & (tlo - dt > so.T_MIN))
        cls = np.where(bad, -1, cls)
        dtr = np.maximum(thi - t, t - tlo)
        tlo = np.where(acc, tlo - dt, tlo)
        thi = np.where(acc, thi + dt, thi)
        m = len(oo)
        rows = np.arange(m)
        w = np.argmin(t, 1)
        hit = np.isfinite(t[rows, w])
        tlo_o = tlo.copy(); tlo_o[rows, w] = np.inf
        well = (cls >= 0).all(1) & (~hit | (thi[rows, w] < tlo_o.min(1)))
        if pad:                       # form 0's padded sphere (10000^3, r^2 = 0) must be certainly rejected
            pc, *_ = so.classify(*_widened(oo, dd, e1, e2, np.full((1, 1, 3), so.PAD), np.zeros((1, 1)), expanded))
            well &= pc[:, 0] == 0
        out["id"][sl] = np.where(hit, w, -1)
        out["t"][sl] = np.where(hit, t[rows, w], 0)
        out["tlo"][sl] = np.where(hit, tlo[rows, w], 0)
        out["thi"][sl] = np.where(hit, thi[rows, w], 0)
        out["dtr"][sl] = np.where(hit, dtr[rows, w], 0)
        out["well"][sl] = well
    return out


def sky(d, mitsuba):
    """Test.cpp:224-232 in float64 for unit directions d [n, 3]."""
    if mitsuba:
        return np.broadcast_to(F.MITSUBA_SKY.astype(np.float64), d.shape).copy()
    return F.gradient_sky(d[:, 1])


def chains(rays, sph, mats, mitsuba=False, expanded=None, dir_err=DIR_ERR):
    """The oracle for rays float32 [n, 6] (directions of any length). Returns a dict:
      ids [n, 11]    the nearest hit of each segment (-1 sky), -2 past the chain's end under the cpu rule
      seg_cpu/gpu    segments traced under each rule
      v_cpu/gpu      [n, 3] the value under each rule
      tol_cpu/gpu    [n] the value tolerance (float32 rounding of the sums and products, and the gradient sky's
                     sensitivity to the direction's uncertainty)
      well           [n] every segment of the cpu rule's chain well conditioned
      cap            [n] the cpu chain reaches the cap (an 11th segment that hits a sphere)."""
    n = len(rays)
    count = len(sph)
    if expanded is None:
        expanded = so.gate_passes(sph)
    centres, r2 = so.scene_arrays(sph)
    S, R2 = centres.astype(np.float64)[None], r2.astype(np.float64)[None]
    inv = sph["invRadius"].astype(np.float64)
    alb, emis = mats["albedo"].astype(np.float64), mats["emissive"].astype(np.float64)
    o = rays[:, :3].astype(np.float64)
    d = rays[:, 3:].astype(np.float64)
    d = d / np.linalg.norm(d, axis=1, keepdims=True)
    eo, ed = np.zeros(n), np.full(n, dir_err)
    self_id, eo_self = np.full(n, -1), np.zeros(n)      # the sphere the origin lies on, the origin's error along its normal
    T, acc, mag = np.ones((n, 3)), np.zeros((n, 3)), np.zeros(n)
    res = dict(ids=np.full((n, 11), -2), seg_cpu=np.zeros(n, int), seg_gpu=np.zeros(n, int), v_cpu=np.zeros((n, 3)),
               v_gpu=np.zeros((n, 3)), tol_cpu=np.zeros(n), tol_gpu=np.zeros(n), well=np.ones(n, bool),
               cap=np.zeros(n, bool))
    alive = np.ones(n, bool)

    def end(idx, rule, k, v, extra):
        res[f"v_{rule}"][idx] = v
        res[f"seg_{rule}"][idx] = k + 1
        m = mag[idx] + np.abs(v).max(1)
        res[f"tol_{rule}"][idx] = (4 * k + 12) * U * m + extra + 1e-9

    for k in range(11):
        idx = np.nonzero(alive)[0]
        if not len(idx):
            break
        h = _nearest(o[idx], d[idx], eo[idx], ed[idx], S, R2, expanded, count, self_id[idx], eo_self[idx])
        res["well"][idx] &= h["well"]
        hid = h["id"]
        res["ids"][idx, k] = hid
        miss = hid < 0
        mi = idx[miss]
        if len(mi):
            sv = T[mi] * sky(d[mi], mitsuba)
            extra = 0.0 if mitsuba else SKY_SLOPE * ed[mi] * T[mi].max(1)
            v = acc[mi] + sv
            end(mi, "cpu", k, v, extra)
            if k < 10:
                end(mi, "gpu", k, v, extra)
            alive[mi] = False
        hi, hid = idx[~miss], hid[~miss]
        if not len(hi):
            continue
        E = T[hi] * emis[hid]
        if k == 10:                                    # the cap: the hit's emission ends the cpu chain
            end(hi, "cpu", k, acc[hi] + E, 0.0)
            res["cap"][hi] = True
            alive[hi] = False
            break
        # the next ray: pos, normal, mirror direction, and how far the kernel's can be from them. The kernel's hit point
        # o' + t' d' is the surface point its ray meets, moved along d' by the rounding of its root (the winner's
        # rounding enclosure dtr) and by the fma. Its ray is displaced by delta = eo + t ed at the hit, which moves the
        # point it meets by the oblique projection onto the tangent plane along d: at most |delta| / cos (10 % added for
        # the second order).
        oo, dd = o[hi], d[hi]
        t = h["t"][~miss]
        dtr = h["dtr"][~miss]
        sw = centres[hid].astype(np.float64)
        pos = oo + t[:, None] * dd
        nrm = (pos - sw) * inv[hid][:, None]
        nn = np.linalg.norm(nrm, axis=1)
        dn = (dd * nrm).sum(1)
        cos = np.abs(dn) / nn
        epos = 1.1 * (eo[hi] + t * ed[hi]) / cos + dtr * (1 + ed[hi]) + 4 * U * (np.linalg.norm(oo, axis=1) + t)
        en = epos * inv[hid] + 4 * U * nn
        refl = dd - 2 * dn[:, None] * nrm
        # reflect is the Householder map I - 2 n n^T (norm max(1, |2|n|^2 - 1|)); a normal error moves it by <= 4 en
        er = ed[hi] * np.maximum(1.0, np.abs(2 * nn * nn - 1)) + en * (2 * np.abs(dn) + 2 * nn + 2 * en) + 24 * U
        rl = np.linalg.norm(refl, axis=1)
        dnext = refl / rl[:, None]
        ednext = 1.01 * er / rl + NORM_ERR
        up = (dnext * nrm).sum(1)
        margin = ednext * nn + en + 1e-6
        res["well"][hi] &= (np.abs(up) > margin) & (cos > 0.02) & np.isfinite(epos)
        inside = up < 0                                # the reflection points into the surface: Metal ends the chain
        acc_h = acc[hi] + E
        mag[hi] += np.abs(E).max(1)
        for rule in ("cpu", "gpu"):
            if inside.any():
                end(hi[inside], rule, k, acc_h[inside], 0.0)
        if k == 9:                                     # the gpu rule's 10th segment: no terminal sky or emission
            go = ~inside
            end(hi[go], "gpu", k, acc_h[go], 0.0)
        alive[hi[inside]] = False
        acc[hi] = acc_h
        T[hi] = T[hi] * alb[hid]
        o[hi], d[hi], eo[hi], ed[hi] = pos, dnext, epos, ednext
        # off the surface the kernel's point is only by the rounding of the root and the fma, and by the curvature over
        # the tangential displacement (the displaced ray's hit point lies on the surface)
        self_id[hi] = hid
        eo_self[hi] = dtr * (1 + ed[hi]) + 4 * U * (np.linalg.norm(oo, axis=1) + t) + epos * epos * inv[hid]
    return res


def pick_chains(res, per_len: int, rng_seed: int = 0, rule: str = "cpu"):
    """Indices of up to `per_len` well-conditioned rays of every segment count 1 .. CAP[rule] under `rule`."""
    rng = np.random.default_rng(rng_seed)
    out = []
    for L in range(1, CAP[rule] + 1):
        cand = np.nonzero(res["well"] & (res[f"seg_{rule}"] == L))[0]
        if len(cand):
            out.append(rng.choice(cand, min(per_len, len(cand)), replace=False))
    return np.sort(np.concatenate(out)) if out else np.zeros(0, int)


def subset(res, sel):
    return {k: v[sel] for k, v in res.items()}


def oracle_scene(count, layout):
    """The scenes test_gpu_mirror_chains.py runs, with their candidate rays and the oracle's results for all of them:
    (spheres, materials, light ids, rays, results). count is a sphere count, "max" (the largest scene the slab queue
    stages, no light table) or "1000L" (1 000 spheres, every one in the light table: <= 1024 spheres with a blob past
    64 KB)."""
    if count == "max":
        from test_gpu_rays import max_queue_count
        n = max_queue_count(0)
    else:
        n = 1000 if count == "1000L" else count
    s, m, em = corridor(n, layout)
    if count == "max":
        em = np.zeros(0, np.int32)
    elif count == "1000L":
        em = np.arange(n, dtype=np.int32)
    rays = candidate_rays(s, 1500 if n <= 1300 else 400, seed=17 + n)
    return s, m, em, rays, chains(rays, s, m)


# ---- coverage table: every __global__ kernel of libtpt_b200.so (as toypathtracer_b200.kernel_signature names it), and
# the check of test_gpu_mirror_chains.py that ties it to an exact multi-bounce answer, or why it is left out. The fast
# (k_fast_*) instances it drives are also each tied to the sample replay by test_gpu_sample_replay.py ----------------------
_Q = [(128, 6, 0), (128, 6, 1), (128, 6, 2), (128, 6, 3), (128, 6, 4), (128, 8, 2), (128, 8, 4),
      (768, 1, 0), (768, 1, 1), (768, 1, 2), (768, 1, 3)]
_S = [(128, 6, 0), (128, 6, 1), (128, 6, 2), (128, 6, 3), (128, 8, 2), (768, 1, 0), (768, 1, 1), (768, 1, 2), (768, 1, 3)]
COVERAGE = {}
for _nl in ("", "_nolight"):
    for _t, _m, _k in _Q:
        COVERAGE[f"k_fast_rays{_nl}<{_t}, {_m}, {_k}>"] = "test_caller_rays"
    for _t, _m, _k in _Q + [(128, 7, k) for k in range(4)]:
        COVERAGE[f"k_fast_queue{_nl}<{_t}, {_m}, {_k}>"] = "test_images"
    for _t, _m, _k in _S:
        for _mo in ("false", "true"):
            COVERAGE[f"k_fast_samples{_nl}<{_t}, {_m}, {_k}, {_mo}>"] = "test_pixel_lists"
    for _k in range(3):
        for _a in ("false", "true"):
            COVERAGE[f"k_fast_group{_nl}<6, {_k}, {_a}>"] = "test_images"
for _k in range(3):
    COVERAGE[f"k_fast_tileq<6, {_k}>"] = "test_images"
for _n in ("k_fast_wave<3>", "k_fast_wave<4>", "k_fast_persistent<2>", "k_fast_persistent<3>", "k_fast_mega",
           "k_refgpu<true, RgSetupPlain<true>>", "k_refgpu<false, RgSetupPlain<false>>", "k_refgpu<false, RgSetupK2>",
           "k_trace_exact<1>", "k_trace_exact<8>", "k_trace_exact<32>", "k_trace_exact_flat<1>", "k_trace_exact_flat<8>",
           "k_trace_exact_split<1, 0, 1>", "k_trace_exact_split<2, 0, 1>", "k_trace_exact_split<3, 0, 1>",
           "k_trace_exact_split<4, 0, 1>", "k_trace_exact_split<2, 0, 2>", "k_trace_exact_cluster"):
    COVERAGE[_n] = "test_images"
for _r in (False, True):
    for _k in range(4):
        COVERAGE[f"k_fast_aov<{str(_r).lower()}, {_k}>"] = ("excluded: first-hit AOVs, no bounce; test_gpu_aovs checks them "
                                                             "against the nearest-hit oracle")
for _k in range(5):
    COVERAGE[f"k_debug_hit<{_k}>"] = "excluded: tpt_debug_hit's diagnostic sweep, checked by test_gpu_sweep_oracle"
COVERAGE["k_debug_libm"] = "excluded: tpt_debug_libm's diagnostic, no ray tracing"
COVERAGE["k_trace_exact_split<2, 1, 1>"] = "excluded: exact_lanes 69, a timing probe whose image is not valid"
COVERAGE["k_trace_exact_split<2, 2, 1>"] = "excluded: exact_lanes 68, a timing probe whose image is not valid"
for _n in ("k_accumulate_rays", "k_check_pixels", "k_prepare_image", "k_resolve_exact", "k_tonemap_rgba8"):
    COVERAGE[_n] = "excluded: not a trace kernel (counters, list check, blend or tone map around one)"
